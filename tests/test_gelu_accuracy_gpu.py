"""The GELU of the GEMM epilogues and of dvt_gelu, and the GELU derivative of the backward epilogue, over every bf16 input.

The pre-activations reach the epilogue exactly: A [512, 128] holds all 65 536 bf16 bit patterns and B is the 128 x 128
identity, so the fp32 accumulator of element (m, n) is A[m, n] itself.  The 65 280 finite patterns fill rows 0..509; the
256 patterns with an all-ones exponent (+-inf and the NaNs) fill rows 510 and 511, which the product turns into NaN rows
(inf * 0 and NaN * 0 are NaN), so those rows test NaN propagation.

  - finite x: the fp32 GELU (generic epilogue, SIMT epilogue) is within 1e-6 of fp64 x Phi(x) and the derivative within
    2e-6 of fp64 Phi(x) + x phi(x);
  - the bf16 fast path (gelu_erf2 on pairs) equals the bf16 rounding of the fp32 generic path (gelu_erf), bit for bit;
  - dvt_gelu equals the fc1 epilogue bit for bit;
  - NaN in, NaN out, forward and derivative.  +-inf are implementation-defined (torch's x Phi(x) gives NaN at -inf); the
    kernels give GELU(+inf) = +inf and GELU(-inf) = -3.7e-17, which is pinned here so that a change is noticed."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

BF16, F32 = 0, 1


def _L():
    from dvt import _lib
    return _lib


def _call(name, *args):
    L = _L()
    L.check(getattr(L.lib(), name)(*args), name)


@pytest.fixture(scope="module")
def patterns():
    """A bf16 [512, 128] with every bit pattern once: finite values in rows 0..509, the rest in rows 510..511."""
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    finite_mask = ((bits.int() >> 7) & 0xFF) != 0xFF
    ordered = torch.cat([bits[finite_mask], bits[~finite_mask]])
    assert ordered.numel() == 65536 and int(finite_mask.sum()) == 510 * 128
    a = ordered.view(torch.bfloat16).reshape(512, 128).cuda()
    x64 = a.double()
    finite = torch.zeros(512, 128, dtype=torch.bool, device="cuda")
    finite[:510] = True
    assert bool(torch.isfinite(x64[:510]).all()) and not bool(torch.isfinite(x64[510:]).any())
    return a, x64, finite


def _gemm_gelu(a, out_dtype):
    eye = torch.eye(128, device="cuda", dtype=torch.bfloat16)
    out = torch.empty(512, 128, device="cuda", dtype=torch.bfloat16 if out_dtype == BF16 else torch.float32)
    _call("dvt_gemm_tn", a.data_ptr(), 128, eye.data_ptr(), 128, BF16, 512, 128, 128, None, 1, out.data_ptr(), 128,
          out_dtype, 1, _L().cur_stream())
    torch.cuda.synchronize()
    return out


def _ref_gelu(x64):
    return x64 * 0.5 * (1.0 + torch.erf(x64 / math.sqrt(2.0)))


def _ref_gelu_grad(x64):
    return 0.5 * (1.0 + torch.erf(x64 / math.sqrt(2.0))) + x64 * torch.exp(-0.5 * x64 * x64) / math.sqrt(2.0 * math.pi)


def _max_err(got, ref, mask):
    return (got.double() - ref).abs()[mask].max().item()


def test_gelu_generic_and_fast_paths(patterns):
    a, x64, finite = patterns
    f32 = _gemm_gelu(a, F32)                       # generic epilogue: gelu_erf per element
    b16 = _gemm_gelu(a, BF16)                      # fast path: gelu_erf2 on pairs, bf16 pack
    ref = _ref_gelu(x64)
    err = _max_err(f32, ref, finite)
    assert err <= 1e-6, f"fp32 GELU max abs error {err:.3g} over the finite bf16 inputs"
    assert bool(torch.isnan(f32[~finite]).all()), "GELU(NaN) must be NaN (generic epilogue)"
    assert bool(torch.isnan(b16[~finite]).all()), "GELU(NaN) must be NaN (bf16 fast path)"
    rounded = f32[finite].bfloat16()
    same = b16[finite].view(torch.int16) == rounded.view(torch.int16)
    assert bool(same.all()), (f"bf16 fast path differs from the rounded generic path on {int((~same).sum())} inputs, e.g. "
                              f"x={a[finite][~same][:4].tolist()}")
    assert _L().device_error() == 0


def test_gelu_simt_path(patterns):
    a, x64, finite = patterns
    tc = _gemm_gelu(a, F32)
    _L().check(_L().lib().dvt_set_debug_impl(1))
    try:
        simt = _gemm_gelu(a, F32)
    finally:
        _L().check(_L().lib().dvt_set_debug_impl(-1))
    err = _max_err(simt, _ref_gelu(x64), finite)
    assert err <= 1e-6, f"SIMT fp32 GELU max abs error {err:.3g}"
    assert bool(torch.isnan(simt[~finite]).all()), "GELU(NaN) must be NaN (SIMT epilogue)"
    assert torch.equal(simt[finite].view(torch.int32), tc[finite].view(torch.int32)), "SIMT and tensor-core GELU differ"
    assert _L().device_error() == 0


def test_dvt_gelu_matches_the_fc1_epilogue(patterns):
    a, x64, finite = patterns
    out = torch.empty_like(a)
    _call("dvt_gelu", a.data_ptr(), out.data_ptr(), a.numel(), _L().cur_stream())
    torch.cuda.synchronize()
    fc1 = _gemm_gelu(a, BF16)
    assert torch.equal(out[finite].view(torch.int16), fc1[finite].view(torch.int16)), "dvt_gelu differs from the fc1 epilogue"
    # dvt_gelu sees the non-finite inputs themselves
    xs = x64[~finite]
    got = out[~finite].double()
    nan_in = torch.isnan(xs)
    assert bool(torch.isnan(got[nan_in]).all()), "dvt_gelu(NaN) must be NaN"
    assert bool((got[xs == math.inf] == math.inf).all()), "dvt_gelu(+inf) = +inf"
    assert bool((got[xs == -math.inf].abs() < 1e-16).all()), "dvt_gelu(-inf) ~ -3.7e-17"
    assert _L().device_error() == 0


def test_gelu_derivative_epilogue(patterns):
    """dvt_gemm_bf16(..., gelu_preact=X) with A . B^T = 1 everywhere: out = gelu'(X) exactly as the epilogue computes it."""
    pre, x64, _ = patterns
    A = torch.zeros(512, 64, device="cuda", dtype=torch.bfloat16)
    B = torch.zeros(128, 64, device="cuda", dtype=torch.bfloat16)
    A[:, 0] = 1
    B[:, 0] = 1
    outs = {}
    for impl in (0, 1):
        _L().check(_L().lib().dvt_set_debug_impl(impl))
        try:
            out = torch.empty(512, 128, device="cuda")
            _call("dvt_gemm_bf16", A.data_ptr(), 64, 0, B.data_ptr(), 64, 0, 512, 128, 64, out.data_ptr(), 128, F32, 1,
                  pre.data_ptr(), 128, None, _L().cur_stream())
            torch.cuda.synchronize()
        finally:
            _L().check(_L().lib().dvt_set_debug_impl(-1))
        outs[impl] = out
    finite = torch.isfinite(x64)
    ref = _ref_gelu_grad(x64)
    for impl, out in outs.items():
        err = _max_err(out, ref, finite)
        assert err <= 2e-6, f"GELU' max abs error {err:.3g} (impl {impl})"
        assert bool(torch.isnan(out[torch.isnan(x64)]).all()), f"GELU'(NaN) must be NaN (impl {impl})"
    assert _L().device_error() == 0
