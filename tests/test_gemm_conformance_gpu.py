"""Conformance of every GEMM entry point and epilogue path against an fp64 reference, at tile edges.

Reference: the fp64 product of the operands the kernel actually multiplies -- the bf16 values for bf16 calls, the
TF32-truncated values (low 13 mantissa bits cleared) for TF32 calls, hi + lo for 3xTF32 -- with the epilogue applied in
fp64 (exact erf GELU, exact GELU derivative).

Bound: per element, scaled by the fp64 absolute product P = |A| . |B|^T, so that cancellation in the sum cannot hide an
error:
  bf16 operands, fp32 accumulation   2^-18 P      (fp32 accumulation over K <= 1000 of products that are exact in fp32)
  3xTF32                             2^-18 P      (the dropped A_lo B_lo term and the TF32 rounding of the lo planes are
                                                   ~2^-22 relative)
  TF32                               2^-9 P       (operands truncated to 10 mantissa bits)
  + 2^-23 |ref|                      fp32 rounding of the epilogue arithmetic (bias add, LayerScale FMA, residual)
  + 2^-8 |ref|                       bf16 output
  + 1e-6 (GELU) / 2e-6 |acc| (GELU')  the polynomial GELU and the fast-erf GELU derivative of the epilogue
  GELU / GELU' scale the accumulator error by their Lipschitz constant (<= 1.13 for both).

The checker's teeth are shown on the host (no GPU needed): simulated wrong results built from the same operands -- one
64-wide k-block dropped, a K tail read as garbage, 3xTF32 without its A_lo B_hi term, plain TF32 in place of 3xTF32, an
M tail shifted by one row -- must all be rejected.

Operands are column windows of wider buffers whose other elements are NaN (a read outside the window poisons the
result); outputs go into a column/row window of a wider NaN-sentinel buffer, and every sentinel outside [M, N] must be
unchanged afterwards (stray tail stores)."""
import math
import zlib

import pytest
import torch

REL_BF16 = 2.0 ** -18
REL_X3 = 2.0 ** -18
REL_TF32 = 2.0 ** -9
LIP = 1.13          # max |d GELU / dx| = 1.1289 (at x = sqrt 2): how far GELU can magnify an accumulator error
BF16, F32 = 0, 1

M_SET = (1, 64, 127, 128, 129, 383)
N_SET = (8, 124, 128, 132, 260, 13, 130)       # 13, 130: N % 4 != 0, the scalar tail (padded ldo)
K_SET = (8, 56, 64, 72, 200, 1000)
# pairwise covering set: every (M, N), (M, K) and (N, K) pair occurs (K = K_SET[(i + j) % 6] runs through all six K for a
# fixed M as j runs over the seven N, and through all six for a fixed N as i runs over the six M)
CASES = [(M_SET[i], N_SET[j], K_SET[(i + j) % 6]) for i in range(6) for j in range(7)]
RAGGED = (383, 130, 1000)


# ------------------------------------------------------------------------------------------------ reference and bound
def tf32_trunc(x):
    return (x.float().contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def gelu64(x):
    return x * 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_grad64(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def excess(out, ref, P, rel, *, lip=1.0, bf16_out=False, abs_extra=0.0, mag=None):
    """max over elements of |out - ref| / bound (> 1: out of bound; NaN in out counts as infinitely far).
    mag: magnitude whose fp32 rounding the epilogue may add (default |ref|)."""
    ref = ref.double()
    mag = ref.abs() if mag is None else mag
    bound = rel * lip * P + 2.0 ** -23 * mag + abs_extra + 1e-300
    if bf16_out:
        bound = bound + 2.0 ** -8 * ref.abs()
    err = (out.double() - ref).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    return (err / bound).max().item()


def assert_close(out, ref, P, rel, what, **kw):
    x = excess(out, ref, P, rel, **kw)
    assert x <= 1.0, f"{what}: error {x:.3g} x the bound"


# ------------------------------------------------------------------------------------------------ CPU self-checks
def _mut_operands(M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g, dtype=torch.float64).float()
    b = torch.randn(N, K, generator=g, dtype=torch.float64).float()
    return a, b


@pytest.mark.parametrize("K", [200, 1000])
def test_selfcheck_rejects_a_dropped_k_block(K):
    a, b = _mut_operands(129, 130, K, 1)
    a, b = a.bfloat16().double(), b.bfloat16().double()
    ref, P = a @ b.T, a.abs() @ b.abs().T
    assert excess(ref.float(), ref, P, REL_BF16) <= 1.0
    bad = ref - a[:, 64:128] @ b[:, 64:128].T
    assert excess(bad.float(), ref, P, REL_BF16) > 1.0


@pytest.mark.parametrize("K", [8, 56, 72, 200])
def test_selfcheck_rejects_a_garbage_k_tail(K):
    a, b = _mut_operands(128, 132, K, 2)
    a, b = a.bfloat16().double(), b.bfloat16().double()
    ref, P = a @ b.T, a.abs() @ b.abs().T
    pad = (K + 63) // 64 * 64 - K
    g = torch.Generator().manual_seed(3)
    ta, tb = (torch.rand(128, pad, generator=g, dtype=torch.float64) * 1e-2,
              torch.rand(132, pad, generator=g, dtype=torch.float64) * 1e-2)     # small garbage, one sign
    bad = ref + ta @ tb.T
    assert excess(bad.float(), ref, P, REL_BF16) > 1.0


@pytest.mark.parametrize("K", [8, 72, 1000])
def test_selfcheck_rejects_3xtf32_without_alo_bhi(K):
    a, b = _mut_operands(127, 124, K, 4)
    ah, bh = tf32_trunc(a).double(), tf32_trunc(b).double()
    al, bl = a.double() - ah, b.double() - bh
    x, y = a.double(), b.double()
    ref, P = x @ y.T, x.abs() @ y.abs().T
    assert excess((ah @ bh.T + ah @ bl.T + al @ bh.T).float(), ref, P, REL_X3) <= 1.0
    assert excess((ah @ bh.T + ah @ bl.T).float(), ref, P, REL_X3) > 1.0
    assert excess((ah @ bh.T).float(), ref, P, REL_X3) > 1.0          # plain TF32 where 3xTF32 is expected


def test_selfcheck_rejects_a_shifted_m_tail():
    a, b = _mut_operands(383, 8, 56, 5)
    a, b = a.bfloat16().double(), b.bfloat16().double()
    ref, P = a @ b.T, a.abs() @ b.abs().T
    bad = ref.clone()
    bad[256:] = ref[255:-1]                                             # rows of the last (ragged) M tile one row off
    assert excess(bad.float(), ref, P, REL_BF16) > 1.0


def test_selfcheck_bf16_output_and_gelu_terms():
    """The bf16-output and GELU terms admit a correctly rounded result, and not a 1-ulp-of-bf16 shift."""
    a, b = _mut_operands(64, 128, 64, 6)
    a, b = a.bfloat16().double(), b.bfloat16().double()
    acc, P = a @ b.T, a.abs() @ b.abs().T
    ref = gelu64(acc)
    good = ref.float().bfloat16()
    assert excess(good, ref, P, REL_BF16, lip=LIP, bf16_out=True, abs_extra=1e-6) <= 1.0
    bits = good.view(torch.int16) + 2                                    # two bf16 ulps off
    assert excess(bits.view(torch.bfloat16), ref, P, REL_BF16, lip=LIP, bf16_out=True, abs_extra=1e-6) > 1.0


# ------------------------------------------------------------------------------------------------ GPU helpers
def _L():
    from dvt import _lib
    return _lib


def _call(name, *args):
    L = _L()
    L.check(getattr(L.lib(), name)(*args), name)


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return _L().cur_stream()


def _window(rows, cols, dtype, gen, lead=None, scale=1.0):
    """[rows, cols] random values (rounded to `dtype`) as a column window of a wider NaN-filled buffer: the returned
    view has stride(0) > cols and starts 16 bytes or more into its row."""
    elem = 2 if dtype == torch.bfloat16 else 4
    al = 16 // elem
    lead = al if lead is None else lead
    width = lead + (cols + al - 1) // al * al + al
    buf = torch.full((rows, width), float("nan"), device="cuda", dtype=dtype)
    v = buf[:, lead:lead + cols]
    v.copy_((torch.randn(rows, cols, device="cuda", generator=gen) * scale).to(dtype))
    return v


def _x3_planes(x):
    """fp32 matrix -> (hi view, plane offset in elements, hi64 + lo64 as fp64): hi / lo planes inside one NaN-padded
    buffer, hi at the returned view, lo `plane` elements further."""
    rows, cols = x.shape
    width = 4 + (cols + 3) // 4 * 4 + 4
    buf = torch.full((2, rows, width), float("nan"), device="cuda", dtype=torch.float32)
    hi = tf32_trunc(x)
    buf[0, :, 4:4 + cols] = hi
    buf[1, :, 4:4 + cols] = x - hi
    return buf[0, :, 4:4 + cols], rows * width, buf


class Out:
    """A [M, N] output window (rows 1..M, columns 4..4+N) of a NaN-sentinel buffer, optionally initialised."""

    def __init__(self, M, N, dtype, init=None, width=None):
        self.M, self.N = M, N
        width = width or 4 + (N + 3) // 4 * 4 + 8
        self.buf = torch.full((M + 2, width), float("nan"), device="cuda", dtype=dtype)
        self.view = self.buf[1:M + 1, 4:4 + N]
        if init is not None:
            self.view.copy_(init)
        self.before = self.buf.clone()

    @property
    def ld(self):
        return self.buf.stride(0)

    def check_sentinels(self, what):
        inside = torch.zeros_like(self.buf, dtype=torch.bool)
        inside[1:self.M + 1, 4:4 + self.N] = True
        it = torch.int16 if self.buf.dtype == torch.bfloat16 else torch.int32
        same = self.buf.view(it) == self.before.view(it)
        assert bool(same[~inside].all()), f"{what}: {int((~same[~inside]).sum())} elements outside [M, N] were written"


class impl_mode:
    def __init__(self, impl):
        self.impl = impl

    def __enter__(self):
        _L().check(_L().lib().dvt_set_debug_impl(self.impl))

    def __exit__(self, *a):
        _L().check(_L().lib().dvt_set_debug_impl(-1))


def _gen(*key):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(key).encode()))


def _prod(a64, b64):
    return a64 @ b64.T, a64.abs() @ b64.abs().T


# ------------------------------------------------------------------------------------------------ dvt_gemm_tn
def run_gemm_tn(M, N, K, dtype, act, use_bias, out_dtype, gen, repeat=True):
    tdt = torch.bfloat16 if dtype == BF16 else torch.float32
    a = _window(M, K, tdt, gen)
    b = _window(N, K, tdt, gen, scale=K ** -0.5)
    bias = torch.randn(N + 4, device="cuda", generator=gen)[:N] if use_bias else None
    odt = torch.bfloat16 if out_dtype == BF16 else torch.float32
    results = []
    for _ in range(2 if repeat else 1):
        o = Out(M, N, odt)
        _call("dvt_gemm_tn", _p(a), a.stride(0), _p(b), b.stride(0), dtype, M, N, K, _p(bias), act, _p(o.view), o.ld,
              out_dtype, 1, _stream())
        results.append(o)
    torch.cuda.synchronize()
    if dtype == BF16:
        a64, b64, rel = a.double(), b.double(), REL_BF16
    else:
        a64, b64, rel = tf32_trunc(a).double(), tf32_trunc(b).double(), REL_TF32
    acc, P = _prod(a64, b64)
    pre = acc + (bias.double() if use_bias else 0.0)
    ref = {0: pre, 1: gelu64(pre), 2: pre.clamp_min(0.0)}[act]
    what = f"dvt_gemm_tn M={M} N={N} K={K} dtype={dtype} act={act} bias={use_bias} out={out_dtype}"
    o = results[0]
    o.check_sentinels(what)
    assert_close(o.view, ref, P, rel, what, lip=LIP if act == 1 else 1.0, bf16_out=out_dtype == BF16,
                 abs_extra=1e-6 if act == 1 else 0.0, mag=pre.abs())
    if repeat:
        it = torch.int16 if odt == torch.bfloat16 else torch.int32
        assert torch.equal(results[0].buf.view(it), results[1].buf.view(it)), f"{what}: second run differs"


def run_gemm_tn_splitk(M, N, K, dtype, splits, gen):
    tdt = torch.bfloat16 if dtype == BF16 else torch.float32
    a = _window(M, K, tdt, gen)
    b = _window(N, K, tdt, gen, scale=K ** -0.5)
    o = Out(M, N, torch.float32, init=torch.zeros(M, N, device="cuda"))
    _call("dvt_gemm_tn", _p(a), a.stride(0), _p(b), b.stride(0), dtype, M, N, K, None, 0, _p(o.view), o.ld, F32, splits,
          _stream())
    torch.cuda.synchronize()
    if dtype == BF16:
        a64, b64, rel = a.double(), b.double(), REL_BF16
    else:
        a64, b64, rel = tf32_trunc(a).double(), tf32_trunc(b).double(), REL_TF32
    acc, P = _prod(a64, b64)
    what = f"dvt_gemm_tn split-K M={M} N={N} K={K} dtype={dtype} splits={splits}"
    o.check_sentinels(what)
    assert_close(o.view, acc, P, rel, what)


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", CASES)
def test_gemm_tn(M, N, K):
    i = CASES.index((M, N, K))
    g = _gen("tn", M, N, K)
    act, use_bias, out_dtype = i % 3, i % 2 == 0, (F32, BF16)[(i // 2) % 2]
    run_gemm_tn(M, N, K, BF16, act, use_bias, out_dtype, g)
    run_gemm_tn(M, N, K, F32, (act + 1) % 3, not use_bias, (BF16, F32)[(i // 2) % 2], g)
    run_gemm_tn_splitk(M, N, K, (BF16, F32)[i % 2], (2, 3, 16)[i % 3], g)
    assert _L().device_error() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("splits", [2, 3, 16])
def test_gemm_tn_empty_splits(splits):
    """K = 8: one k-block, so all splits but the first have no k-block at all and must add exactly zero."""
    g = _gen("empty", splits)
    for dtype in (BF16, F32):
        run_gemm_tn_splitk(129, 132, 8, dtype, splits, g)
        run_gemm_tn_splitk(64, 13, 72, dtype, splits, g)
    assert _L().device_error() == 0


# ------------------------------------------------------------------------------------------------ dvt_gemm_tn_residual
def run_residual(M, N, K, dtype, use_gamma, use_branch, gen, repeat=True):
    tdt = torch.bfloat16 if dtype == BF16 else torch.float32
    a = _window(M, K, tdt, gen)
    b = _window(N, K, tdt, gen, scale=K ** -0.5)
    bias = torch.randn(N, device="cuda", generator=gen)
    gamma = (torch.rand(N, device="cuda", generator=gen) + 0.5) if use_gamma else None
    x0 = torch.randn(M, N, device="cuda", generator=gen) * 4
    outs = []
    for _ in range(2 if repeat else 1):
        o = Out(M, N, torch.float32, init=x0)
        br = Out(M, N, torch.bfloat16) if use_branch else None
        _call("dvt_gemm_tn_residual", _p(a), a.stride(0), _p(b), b.stride(0), dtype, M, N, K, _p(bias), _p(gamma),
              _p(o.view), o.ld, _p(br.view) if br else None, br.ld if br else 0, _stream())
        outs.append((o, br))
    torch.cuda.synchronize()
    if dtype == BF16:
        a64, b64, rel = a.double(), b.double(), REL_BF16
    else:
        a64, b64, rel = tf32_trunc(a).double(), tf32_trunc(b).double(), REL_TF32
    acc, P = _prod(a64, b64)
    v = acc + bias.double()
    g64 = gamma.double() if use_gamma else torch.ones(N, device="cuda", dtype=torch.float64)
    ref = x0.double() + g64 * v
    what = f"dvt_gemm_tn_residual M={M} N={N} K={K} dtype={dtype} gamma={use_gamma} branch={use_branch}"
    o, br = outs[0]
    o.check_sentinels(what)
    assert_close(o.view, ref, P * g64, rel, what, mag=ref.abs() + x0.double().abs() + (g64 * v).abs())
    if use_branch:
        br.check_sentinels(what + " (branch)")
        assert_close(br.view, v, P, rel, what + " (branch)", bf16_out=True, mag=v.abs())
    if repeat:
        assert torch.equal(outs[0][0].buf.view(torch.int32), outs[1][0].buf.view(torch.int32)), f"{what}: second run differs"


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", CASES[::3] + [RAGGED])
def test_gemm_tn_residual(M, N, K):
    i = CASES.index((M, N, K)) if (M, N, K) in CASES else 0
    g = _gen("resid", M, N, K)
    for use_gamma, use_branch in ((True, True), (False, False), (i % 2 == 0, i % 2 == 1)):
        run_residual(M, N, K, BF16, use_gamma, use_branch, g)
    run_residual(M, N, K, F32, i % 2 == 1, False, g)
    assert _L().device_error() == 0


# ------------------------------------------------------------------------------------------------ dvt_gemm_bf16
def _operand_bf16(rows, K, mn, gen, scale=1.0):
    """Logical [rows, K] bf16 operand, stored K-major ([rows, K] window) or MN-major ([K, rows] window).  Returns the
    stored view and the logical fp64 matrix."""
    if mn:
        s = _window(K, rows, torch.bfloat16, gen, scale=scale)
        return s, s.double().T
    s = _window(rows, K, torch.bfloat16, gen, scale=scale)
    return s, s.double()


def run_gemm_bf16(M, N, K, layout, gen, *, out_dtype=F32, splits=1, preact=False, last_col=False, repeat=True):
    a_mn, b_mn = layout
    a, a64 = _operand_bf16(M, K, a_mn, gen)
    b, b64 = _operand_bf16(N, K, b_mn, gen, scale=K ** -0.5)
    n_out = N - 1 if last_col else N
    atomic = splits > 1 or last_col
    odt = torch.bfloat16 if out_dtype == BF16 else torch.float32
    pre = _window(M, N, torch.bfloat16, gen, scale=2.0) if preact else None
    outs = []
    for _ in range(2 if repeat and not atomic else 1):
        o = Out(M, n_out, odt, init=torch.zeros(M, n_out, device="cuda") if atomic else None)
        lc = Out(1, M, torch.float32, init=torch.zeros(1, M, device="cuda")) if last_col else None
        _call("dvt_gemm_bf16", _p(a), a.stride(0), a_mn, _p(b), b.stride(0), b_mn, M, N, K, _p(o.view), o.ld, out_dtype,
              splits, _p(pre), pre.stride(0) if preact else 0, _p(lc.view) if lc else None, _stream())
        outs.append((o, lc))
    torch.cuda.synchronize()
    acc, P = _prod(a64, b64)
    what = f"dvt_gemm_bf16 M={M} N={N} K={K} layout={layout} out={out_dtype} splits={splits} preact={preact} last_col={last_col}"
    o, lc = outs[0]
    o.check_sentinels(what)
    if preact:
        gp = gelu_grad64(pre.double())
        ref = acc * gp
        assert_close(o.view, ref, P * gp.abs(), REL_BF16, what, bf16_out=out_dtype == BF16,
                     abs_extra=2e-6 * acc.abs(), mag=ref.abs())
    else:
        assert_close(o.view, acc[:, :n_out], P[:, :n_out], REL_BF16, what, bf16_out=out_dtype == BF16)
    if last_col:
        lc.check_sentinels(what + " (last_col_out)")
        assert_close(lc.view[0], acc[:, N - 1], P[:, N - 1], REL_BF16, what + " (last_col_out)")
    if len(outs) == 2:
        it = torch.int16 if odt == torch.bfloat16 else torch.int32
        assert torch.equal(outs[0][0].buf.view(it), outs[1][0].buf.view(it)), f"{what}: second run differs"
    return a, b, acc, P


LAYOUTS = [(0, 0), (0, 1), (1, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", CASES)
def test_gemm_bf16(M, N, K):
    i = CASES.index((M, N, K))
    g = _gen("bf16", M, N, K)
    layout = LAYOUTS[i % 3]
    run_gemm_bf16(M, N, K, layout, g, out_dtype=(F32, BF16)[(i // 3) % 2])
    run_gemm_bf16(M, N, K, LAYOUTS[(i + 1) % 3], g, out_dtype=(BF16, F32)[i % 2], preact=True)
    run_gemm_bf16(M, N, K, LAYOUTS[(i + 2) % 3], g, splits=(2, 5, 16)[i % 3])
    n_lc = (N - 1 + 3) // 4 * 4 + 1                                    # last_col_out needs (N - 1) % 4 == 0
    run_gemm_bf16(M, n_lc, K, (1, 1), g, splits=(1, 3)[i % 2], last_col=True)
    assert _L().device_error() == 0


# ------------------------------------------------------------------------------------------------ wgrad, ordered split-K
@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", [(64, 128, 1000), (129, 260, 200), (383, 132, 72), (127, 8, 56), (1, 124, 1000)])
def test_gemm_bf16_wgrad_ordered(M, N, K):
    """out = dy^T x with dy [K, M], x [K, N] (both MN-major), k split into planes added in split order: within the bound of
    the fp64 product, close to the atomic split-K form, bit-identical across repeats."""
    g = _gen("wgrad", M, N, K)
    dy = _window(K, M, torch.bfloat16, g)
    x = _window(K, N, torch.bfloat16, g, scale=K ** -0.5)
    acc, P = _prod(dy.double().T, x.double().T)
    kb_total = (K + 63) // 64
    for splits in (1, 2, 5, kb_total + 3):
        runs = []
        for _ in range(2):
            o = Out(M, N, torch.float32)
            ws = torch.full((splits, M, o.ld), float("nan"), device="cuda")    # [splits, M, ldo] planes
            _call("dvt_gemm_bf16_wgrad_ordered", _p(dy), dy.stride(0), _p(x), x.stride(0), M, N, K, _p(o.view), o.ld, splits,
                  _p(ws), _stream())
            runs.append(o)
        torch.cuda.synchronize()
        what = f"dvt_gemm_bf16_wgrad_ordered M={M} N={N} K={K} splits={splits}"
        runs[0].check_sentinels(what)
        assert_close(runs[0].view, acc, P, REL_BF16, what)
        assert torch.equal(runs[0].buf.view(torch.int32), runs[1].buf.view(torch.int32)), f"{what}: repeat differs"
        at = Out(M, N, torch.float32, init=torch.zeros(M, N, device="cuda"))
        _call("dvt_gemm_bf16", _p(dy), dy.stride(0), 1, _p(x), x.stride(0), 1, M, N, K, _p(at.view), at.ld, F32, splits,
              None, 0, None, _stream())
        torch.cuda.synchronize()
        assert_close(runs[0].view, at.view.double(), 2 * P, REL_BF16, what + " vs the atomic form")
    assert _L().device_error() == 0


# ------------------------------------------------------------------------------------------------ 3xTF32
def run_x3(M, N, K, layout, gen, *, splits=1, last_col=False, repeat=True):
    a_mn, b_mn = layout
    a_log = torch.randn(M, K, device="cuda", generator=gen)
    b_log = torch.randn(N, K, device="cuda", generator=gen) * K ** -0.5
    a_st = a_log.T.contiguous() if a_mn else a_log
    b_st = b_log.T.contiguous() if b_mn else b_log
    a, plane_a, _ka = _x3_planes(a_st)
    b, plane_b, _kb = _x3_planes(b_st)
    n_out = N - 1 if last_col else N
    atomic = splits > 1 or last_col
    outs = []
    for _ in range(2 if repeat and not atomic else 1):
        o = Out(M, n_out, torch.float32, init=torch.zeros(M, n_out, device="cuda") if atomic else None)
        lc = Out(1, M, torch.float32, init=torch.zeros(1, M, device="cuda")) if last_col else None
        _call("dvt_gemm_f32x3", _p(a), a.stride(0), plane_a, a_mn, _p(b), b.stride(0), plane_b, b_mn, M, N, K, _p(o.view),
              o.ld, splits, _p(lc.view) if lc else None, _stream())
        outs.append((o, lc))
    torch.cuda.synchronize()
    acc, P = _prod(a_log.double(), b_log.double())          # hi + lo == the fp32 value exactly
    what = f"dvt_gemm_f32x3 M={M} N={N} K={K} layout={layout} splits={splits} last_col={last_col}"
    o, lc = outs[0]
    o.check_sentinels(what)
    assert_close(o.view, acc[:, :n_out], P[:, :n_out], REL_X3, what)
    if last_col:
        lc.check_sentinels(what + " (last_col_out)")
        assert_close(lc.view[0], acc[:, N - 1], P[:, N - 1], REL_X3, what + " (last_col_out)")
    if len(outs) == 2:
        assert torch.equal(outs[0][0].buf.view(torch.int32), outs[1][0].buf.view(torch.int32)), f"{what}: second run differs"


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", CASES)
def test_gemm_f32x3(M, N, K):
    i = CASES.index((M, N, K))
    g = _gen("x3", M, N, K)
    run_x3(M, N, K, LAYOUTS[i % 3], g)
    run_x3(M, N, K, LAYOUTS[(i + 1) % 3], g, splits=(2, 3, 16)[i % 3])
    n_lc = (N - 1 + 3) // 4 * 4 + 1
    run_x3(M, n_lc, K, (1, 1), g, splits=(1, 4)[i % 2], last_col=True)
    assert _L().device_error() == 0


# ------------------------------------------------------------------------------------------------ SwiGLU backward
def run_swiglu(M, Hh, K, gen):
    dy = _window(M, K, torch.bfloat16, gen)
    w = _window(K, Hh, torch.bfloat16, gen, scale=K ** -0.5)          # fc2 weight [C = K, Hh], read MN-major
    hpre = _window(M, 2 * Hh, torch.bfloat16, gen, scale=2.0)
    outs = []
    for _ in range(2):
        o = Out(M, 2 * Hh, torch.bfloat16)
        _call("dvt_gemm_bf16_dgrad_swiglu", _p(dy), dy.stride(0), _p(w), w.stride(0), M, Hh, K, _p(hpre), hpre.stride(0),
              _p(o.view), o.ld, _stream())
        outs.append(o)
    torch.cuda.synchronize()
    dh, P = _prod(dy.double(), w.double().T)
    gg, u = hpre[:, :Hh].double(), hpre[:, Hh:].double()
    s = torch.sigmoid(gg)
    dg_fac, du_fac = u * (s + gg * s * (1 - s)), gg * s
    ref = torch.cat([dh * dg_fac, dh * du_fac], 1)
    Pf = torch.cat([P * dg_fac.abs(), P * du_fac.abs()], 1)
    what = f"dvt_gemm_bf16_dgrad_swiglu M={M} Hh={Hh} K={K}"
    outs[0].check_sentinels(what)
    # __expf and the fp32 sigmoid: ~2^-21 relative on each factor, folded into the abs term
    assert_close(outs[0].view, ref, Pf, REL_BF16, what, bf16_out=True, abs_extra=2.0 ** -20 * ref.abs())
    assert torch.equal(outs[0].buf.view(torch.int16), outs[1].buf.view(torch.int16)), f"{what}: second run differs"


@pytest.mark.gpu
@pytest.mark.parametrize("M,Hh,K", [(383, 132, 200), (129, 130, 72)])
def test_gemm_bf16_dgrad_swiglu(M, Hh, K):
    run_swiglu(M, Hh, K, _gen("swiglu", M, Hh, K))
    assert _L().device_error() == 0


# ------------------------------------------------------------------------------------------------ SIMT debug path
@pytest.mark.gpu
def test_simt_debug_path_every_entry_point():
    """Every entry point once on the SIMT debug kernels at the most ragged shape, against the same bounds."""
    M, N, K = RAGGED
    g = _gen("simt")
    with impl_mode(1):
        for dtype, act, bias, od in ((BF16, 1, True, BF16), (BF16, 2, False, F32), (F32, 0, True, F32)):
            run_gemm_tn(M, N, K, dtype, act, bias, od, g)
        run_gemm_tn_splitk(M, N, K, BF16, 3, g)
        run_residual(M, N, K, BF16, True, True, g)
        for layout in LAYOUTS:
            run_gemm_bf16(M, N, K, layout, g, preact=layout == (0, 1))
        run_gemm_bf16(M, 133, K, (1, 1), g, splits=2, last_col=True)
        for layout in LAYOUTS:
            run_x3(M, N, K, layout, g)
        run_x3(M, 133, K, (1, 1), g, splits=2, last_col=True)
        run_swiglu(M, 132, K, g)
    assert _L().device_error() == 0
