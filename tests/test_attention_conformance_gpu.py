"""Flash attention (forward, lse, backward, deterministic backward) at head_dim 64 and 80 on structured inputs, against
fp64 attention of the same bf16 qkv.

Inputs (B = 2, heads = 3, every N from 1 to 257 around the key-tile edges):
  randn     i.i.d. Gaussian qkv
  q0        q = 0: every key gets the same weight, so out is the mean of V over exactly N keys.  V has mean 1, so a key
            block whose zero-filled padding is not masked scales the output by N / padded N and cannot hide.
  first     one outlier key (a high-norm artifact token): k_j += a u with the queries given a component along u, so its
            logit exceeds the rest by ~30-60; placed in the first key tile
  last      the same in the last, ragged key tile
  two       two outliers in different tiles, the later one larger: the row maximum changes mid-row and the running
            rescale of the partial sums is exercised
  massive   a few V and dout channels ~100x the rest (massive activations)

Bounds: forward |out - ref| <= 2^-7 max|v| + 2^-8 |ref| per head (bf16 P and bf16 output); lse within 2e-3 (log2 units).
Backward: the kernel's max error against fp64 is at most twice torch SDPA's (flash backend, bf16) plus a floor of
2^-9 max|ref| (half a bf16 ulp of the largest gradient) + 2^-16 max|dout| max|v|.  The second term is for gradients that
are zero in exact arithmetic: with N = 1, dQ = scale (dP - delta) k is 0, but dP = dout . v (tensor cores) and
delta = rowsum(dout * out) (fp32, another order) differ by fp32 rounding, ~1e-7 on the H100, where SDPA happens to
give exactly 0.  dvt_attention_bwd_det's dK / dV are bit-identical to dvt_attention_bwd's."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

NS = (1, 2, 17, 127, 128, 129, 255, 256, 257)
KINDS = ("randn", "q0", "first", "last", "two", "massive")
B, H = 2, 3


def _L():
    from dvt import _lib
    return _lib


def _call(name, *args):
    L = _L()
    L.check(getattr(L.lib(), name)(*args), name)


def _inputs(kind, N, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(B, H, N, D, device="cuda", generator=g)
    k = torch.randn(B, H, N, D, device="cuda", generator=g)
    v = torch.randn(B, H, N, D, device="cuda", generator=g)
    dout = torch.randn(B, H, N, D, device="cuda", generator=g)
    scale = D ** -0.5
    if kind == "q0":
        q.zero_()
        v = 1.0 + 0.25 * v
    elif kind in ("first", "last", "two"):
        u = torch.randn(D, device="cuda", generator=g)
        u = u / u.norm()
        beta = 4.0                                  # query component along u
        q = q + beta * u
        # a key with alpha u has logit ~ alpha beta scale above the rest: 30..60 over the queries
        alpha = 45.0 / (beta * scale)
        pos = {"first": [min(3, N - 1)], "last": [N - 1], "two": [min(1, N - 1), max(N - 2, 0)]}[kind]
        for i, j in enumerate(pos):
            k[:, :, j] += (1.0 + 0.3 * i) * alpha * u   # the later outlier is larger
    elif kind == "massive":
        v[..., 5] *= 100.0
        v[..., 17] *= 100.0
        dout[..., 5] *= 100.0
        dout[..., 33] *= 100.0
    qkv = torch.stack([q, k, v], 2).permute(0, 3, 2, 1, 4).reshape(B, N, 3 * H * D).bfloat16().contiguous()
    return qkv, dout.permute(0, 2, 1, 3).reshape(B, N, H * D).bfloat16().contiguous()


def _split(qkv, N, D):
    """bf16 [B, N, 3 H D] -> q, k, v [B, H, N, D] (timm's reshape(B, N, 3, H, D))."""
    t = qkv.reshape(B, N, 3, H, D).permute(2, 0, 3, 1, 4)
    return t[0], t[1], t[2]


def _heads(x, N, D):
    return x.reshape(B, N, H, D).permute(0, 2, 1, 3)


def _ref(qkv, dout, N, D):
    q, k, v = (t.double().requires_grad_(True) for t in _split(qkv, N, D))
    s = (q @ k.transpose(-1, -2)) * D ** -0.5
    out = torch.softmax(s, -1) @ v
    out.backward(_heads(dout, N, D).double())
    lse2 = torch.logsumexp(s, -1) / math.log(2.0)
    return out.detach(), lse2.detach(), (q.grad, k.grad, v.grad), v.detach()


def _kernel_fwd(qkv, N, D):
    out = torch.empty(B, N, H * D, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(B, H, N, device="cuda")
    _call("dvt_attention_fwd", qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, N, H, D, _L().cur_stream())
    out2 = torch.empty_like(out)
    _call("dvt_attention_fwd", qkv.data_ptr(), out2.data_ptr(), None, B, N, H, D, _L().cur_stream())
    torch.cuda.synchronize()
    return out, lse, out2


def _kernel_bwd(qkv, out, dout, lse, N, D, det):
    dqkv = torch.empty_like(qkv)
    delta = torch.empty(B, H, N, device="cuda")
    if det:
        _call("dvt_attention_bwd_det", qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(),
              delta.data_ptr(), B, N, H, D, _L().cur_stream())
    else:
        dq_ws = torch.empty(B, N, H * D, device="cuda")
        _call("dvt_attention_bwd", qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(),
              dq_ws.data_ptr(), delta.data_ptr(), B, N, H, D, _L().cur_stream())
    torch.cuda.synchronize()
    return dqkv


def _sdpa_grads(qkv, dout, N, D):
    from torch.nn.attention import SDPBackend, sdpa_kernel
    q, k, v = (t.contiguous().requires_grad_(True) for t in _split(qkv, N, D))
    with sdpa_kernel(SDPBackend.FLASH_ATTENTION):
        o = torch.nn.functional.scaled_dot_product_attention(q, k, v)
    o.backward(_heads(dout, N, D).contiguous())
    return q.grad, k.grad, v.grad


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("D", [64, 80])
def test_attention_conformance(D, N, kind):
    seed = 1000 * D + 10 * N + KINDS.index(kind)
    qkv, dout = _inputs(kind, N, D, seed)
    ref_out, ref_lse, ref_grads, v64 = _ref(qkv, dout, N, D)
    what = f"D={D} N={N} {kind}"

    # ---- forward and lse ----
    out, lse, out_nolse = _kernel_fwd(qkv, N, D)
    got = _heads(out, N, D).double()
    vmax = v64.abs().amax(dim=(2, 3), keepdim=True)                    # per (batch, head)
    bound = 2.0 ** -7 * vmax + 2.0 ** -8 * ref_out.abs()
    ratio = ((got - ref_out).abs() / bound).max().item()
    assert ratio <= 1.0, f"{what}: forward error {ratio:.3g} x the bound"
    lse_err = (lse.double() - ref_lse).abs().max().item()
    assert lse_err <= 2e-3, f"{what}: lse error {lse_err:.3g} (log2 units)"
    assert torch.equal(out.view(torch.int16), out_nolse.view(torch.int16)), f"{what}: out differs with and without lse"
    if kind == "q0":                                                    # the mean of V over exactly N keys
        mean = v64.mean(2, keepdim=True).expand_as(got)
        assert ((got - mean).abs() <= 2.0 ** -8 * mean.abs() + 2.0 ** -12 * vmax).all(), f"{what}: not the mean of V"

    # ---- backward: both forms against fp64, peer-checked against SDPA ----
    dqkv = _kernel_bwd(qkv, out, dout, lse, N, D, det=False)
    dqkv_det = _kernel_bwd(qkv, out, dout, lse, N, D, det=True)
    sd = _sdpa_grads(qkv, dout, N, D)
    gscale = dout.abs().max().item() * v64.abs().max().item()        # size of the terms of dP = dout . v
    for form, g in (("bwd", dqkv), ("bwd_det", dqkv_det)):
        parts = _split(g, N, D)
        for name, gk, gs, gr in zip("qkv", parts, sd, ref_grads):
            e_k = (gk.double() - gr).abs().max().item()
            e_s = (gs.double() - gr).abs().max().item()
            floor = 2.0 ** -9 * gr.abs().max().item() + 2.0 ** -16 * gscale
            assert e_k <= 2 * e_s + floor, f"{what} {form}: d{name} error {e_k:.3g} vs SDPA {e_s:.3g} (floor {floor:.3g})"
    kd, vd = _split(dqkv, N, D)[1:], _split(dqkv_det, N, D)[1:]
    for name, a, b in zip("kv", kd, vd):
        assert torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16)), \
            f"{what}: d{name} of bwd_det differs from bwd"
    assert _L().device_error() == 0
