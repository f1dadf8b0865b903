"""GEMM kernel parity (tensor-core path and SIMT debug path) against torch fp32 matmul of the same rounded operands."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from dvt import _lib
    return _lib


def _ref(a, w, bias, act):
    y = a.float() @ w.float().t()
    if bias is not None:
        y = y + bias
    if act == "gelu":
        y = torch.nn.functional.gelu(y)
    elif act == "relu":
        y = torch.relu(y)
    return y


SHAPES = [
    (128, 128, 64),      # one tile, one k-block
    (128, 256, 128),     # wide tile
    (256, 384, 128),     # narrow tiles, N not multiple of 256
    (300, 200, 72),      # ragged M, N, K tails
    (2048, 768, 384),    # fit GEMM
    (2740, 2304, 768),   # QKV for 2 views
    (1370, 768, 3072),   # fc2 for 1 view
]


@pytest.mark.parametrize("impl", [1, 0], ids=["simt", "tcgen05"])
@pytest.mark.parametrize("shape", SHAPES)
def test_gemm_bf16(impl, shape):
    from dvt import ops
    L = _lib()
    M, N, K = shape
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    L.check(L.lib().dvt_set_debug_impl(impl))
    try:
        for act in (None, "gelu", "relu"):
            y = ops.gemm_tn(a, w, bias, act, out_dtype=torch.float32)
            torch.cuda.synchronize()
            ref = _ref(a, w, bias, act)
            err = (y - ref).abs().max().item()
            assert err < 2e-3, f"impl={impl} act={act} shape={shape} max err {err}"
            yb = ops.gemm_tn(a, w, bias, act, out_dtype=torch.bfloat16)
            torch.cuda.synchronize()
            errb = (yb.float() - ref).abs().max().item()
            assert errb < 3e-2, f"bf16 out impl={impl} act={act} shape={shape} max err {errb}"
    finally:
        L.check(L.lib().dvt_set_debug_impl(-1))
    assert L.device_error() == 0


@pytest.mark.parametrize("impl", [1, 0], ids=["simt", "tcgen05"])
def test_gemm_tf32(impl):
    from dvt import ops
    L = _lib()
    M, N, K = 2048, 384, 128
    g = torch.Generator(device="cuda").manual_seed(5)
    a = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    L.check(L.lib().dvt_set_debug_impl(impl))
    try:
        y = ops.gemm_tn(a, w, None, None, out_dtype=torch.float32)
        torch.cuda.synchronize()
    finally:
        L.check(L.lib().dvt_set_debug_impl(-1))
    ref = a @ w.t()
    err = (y - ref).abs().max().item()
    assert err < 2e-2, f"tf32 impl={impl} err {err}"


@pytest.mark.parametrize("impl", [1, 0], ids=["simt", "tcgen05"])
def test_gemm_splitk_and_residual(impl):
    from dvt import ops
    L = _lib()
    g = torch.Generator(device="cuda").manual_seed(11)
    L.check(L.lib().dvt_set_debug_impl(impl))
    try:
        # split-K: dW-like shape
        a = torch.randn(768, 2048, device="cuda", generator=g).bfloat16()
        w = torch.randn(384, 2048, device="cuda", generator=g).bfloat16()
        y = ops.gemm_tn(a, w, None, None, out_dtype=torch.float32, splits=8)
        torch.cuda.synchronize()
        ref = a.float() @ w.float().t()
        assert (y - ref).abs().max().item() < 5e-2
        # residual with LayerScale
        x = torch.randn(1370, 768, device="cuda", generator=g)
        x0 = x.clone()
        aa = torch.randn(1370, 768, device="cuda", generator=g).bfloat16()
        ww = (torch.randn(768, 768, device="cuda", generator=g) / 28).bfloat16()
        b = torch.randn(768, device="cuda", generator=g)
        gam = torch.rand(768, device="cuda", generator=g) + 0.5
        ops.gemm_tn_residual_(x, aa, ww, b, gam)
        torch.cuda.synchronize()
        ref = x0 + gam * (aa.float() @ ww.float().t() + b)
        assert (x - ref).abs().max().item() < 2e-3
    finally:
        L.check(L.lib().dvt_set_debug_impl(-1))
    assert L.device_error() == 0


@pytest.mark.parametrize("shape", [(256, 256, 64), (257, 512, 128), (511, 1100, 200), (2740, 2304, 768), (43840, 768, 3072),
                                   (1000, 3072, 768), (21904, 2304, 768)])
def test_gemm_cta_pair_kernel(shape):
    """The tensor-core kernel on the ViT's GEMM shapes against torch -- ragged M, ragged N > 1024, K tails, and every fused
    epilogue the ViT uses -- and bit-exact on a second run (fixed k-order of the fp32 accumulation, no atomics)."""
    from dvt import ops
    L = _lib()
    M, N, K = shape
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    gam = torch.rand(N, device="cuda", generator=g) + 0.5
    x0 = torch.randn(M, N, device="cuda", generator=g)
    outs = {}
    for run in (0, 1):
        y32 = ops.gemm_tn(a, w, bias, None, out_dtype=torch.float32)
        yg = ops.gemm_tn(a, w, bias, "gelu", out_dtype=torch.bfloat16)
        x = x0.clone()
        ops.gemm_tn_residual_(x, a, w, bias, gam)
        torch.cuda.synchronize()
        outs[run] = (y32, yg, x)
    assert L.device_error() == 0
    ref = a.float() @ w.float().t() + bias
    assert (outs[0][0] - ref).abs().max().item() < 2e-3 * max(1.0, ref.abs().max().item())
    assert (outs[0][1].float() - torch.nn.functional.gelu(ref)).abs().max().item() < 3e-2
    assert (outs[0][2] - (x0 + gam * ref)).abs().max().item() < 4e-3 * max(1.0, ref.abs().max().item())
    for k in range(3):
        assert torch.equal(outs[0][k], outs[1][k]), f"second run differs (output {k})"
