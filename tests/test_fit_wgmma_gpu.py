"""The 3xTF32 wgmma GEMM (both operands K-major: the forward linears and the data gradients of the stage-1 fit) against
float64 at the fit's shapes -- 2048 rows by 128 / 192 / 384 / 768 columns and reductions -- and at tile edges: M and N
not multiples of the 128 x 64 tile, N = 769 through the ones column, K = 128, split K."""
import pytest
import torch

pytestmark = pytest.mark.gpu

FIT_DIMS = (128, 192, 384, 768)


def _rel(a, b):
    return ((a.double() - b).norm() / b.norm()).item()


def _operands(M, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    return x, w


@pytest.mark.parametrize("N", FIT_DIMS)
@pytest.mark.parametrize("K", FIT_DIMS)
def test_wgmma_x3_fit_shapes_match_fp64(N, K):
    from dvt import _lib, ops
    x, w = _operands(2048, N, K, seed=N * 1000 + K)
    y = ops.gemm_f32x3(x, w, 2048, N, K)
    y2 = ops.gemm_f32x3(x, w, 2048, N, K)
    torch.cuda.synchronize()
    err = _rel(y, x.double() @ w.double().t())
    assert err < 1e-5, f"M=2048 N={N} K={K}: relative error vs fp64 {err}"
    assert torch.equal(y, y2), "two runs of the same product differ"
    assert _lib.device_error() == 0


@pytest.mark.parametrize("M,N,K", [(2048, 769, 384), (2000, 130, 128), (200, 64, 128), (77, 133, 40), (2048, 1, 192)])
def test_wgmma_x3_edges_match_fp64(M, N, K):
    from dvt import _lib, ops
    x, w = _operands(M, N, K, seed=M + N + K)
    y = ops.gemm_f32x3(x, w, M, N, K)
    torch.cuda.synchronize()
    err = _rel(y, x.double() @ w.double().t())
    assert err < 1e-5, f"M={M} N={N} K={K}: relative error vs fp64 {err}"
    assert _lib.device_error() == 0


@pytest.mark.parametrize("splits", [1, 3, 8])
def test_wgmma_x3_ones_column_and_split_k_match_fp64(splits):
    """Atomic output with the last column redirected (the bias gradient through a ones column): N = 769."""
    from dvt import _lib, ops
    M, N, K = 384, 769, 768
    x, w = _operands(M, N, K, seed=splits)
    w[-1] = 1.0
    out, col = ops.gemm_f32x3(x, w, M, N, K, splits=splits, last_col=True)
    torch.cuda.synchronize()
    ref = x.double() @ w.double().t()
    errs = {"out": _rel(out, ref[:, :N - 1]), "last column": _rel(col, ref[:, N - 1])}
    assert all(v < 1e-5 for v in errs.values()), f"splits={splits}: relative errors vs fp64 {errs}"
    assert _lib.device_error() == 0
