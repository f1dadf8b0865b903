"""Deterministic training, CPU part: the fp32 weight matrices that `dvt.train_ops.resample_weights` reads off ATen (a
one-hot basis through F.interpolate(bicubic, antialias=True)) reproduce F.interpolate itself, and contracting a gradient
with their transposes (what the fixed-order CUDA resample backward computes) is the torch autograd gradient."""
import pytest
import torch
import torch.nn.functional as F

SHAPES = [((37, 37), (73, 73)), ((14, 14), (32, 32)), ((24, 24), (14, 14)), ((5, 7), (9, 4)), ((16, 9), (7, 20))]


def _resample(g, h, w):
    return F.interpolate(g, size=(h, w), mode="bicubic", antialias=True)


@pytest.mark.parametrize("src,dst", SHAPES)
def test_weight_matrices_reproduce_interpolate(src, dst):
    from dvt import train_ops
    (gh, gw), (h, w) = src, dst
    C = 6
    g = torch.randn(1, C, gh, gw, generator=torch.Generator().manual_seed(gh * 100 + w))
    wh, ww = train_ops.resample_weights(gh, h, "cpu"), train_ops.resample_weights(gw, w, "cpu")
    assert wh.shape == (h, gh) and ww.shape == (w, gw) and wh.dtype == torch.float32
    assert torch.allclose(wh.sum(1), torch.ones(h), atol=1e-6)        # rows of an interpolation matrix sum to one
    ref = _resample(g, h, w)
    got = torch.einsum("yi,xj,cij->cyx", wh.double(), ww.double(), g[0].double())
    assert (got - ref[0].double()).abs().max().item() < 1e-5 * max(1.0, g.abs().max().item())


@pytest.mark.parametrize("src,dst", SHAPES)
def test_transpose_contraction_is_the_autograd_gradient(src, dst):
    from dvt import train_ops
    (gh, gw), (h, w) = src, dst
    C = 5
    gen = torch.Generator().manual_seed(gh + 7 * h)
    g = torch.randn(1, C, gh, gw, generator=gen, dtype=torch.float64).requires_grad_(True)
    dout = torch.randn(1, C, h, w, generator=gen, dtype=torch.float64)
    _resample(g, h, w).backward(dout)
    wh, ww = train_ops.resample_weights(gh, h, "cpu").double(), train_ops.resample_weights(gw, w, "cpu").double()
    got = torch.einsum("yi,xj,cyx->cij", wh, ww, dout[0])
    # fp32 weights against the float64 autograd of the same op: agreement to fp32 rounding of the weights
    assert (got - g.grad[0]).abs().max().item() < 1e-5 * dout.abs().sum().item() / (h * w) * max(h / gh, w / gw, 1.0) + 1e-5


def test_weights_are_cached():
    from dvt import train_ops
    a = train_ops.resample_weights(11, 17, "cpu")
    assert train_ops.resample_weights(11, 17, "cpu") is a
