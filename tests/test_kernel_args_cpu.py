"""Argument validation of the LayerNorm, column-sum, LayerScale / token-assembly backward, loss, AdamW, resample, im2col
and segmentation-loss entry points: a pointer the kernel would touch with a vector access (float4 / uint2 / bf16x2) at a
misaligned address, a row pitch smaller than the row, a bad in_group / skip pair or an unsupported width is reported as
DVT_ERR_INVALID with a message that names the argument, before any CUDA call.

As in test_gemm_args_cpu.py the pointers are fake integers and nothing is dereferenced.  The file runs only where there is
no GPU: a call that passes every check goes on to the CUDA runtime, finds no device and returns DVT_ERR_CUDA, so a missing
check fails the test cleanly instead of launching a kernel on misaligned memory."""
import inspect

import pytest
import torch

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="fake device pointers: run on a machine without a GPU")

DVT_OK, DVT_ERR_INVALID, DVT_ERR_CUDA = 0, 1, 2
BF16, F32 = 0, 1

BASE = 1 << 32                      # 256-byte aligned fake device addresses, far apart
P = [BASE + i * (1 << 24) for i in range(12)]


@pytest.fixture(scope="module")
def L():
    from dvt import _lib
    return _lib


# One builder per entry point: keyword overrides of a well-formed call.  Pointer arguments are named as in the header.
def _layernorm(L, x=P[0], ldx=768, gamma=P[1], beta=P[2], y=P[3], ldy=768, y_dtype=F32, rows=25, C=768, in_group=1,
               skip=0):
    return L.lib().dvt_layernorm(x, ldx, gamma, beta, y, ldy, y_dtype, rows, C, 1e-6, in_group, skip, None)


def _layernorm_bwd(L, x=P[0], gamma=P[1], dy=P[2], dx_accum=P[3], dgamma=P[4], dbeta=P[5], rows=25, C=768):
    return L.lib().dvt_layernorm_bwd(x, gamma, dy, dx_accum, dgamma, dbeta, rows, C, 1e-6, None)


def _layernorm_bwd_grouped(L, x=P[0], gamma=P[1], dy=P[2], dx_accum=P[3], dgamma=P[4], dbeta=P[5], workspace=P[6], rows=30,
                           C=768, in_group=10, skip=3):
    return L.lib().dvt_layernorm_bwd_grouped(x, gamma, dy, dx_accum, dgamma, dbeta, workspace, rows, C, 1e-6, in_group, skip,
                                             None)


def _colsum(L, inp=P[0], dtype=F32, ld=132, rows=100, cols=132, out=P[1]):
    return L.lib().dvt_colsum(inp, dtype, ld, rows, cols, out, None)


def _colsum_ordered(L, inp=P[0], dtype=F32, ld=132, rows=100, cols=132, out=P[1], workspace=P[2]):
    return L.lib().dvt_colsum_ordered(inp, dtype, ld, rows, cols, out, workspace, None)


def _layerscale_bwd(L, dx=P[0], ldx=768, branch=P[1], gamma=P[2], dbranch=P[3], dbias=P[4], dgamma=P[5], workspace=P[6],
                    rows=100, C=768):
    return L.lib().dvt_layerscale_bwd(dx, ldx, branch, gamma, dbranch, dbias, dgamma, workspace, rows, C, None)


def _embed_fwd(L, patches=P[0], Kp=592, w=P[1], bias=P[2], pos_patch=P[3], prefix_rows=P[4], B=2, np_=37, prefix=1, C=384,
               out=P[5]):
    return L.lib().dvt_vit_embed_fwd(patches, Kp, w, bias, pos_patch, prefix_rows, B, np_, prefix, C, out, None)


def _embed_bwd(L, dx0=P[0], B=2, ntok=38, prefix=1, C=384, dpatch=P[1], dpos=P[2], dprefix=P[3], dbias=P[4],
               workspace=P[5]):
    return L.lib().dvt_vit_embed_bwd(dx0, B, ntok, prefix, C, dpatch, dpos, dprefix, dbias, workspace, None)


def _loss(L, pred=P[0], target=P[1], dpred=P[2], losses3=P[3], rows=25, C=768):
    return L.lib().dvt_denoise_loss(pred, target, dpred, losses3, rows, C, 1.0, None)


def _loss_ordered(L, pred=P[0], target=P[1], dpred=P[2], losses3=P[3], workspace=P[4], rows=25, C=768):
    return L.lib().dvt_denoise_loss_ordered(pred, target, dpred, losses3, workspace, rows, C, 1.0, None)


def _adamw(L, p=P[0], g=P[1], m=P[2], v=P[3], n=1024, step=1):
    return L.lib().dvt_adamw(p, g, m, v, n, 1e-3, 0.9, 0.999, 1e-8, 0.05, step, None)


BUILDERS = {"layernorm": _layernorm, "layernorm_bwd": _layernorm_bwd, "layernorm_bwd_grouped": _layernorm_bwd_grouped,
            "colsum": _colsum, "colsum_ordered": _colsum_ordered, "layerscale_bwd": _layerscale_bwd,
            "vit_embed_fwd": _embed_fwd, "vit_embed_bwd": _embed_bwd, "denoise_loss": _loss,
            "denoise_loss_ordered": _loss_ordered, "adamw": _adamw}


def _expect_invalid(L, rc, *words):
    msg = L.lib().dvt_last_error().decode()
    assert rc == DVT_ERR_INVALID, f"expected DVT_ERR_INVALID, got {rc} ({msg})"
    for w in words:
        assert w in msg, f"message {msg!r} does not mention {w!r}"


def _expect_runtime(L, rc):
    assert rc == DVT_ERR_CUDA, f"got {rc}: {L.lib().dvt_last_error().decode()}"


VALID = [
    ("layernorm", {}), ("layernorm", {"y_dtype": BF16, "y": P[3] + 8}), ("layernorm", {"ldx": 1028, "ldy": 772}),
    ("layernorm", {"rows": 30, "in_group": 10, "skip": 3}), ("layernorm", {"rows": 25, "in_group": 10, "skip": 0}),
    ("layernorm", {"C": 2048, "ldx": 2048, "ldy": 2048}), ("layernorm", {"C": 4, "ldx": 4, "ldy": 4}),
    ("layernorm_bwd", {}), ("layernorm_bwd", {"C": 2048}),
    ("layernorm_bwd_grouped", {}), ("layernorm_bwd_grouped", {"rows": 25, "in_group": 1, "skip": 0}),
    ("colsum", {}), ("colsum", {"dtype": BF16, "inp": P[0] + 4, "cols": 130, "ld": 130}),
    ("colsum", {"inp": P[0] + 4, "cols": 131, "ld": 133}),
    ("colsum_ordered", {}), ("colsum_ordered", {"dtype": BF16, "inp": P[0] + 8, "ld": 256}),
    ("layerscale_bwd", {}), ("layerscale_bwd", {"gamma": None, "branch": None, "dgamma": None, "ldx": 772}),
    ("layerscale_bwd", {"dbranch": None, "branch": P[1] + 8, "dx": P[0] + 16}),
    ("vit_embed_fwd", {}), ("vit_embed_fwd", {"bias": None, "prefix": 5}),
    ("vit_embed_bwd", {}), ("vit_embed_bwd", {"dpatch": P[1] + 8}),
    ("denoise_loss", {}), ("denoise_loss", {"dpred": None}), ("denoise_loss_ordered", {}),
    ("adamw", {}), ("adamw", {"p": P[0] + 16, "n": 4, "step": 10**6}),
]


@pytest.mark.parametrize("name,kw", VALID, ids=[f"{n}-{i}" for i, (n, _) in enumerate(VALID)])
def test_valid_calls_reach_the_cuda_runtime(L, name, kw):
    """Controls: well-formed calls (including the smallest alignment each pointer needs) fail only for lack of a device."""
    _expect_runtime(L, BUILDERS[name](L, **kw))


def test_other_valid_calls_reach_the_cuda_runtime(L):
    lib = L.lib()
    _expect_runtime(L, lib.dvt_resample_bwd(P[0], P[1], P[2], P[3], P[4], 37, 37, 16, 16, 3, None))
    # im2col: odd P / S / W and an input offset by one element take the scalar path; they are not errors
    _expect_runtime(L, lib.dvt_im2col(P[0], F32, P[1], 2, 224, 224, 14, 14, None))
    _expect_runtime(L, lib.dvt_im2col(P[0] + 4, F32, P[1], 2, 31, 33, 7, 3, None))
    _expect_runtime(L, lib.dvt_im2col(P[0] + 2, BF16, P[1], 1, 16, 16, 16, 16, None))
    _expect_runtime(L, lib.dvt_seg_upsample_ce(P[0], 2, 8, 8, 150, P[1], 32, 32, 1.0, P[2], P[3], P[4], None))


# (entry point, pointer argument, byte offset, words of the message)
MISALIGNED = [
    ("layernorm", "x", 4, "x"), ("layernorm", "x", 8, "x"), ("layernorm", "gamma", 4, "gamma"),
    ("layernorm", "beta", 12, "beta"), ("layernorm", "y", 4, "y must be 16-byte"),
    ("layernorm_bwd", "x", 4, "x,"), ("layernorm_bwd", "gamma", 8, "gamma"), ("layernorm_bwd", "dy", 4, "dy"),
    ("layernorm_bwd", "dx_accum", 12, "dx_accum"),
    ("layernorm_bwd_grouped", "x", 4, "x,"), ("layernorm_bwd_grouped", "gamma", 4, "gamma"),
    ("layernorm_bwd_grouped", "dy", 8, "dy"), ("layernorm_bwd_grouped", "dx_accum", 4, "dx_accum"),
    ("colsum", "inp", 2, "in must be"),
    ("colsum_ordered", "inp", 4, "in must be 16-byte"), ("colsum_ordered", "workspace", 4, "workspace"),
    ("layerscale_bwd", "dx", 4, "dx,"), ("layerscale_bwd", "gamma", 8, "gamma"), ("layerscale_bwd", "workspace", 4, "workspace"),
    ("layerscale_bwd", "branch", 4, "branch"), ("layerscale_bwd", "dbranch", 2, "dbranch"),
    ("vit_embed_fwd", "out", 4, "out"), ("vit_embed_fwd", "bias", 8, "bias"), ("vit_embed_fwd", "pos_patch", 4, "pos_patch"),
    ("vit_embed_bwd", "dx0", 4, "dx0"), ("vit_embed_bwd", "dpos", 8, "dpos"), ("vit_embed_bwd", "dprefix", 4, "dprefix"),
    ("vit_embed_bwd", "workspace", 4, "workspace"), ("vit_embed_bwd", "dpatch", 4, "dpatch"),
    ("denoise_loss", "pred", 4, "pred"), ("denoise_loss", "target", 8, "target"), ("denoise_loss", "dpred", 4, "dpred"),
    ("denoise_loss_ordered", "pred", 4, "pred"), ("denoise_loss_ordered", "target", 4, "target"),
    ("denoise_loss_ordered", "dpred", 12, "dpred"),
    ("adamw", "p", 4, "p,"), ("adamw", "g", 4, "g,"), ("adamw", "m", 8, "m "), ("adamw", "v", 12, "v "),
]


@pytest.mark.parametrize("name,arg,off,word", MISALIGNED, ids=[f"{n}-{a}+{o}" for n, a, o, _ in MISALIGNED])
def test_misaligned_pointer(L, name, arg, off, word):
    base = inspect.signature(BUILDERS[name]).parameters[arg].default
    _expect_invalid(L, BUILDERS[name](L, **{arg: base + off}), word, "aligned")


def test_bf16_layernorm_output_needs_8_bytes(L):
    """bf16 y is stored as uint2 (4 x bf16): 8-byte alignment, not 16."""
    _expect_invalid(L, _layernorm(L, y=P[3] + 4, y_dtype=BF16), "y must be 8-byte", "aligned")
    _expect_invalid(L, _layernorm(L, y=P[3] + 2, y_dtype=BF16), "y must be 8-byte", "aligned")


def test_bf16_colsum_ordered_needs_8_bytes(L):
    _expect_invalid(L, _colsum_ordered(L, dtype=BF16, inp=P[0] + 4), "in must be 8-byte", "aligned")


PITCH = [
    ("layernorm", {"ldx": 64, "C": 128, "ldy": 128}, "ldx"), ("layernorm", {"ldy": 764}, "ldy"),
    ("colsum", {"ld": 128, "cols": 132}, "ld=128"), ("colsum", {"dtype": BF16, "ld": 128, "cols": 130}, "ld=128"),
    ("colsum_ordered", {"ld": 128, "cols": 132}, "ld=128"), ("colsum_ordered", {"dtype": BF16, "ld": 64, "cols": 128}, "ld=64"),
    ("layerscale_bwd", {"ldx": 764}, "ldx=764"),
]


@pytest.mark.parametrize("name,kw,word", PITCH, ids=[f"{n}-{i}" for i, (n, _, _) in enumerate(PITCH)])
def test_pitch_smaller_than_the_row(L, name, kw, word):
    _expect_invalid(L, BUILDERS[name](L, **kw), word, ">=")


def test_layernorm_partial_group_with_skip(L):
    """rows = 25, in_group = 10, skip = 3 would write output rows 14 and 15 past the 14 a caller allocates."""
    _expect_invalid(L, _layernorm(L, rows=25, in_group=10, skip=3), "in_group=10", "skip=3", "rows=25")
    _expect_invalid(L, _layernorm_bwd_grouped(L, rows=25, in_group=10, skip=3), "in_group=10", "skip=3", "rows=25")


@pytest.mark.parametrize("in_group,skip", [(1, 1), (4, 4), (4, 5), (4, -1), (0, 0)])
def test_layernorm_skip_must_be_less_than_in_group(L, in_group, skip):
    """(1, 1) used to be accepted: it writes nothing and leaves y uninitialised."""
    _expect_invalid(L, _layernorm(L, rows=24, in_group=in_group, skip=skip), "in_group", "skip")
    _expect_invalid(L, _layernorm_bwd_grouped(L, rows=24, in_group=in_group, skip=skip), "in_group", "skip")


@pytest.mark.parametrize("C", [2052, 4096, 0, 6])
def test_row_width_limits(L, C):
    for name in ("layernorm", "layernorm_bwd", "layernorm_bwd_grouped", "denoise_loss", "denoise_loss_ordered"):
        kw = {"C": C}
        if name == "layernorm":
            kw.update(ldx=max(C, 4) + 2 - (max(C, 4) + 2) % 4, ldy=max(C, 4) + 2 - (max(C, 4) + 2) % 4)
        _expect_invalid(L, BUILDERS[name](L, **kw), f"C={C}", "unsupported")


def test_other_shape_checks(L):
    _expect_invalid(L, _adamw(L, n=6), "multiple of 4")
    _expect_invalid(L, _adamw(L, step=0), "step")
    _expect_invalid(L, _colsum(L, dtype=BF16, cols=131, ld=132), "even")
    _expect_invalid(L, _colsum_ordered(L, cols=130, ld=132), "multiples of 4")
    _expect_invalid(L, _layerscale_bwd(L, C=770, ldx=772), "multiples of 4")
    _expect_invalid(L, _layerscale_bwd(L, branch=None), "dgamma")
    _expect_invalid(L, _embed_bwd(L, ntok=1), "bad shape")
    _expect_invalid(L, _embed_fwd(L, Kp=590), "bad shape")
    _expect_invalid(L, _layernorm(L, y_dtype=7), "y_dtype")
    lib = L.lib()
    _expect_invalid(L, lib.dvt_resample_bwd(P[0], P[1], P[2], P[3], P[4], 0, 37, 16, 16, 3, None), "bad shape")
    _expect_invalid(L, lib.dvt_im2col(P[0], F32, P[1], 2, 13, 224, 14, 14, None), "bad arguments")
    for K in (1, 256):
        _expect_invalid(L, lib.dvt_seg_upsample_ce(P[0], 2, 8, 8, K, P[1], 32, 32, 1.0, P[2], P[3], P[4], None), f"K={K}")
