"""Multi-layer ViT extraction without a GPU: every refusal of dvt_vit_forward_layers that does not need the handle names
its argument (the entry point makes these checks before it looks at the handle, so they run here with a null one), the
inference path still refuses CPU tensors, and the four-layer linear-probe configs (in_index [0, 1, 2, 3] of out_indices
[8, 9, 10, 11]) pass the probes' config checks and size their heads at 4 C.

As in test_kernel_args_cpu.py the device pointers are fake integers and nothing is dereferenced; the file runs only where
there is no GPU.  The refusals that need the handle (an index past the depth, ldo < C) are in test_vit_layers_gpu.py."""
import ctypes
import json
import os

import pytest
import torch

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="fake device pointers: run on a machine without a GPU")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
DVT_ERR_INVALID = 1
F32 = 1
BASE = 1 << 32
P = [BASE + i * (1 << 24) for i in range(12)]
C = 384


@pytest.fixture(scope="module")
def L():
    from dvt import _lib
    return _lib


def _call(L, h=None, x=P[0], pos_patch=P[1], prefix_rows=P[2], rope=None, layers=(8, 9, 10, 11), norm=0, out="concat",
          ldo=4 * C, all_tokens=0, prefix_out=None, n_layers=None):
    n = len(layers) if n_layers is None else n_layers
    idx = (ctypes.c_int * max(len(layers), 1))(*layers) if layers is not None else None
    if out == "concat":
        out = [P[3] + 4 * C * l for l in range(len(layers))]
    outs = (ctypes.c_void_p * max(len(out), 1))(*out) if out is not None else None
    pre = (ctypes.c_void_p * len(prefix_out))(*prefix_out) if prefix_out is not None else None
    return L.lib().dvt_vit_forward_layers(h, x, F32, 2, 224, 224, 14, pos_patch, prefix_rows, rope, n, idx, norm, outs, ldo,
                                          all_tokens, pre, None)


def _refused(L, needle, **kw):
    rc = _call(L, **kw)
    msg = L.lib().dvt_last_error().decode()
    assert rc == DVT_ERR_INVALID and needle in msg, (rc, msg)


def test_a_well_formed_call_gets_as_far_as_the_handle(L):
    _refused(L, "null handle")
    _refused(L, "null handle", prefix_out=[P[5] + l * 4096 for l in range(4)])
    _refused(L, "null handle", layers=(0,), out=[P[3]], ldo=C, all_tokens=1)


@pytest.mark.parametrize("case, needle", [
    (dict(x=None), "x is null"),
    (dict(prefix_rows=None), "prefix_rows is null"),
    (dict(layers=(), out=[]), "n_layers >= 1"),
    (dict(layers=None, n_layers=4, out=[P[3], P[4], P[5], P[6]]), "layer_indices must list"),
    (dict(layers=(-1, 9, 10, 11)), "layer_indices[0]=-1 is negative"),
    (dict(layers=(8, 10, 9, 11)), "strictly ascending (layer_indices[2]=9 after 10)"),
    (dict(layers=(8, 9, 9, 11)), "strictly ascending (layer_indices[2]=9 after 9)"),
    (dict(ldo=4 * C + 2), "ldo=1538 must be a positive multiple of 4"),
    (dict(ldo=0), "ldo=0 must be a positive multiple of 4"),
    (dict(out=None), "out is null"),
    (dict(out=[P[3], P[4], 0, P[6]]), "out[2] is null"),
    (dict(out=[P[3], P[4] + 8, P[5], P[6]]), "out[1] must be 16-byte aligned"),
    (dict(all_tokens=1, prefix_out=[P[5], P[6], P[7], P[8]]), "prefix_out with all_tokens"),
    (dict(prefix_out=[P[5], P[6], P[7], 0]), "prefix_out[3] is null"),
    (dict(prefix_out=[P[5], P[6], P[7] + 4, P[8]]), "prefix_out[2] must be 16-byte aligned"),
], ids=["x", "prefix_rows", "n_layers", "layer_indices", "negative", "unsorted", "duplicated", "ldo_mod4", "ldo_zero",
        "out", "out_entry", "out_aligned", "all_tokens_prefix_out", "prefix_out_entry", "prefix_out_aligned"])
def test_refusals_name_the_argument(L, case, needle):
    _refused(L, needle, **case)


def test_get_intermediate_layers_refuses_a_cpu_tensor(L):
    import dvt.models as DVT
    w = DVT.PretrainedViTWrapper("vit_small_patch14_dinov2.lvd142m", stride=14, allow_random_init=True)
    x = torch.zeros(1, 3, 28, 28)
    for n in ([8, 9, 10, 11], [11, 8, 8], 4):
        with pytest.raises(L.DvtError):
            w.get_intermediate_layers(x, n=n)
    with pytest.raises(L.DvtError):
        w.model.forward_layers_concat(x, [8, 9, 10, 11], norm=False, return_cls=True)
    assert w.get_intermediate_layers(x, n=0) == []


def _golden(name):
    with open(os.path.join(GOLDEN, name)) as fh:
        return json.load(fh)


FOUR = {"model.decode_head.in_index": [0, 1, 2, 3], "model.decode_head.in_channels": [C] * 4}


@pytest.mark.parametrize("config", ["vitb_voc2012_linear_config.py", "vitb_ade20k_linear_config.py"])
def test_four_layer_segmentation_config_is_supported(config):
    import dvt.models as DVT
    from dvt.dense_eval.config import check_supported, merge_options
    from dvt.dense_eval.model import LinearSegHead, ProbeBackbone, in_channels_of
    cfg = merge_options(_golden("dense_eval_configs.json")[config], {**FOUR, "model.decode_head.channels": 4 * C})
    check_supported(cfg)
    head = cfg["model"]["decode_head"]
    assert in_channels_of(head) == [C] * 4
    vit = DVT.PretrainedViTWrapper("vit_small_patch14_dinov2.lvd142m", stride=14, allow_random_init=True)
    probe = ProbeBackbone(vit, cfg["model"]["backbone"]["out_indices"], head["in_index"])
    assert probe.layers == [8, 9, 10, 11] and probe.channels == sum(in_channels_of(head)) == head["channels"] == 4 * C
    assert LinearSegHead(probe.channels, 21).bn.weight.shape == (4 * C,)


def test_four_layer_depth_config_is_supported():
    import dvt.models as DVT
    from dvt.dense_eval.config import check_supported_depth, merge_options
    from dvt.dense_eval.depth import build_head
    from dvt.dense_eval.model import ProbeBackbone, in_channels_of
    cfg = merge_options(_golden("depth_config.json"), {**FOUR, "model.decode_head.channels": 8 * C,
                                                       "model.backbone.out_indices": [8, 9, 10, 11]})
    check_supported_depth(cfg)
    head_cfg = cfg["model"]["decode_head"]
    assert in_channels_of(head_cfg) == [C] * 4
    vit = DVT.PretrainedViTWrapper("vit_small_patch14_dinov2.lvd142m", stride=14, allow_random_init=True)
    probe = ProbeBackbone(vit, cfg["model"]["backbone"]["out_indices"], head_cfg["in_index"], return_cls=True)
    assert probe.layers == [8, 9, 10, 11] and probe.channels == 4 * C
    head = build_head(cfg, probe, "cpu")
    assert head.conv_depth.weight.shape == (int(head_cfg.get("n_bins", 256)), 8 * C, 1, 1) and head.n_maps == 4
