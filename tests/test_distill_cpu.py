"""Stage-3 distillation without a GPU: the drop-in CLI (main_distillation.py) accepts every flag of the reference's parser
with the same type, default, action, nargs and choices (golden: tests/golden/make_distill_cli_golden.py reads the reference
source with ast), and the training path of the ViT wrapper refuses what it does not implement before touching a device."""
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _flags():
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    try:
        from make_cli_golden import flags
    finally:
        sys.path.pop(0)
    return flags


def test_distillation_cli_flags_match_the_reference():
    with open(os.path.join(ROOT, "tests", "golden", "cli_flags_distillation.json")) as fh:
        gold = json.load(fh)
    ours = _flags()(os.path.join(ROOT, "main_distillation.py"))
    ref = gold["main_distillation.py"]
    assert len(ref) >= 30 and "--denoiser_ckpt" in ref and "--grad_checkpointing" in ref
    for name, spec in ref.items():
        assert name in ours, f"main_distillation.py: flag {name} of the reference is missing"
        assert ours[name] == spec, f"main_distillation.py {name}: {ours[name]} != reference {spec}"


def test_distillation_cli_parses_like_the_reference():
    sys.path.insert(0, ROOT)
    import main_distillation as M
    with pytest.raises(SystemExit):          # --denoiser_ckpt is required, as in the reference
        M.get_args([])
    a = M.get_args(["--denoiser_ckpt", "x.pth"])
    assert a.num_iterations is None and a.num_epochs == 10 and a.input_size == [518, 518] and a.stride_size == 14
    assert a.grad_checkpointing is False and a.warmup_iters == 50_000
    a = M.get_args(["--denoiser_ckpt", "x.pth", "--model", "vit_base_patch16_224.dino", "--auto_stride"])
    assert a.stride_size == 16 and a.input_size == [512, 512]


def test_training_path_is_opt_in_and_refuses_unsupported_requests():
    import dvt.models as DVT
    from dvt import _lib
    w = DVT.PretrainedViTWrapper("vit_small_patch14_dinov2.lvd142m", stride=14, allow_random_init=True)
    x = torch.zeros(1, 3, 28, 28)
    with pytest.raises(_lib.DvtError):                       # inference path: CUDA only, as before
        w.get_intermediate_layers(x, n=[11])
    w.set_trainable(True)
    with pytest.raises(NotImplementedError):
        w.get_intermediate_layers(x, n=2)
    with pytest.raises(NotImplementedError):
        w.get_intermediate_layers(x, n=1, return_prefix_tokens=True)
    with pytest.raises(_lib.DvtError):                       # training path: CUDA only too
        w.get_intermediate_layers(x, n=1)
    with torch.no_grad(), pytest.raises(_lib.DvtError):      # no grad: the inference path even when trainable
        w.get_intermediate_layers(x, n=[11])
    w.model.set_grad_checkpointing(True)
    assert w.model._grad_ckpt
