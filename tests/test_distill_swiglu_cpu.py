"""The SwiGLU ViT-g/14 backbones on the stage-3 training path, without a GPU: the path accepts them and, like every other
backbone, refuses CPU tensors with DvtError (there is no CPU fallback)."""
import pytest
import torch


@pytest.mark.parametrize("ident", ["vit_giant_patch14_dinov2.lvd142m", "vit_giant_patch14_reg4_dinov2.lvd142m"])
@pytest.mark.parametrize("ckpt", [False, True], ids=["plain", "checkpointed"])
def test_vitg_training_path_refuses_cpu_tensors_with_dvt_error(ident, ckpt, monkeypatch):
    import dvt.models as DVT
    from dvt import _lib
    from dvt.models import vit_wrapper as VW
    monkeypatch.setitem(VW.ARCHS, ident, {**VW.ARCHS[ident], "depth": 1})   # the layout of ViT-g, one block
    w = DVT.PretrainedViTWrapper(ident, stride=14, allow_random_init=True)
    assert w.model.arch["swiglu"] and w.model.blocks[0].mlp.fc2.in_features * 2 == w.model.blocks[0].mlp.fc1.out_features
    w.set_trainable(True)
    w.model.set_grad_checkpointing(ckpt)
    x = torch.zeros(1, 3, 28, 28)
    try:
        w.get_intermediate_layers(x, n=1)
    except NotImplementedError as e:                          # the SwiGLU backward exists: no refusal any more
        pytest.fail(f"ViT-g training path refused: {e}")
    except _lib.DvtError:
        pass
    else:
        pytest.fail("the training path ran on CPU tensors")
