"""The C-ABI library must load on a CPU-only machine and export every symbol include/dvt_b200.h declares; the ctypes
binding must cover all of them.  No compute calls here."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dvt_b200.h")


def _declared():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dvt_[a-z0-9_]+)\s*\(", src)))


def _lib_path():
    from dvt import _lib
    if not os.path.isfile(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    return _lib.LIB_PATH


def test_header_declares_entry_points():
    names = _declared()
    for must in ("dvt_vit_forward", "dvt_fit_run", "dvt_gemm_tn", "dvt_attention_fwd", "dvt_hashgrid_fwd", "dvt_last_error"):
        assert must in names
    assert len(names) >= 25


def test_library_exports_every_declared_symbol():
    lib = ctypes.CDLL(_lib_path())
    for name in _declared():
        assert hasattr(lib, name), f"{name} declared in include/dvt_b200.h but not exported"


def test_ctypes_binding_covers_header():
    from dvt import _lib
    assert sorted(_lib.SIGNATURES) == _declared()
    L = _lib.lib()
    assert L.dvt_version() == _lib.ABI_VERSION
    assert L.dvt_last_error() is not None


def test_no_cpu_fallback():
    """Operators refuse CPU tensors instead of silently computing on the host."""
    import torch
    from dvt import _lib, ops
    a = torch.zeros(8, 8, dtype=torch.bfloat16)
    with pytest.raises(_lib.DvtError):
        ops.gemm_tn(a, a)
    import dvt.models as DVT
    w = DVT.PretrainedViTWrapper("vit_small_patch14_dinov2.lvd142m", stride=14, allow_random_init=True)
    with pytest.raises(_lib.DvtError):
        w.get_intermediate_layers(torch.zeros(1, 3, 28, 28), n=[11])


def test_error_reporting_without_gpu():
    from dvt import _lib
    L = _lib.lib()
    rc = L.dvt_set_debug_impl(7)
    assert rc == 1 and b"impl must be" in L.dvt_last_error()


def test_missing_weights_raise_unless_random_init_is_explicit(monkeypatch):
    """Advisor finding (round 1): a backbone without pretrained weights must not be a silent fallback -- the reference
    builds it with timm `pretrained=True` and fails when the checkpoint is unavailable (vit_wrapper.py:108-112)."""
    import dvt.models as DVT
    monkeypatch.delenv("DVT_ALLOW_RANDOM_INIT", raising=False)
    monkeypatch.delenv("DVT_WEIGHTS_DIR", raising=False)
    with pytest.raises(FileNotFoundError):
        DVT.PretrainedViTWrapper("vit_small_patch14_dinov2.lvd142m", stride=14)
    w = DVT.PretrainedViTWrapper("vit_small_patch14_dinov2.lvd142m", stride=14, allow_random_init=True)
    assert w.pretrained_loaded is False
    monkeypatch.setenv("DVT_ALLOW_RANDOM_INIT", "1")
    DVT.PretrainedViTWrapper("vit_small_patch14_dinov2.lvd142m", stride=14)
