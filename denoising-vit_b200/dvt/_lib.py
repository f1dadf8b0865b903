"""ctypes binding of include/dvt_b200.h.  Fails loudly when the shared object is missing or a call errors."""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_size_t, c_uint, c_void_p, POINTER

_HERE = os.path.dirname(os.path.abspath(__file__))
# DVT_LIB_PATH: load another build of the library (A/B measurements of two source revisions on one GPU box; symbols the
# other build lacks are skipped)
LIB_PATH = os.environ.get("DVT_LIB_PATH") or os.path.join(os.path.dirname(_HERE), "libdvt_b200.so")
# dvt_version() of the library SIGNATURES describes.  A library with another version is refused: an entry point may keep
# its name across versions but take other arguments, and calling it through these argtypes would pass garbage pointers.
ABI_VERSION = 104


class DvtError(RuntimeError):
    pass


_lib = None

# name -> (restype, argtypes); must list every symbol of include/dvt_b200.h (tests/test_abi.py checks this)
SIGNATURES = {
    "dvt_version": (c_int, []),
    "dvt_last_error": (c_char_p, []),
    "dvt_device_error": (c_int, [POINTER(c_uint)]),
    "dvt_set_debug_impl": (c_int, [c_int]),
    "dvt_launch_count": (ctypes.c_longlong, []),
    "dvt_gemm_tn": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p,
                            c_int, c_int, c_int, c_void_p]),
    "dvt_gemm_tn_residual": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                     c_void_p, c_int, c_void_p, c_int, c_void_p]),
    "dvt_layerscale_bwd": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                   c_void_p]),
    "dvt_vit_embed_fwd": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p,
                                  c_void_p]),
    "dvt_vit_embed_bwd": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_void_p]),
    "dvt_layernorm_bwd_grouped": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                          c_float, c_int, c_int, c_void_p]),
    "dvt_gemm_qkv_rope": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                  c_int, c_void_p, c_int, c_void_p]),
    "dvt_rope_bwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "dvt_swiglu": (c_int, [c_void_p, c_void_p, c_size_t, c_int, c_void_p]),
    "dvt_gemm_bf16_dgrad_swiglu": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p,
                                           c_int, c_void_p]),
    "dvt_attention_bwd_det": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                      c_void_p]),
    "dvt_gemm_bf16_wgrad_ordered": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int,
                                            c_void_p, c_void_p]),
    "dvt_colsum_ordered": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "dvt_denoise_loss_ordered": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p]),
    "dvt_resample_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "dvt_layernorm": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_int,
                              c_int, c_void_p]),
    "dvt_attention_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "dvt_attention_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                  c_int, c_void_p]),
    "dvt_layernorm_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p]),
    "dvt_colsum": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "dvt_gelu": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "dvt_gemm_bf16": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int,
                              c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "dvt_denoise_loss": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p]),
    "dvt_adamw": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_double, c_double, c_double, c_double, c_double,
                          ctypes.c_longlong, c_void_p]),
    "dvt_im2col": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "dvt_gemm_f32x3": (c_int, [c_void_p, c_int, c_size_t, c_int, c_void_p, c_int, c_size_t, c_int, c_int, c_int, c_int,
                               c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "dvt_hashgrid_corners": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                     c_void_p, c_void_p]),
    "dvt_hashgrid_fwd": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                 c_void_p, c_void_p]),
    "dvt_hashgrid_bwd": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                 c_void_p, c_void_p]),
    "dvt_fit_create": (c_int, [POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                               c_void_p, c_void_p]),
    "dvt_fit_destroy": (None, [c_void_p]),
    "dvt_fit_set_param": (c_int, [c_void_p, c_char_p, c_void_p, c_size_t, c_void_p]),
    "dvt_fit_init_params": (c_int, [c_void_p, ctypes.c_ulonglong, c_void_p]),
    "dvt_fit_check": (c_int, [c_void_p]),
    "dvt_fit_set_artifact_grid": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "dvt_fit_losses_async": (c_int, [c_void_p, c_void_p, c_int, c_void_p]),
    "dvt_fit_get_param": (c_int, [c_void_p, c_char_p, c_void_p, c_size_t]),
    "dvt_fit_begin": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_int, c_double, c_double, c_int, c_int,
                              c_double, c_double, c_int, c_void_p]),
    "dvt_fit_run": (c_int, [c_void_p, c_int, c_int, c_void_p]),
    "dvt_fit_losses": (c_int, [c_void_p, c_void_p, c_int]),
    "dvt_fit_query": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "dvt_fit_residual": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "dvt_fit_sweep_once": (c_int, [c_void_p, c_int, c_void_p]),
    "dvt_view_crops": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p,
                               c_int, c_int, c_void_p]),
    "dvt_seg_upsample_ce": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_float, c_void_p, c_void_p,
                                    c_void_p, c_void_p]),
    "dvt_seg_slide_accumulate": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int,
                                         c_int, c_void_p]),
    "dvt_seg_predict_hist": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "dvt_seg_aug_accumulate": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p]),
    "dvt_seg_aug_argmax_hist": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "dvt_depth_head_fwd": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "dvt_depth_head_bwd": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dvt_depth_resize_fwd": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p]),
    "dvt_depth_resize_bwd": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "dvt_depth_eval_sums": (c_int, [c_void_p, c_int, c_uint, c_int, c_int, c_void_p, c_int, c_int, c_float, c_float, c_int,
                                    c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "dvt_vit_create": (c_int, [POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_int,
                               c_int, c_int]),
    "dvt_vit_destroy": (None, [c_void_p]),
    "dvt_vit_load": (c_int, [c_void_p, c_char_p, c_void_p, c_size_t]),
    "dvt_vit_reserve": (c_int, [c_void_p, c_int, c_int, c_int, c_int]),
    "dvt_vit_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                c_int, c_void_p, c_int, c_void_p]),
    "dvt_vit_forward_layers": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                       c_int, POINTER(c_int), c_int, POINTER(c_void_p), c_int, c_int, POINTER(c_void_p),
                                       c_void_p]),
}


def lib():
    global _lib
    if _lib is None:
        if not os.path.isfile(LIB_PATH):
            raise DvtError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback)")
        l = ctypes.CDLL(LIB_PATH)
        l.dvt_version.restype = c_int
        l.dvt_version.argtypes = []
        if l.dvt_version() != ABI_VERSION:
            raise DvtError(f"{LIB_PATH} has ABI version {l.dvt_version()}, this binding needs {ABI_VERSION}: rebuild it")
        for name, (res, args) in SIGNATURES.items():
            if not hasattr(l, name) and os.environ.get("DVT_LIB_PATH"):
                continue
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = lib().dvt_last_error().decode("utf-8", "replace")
        raise DvtError(f"{what} failed (code {rc}): {msg}")


def device_error() -> int:
    code = c_uint(0)
    check(lib().dvt_device_error(ctypes.byref(code)), "dvt_device_error")
    return code.value


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    return None if t is None else c_void_p(t.data_ptr())


def cur_stream():
    import torch
    return c_void_p(torch.cuda.current_stream().cuda_stream)


DT_BF16, DT_F32 = 0, 1
