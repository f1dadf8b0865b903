"""dvt -- drop-in for the hot paths of Denoising-ViT's `dvt` package, backed by libdvt_b200.so (sm_90a).

Mirrors the reference package layout (`dvt.models`, `dvt.utils.misc`) so `import dvt.models as DVT` keeps working
(reference: dvt/models/__init__.py:1-4).  There is no CPU fallback: anything that computes needs the CUDA library.
"""
