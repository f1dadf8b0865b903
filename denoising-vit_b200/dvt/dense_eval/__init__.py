"""Dense-task linear probe (semantic segmentation) of a frozen, optionally denoised, backbone: the reference's
evaluate_dense_tasks.py with its linear configs, without mmcv / mmseg.  The full-resolution loss and the slide inference
run on the sm_90a kernels `dvt_seg_*`; BatchNorm and the 1x1 conv of the head are torch ops under autograd."""
from .config import ConfigError, DictAction, check_supported, load_config, merge_options  # noqa: F401
from .metrics import metrics_from_hist  # noqa: F401
from .trainer import evaluate, poly_lr, train  # noqa: F401
