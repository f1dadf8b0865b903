"""Dense-task linear probes of a frozen, optionally denoised, backbone: the reference's evaluate_dense_tasks.py with its
linear configs, without mmcv / mmseg.  Semantic segmentation: the full-resolution loss and the slide inference run on the
sm_90a kernels `dvt_seg_*`; BatchNorm and the 1x1 conv of the head are torch ops under autograd.  NYU depth (`depth`):
the bin-expectation head, the loss resize and the evaluation run on the kernels `dvt_depth_*`."""
from .config import ConfigError, DictAction, check_supported, check_supported_depth, load_config, merge_options  # noqa: F401
from .metrics import metrics_from_hist  # noqa: F401
from .trainer import evaluate, poly_lr, train  # noqa: F401
