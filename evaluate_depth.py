"""NYU-Depth linear probe on H100 -- the reference's `evaluate_dense_tasks.py --task depth` with
evaluation/configs/vitb_nyu_linear_config.py, without mmcv / mmseg.

Same flags as evaluate_dense_tasks.py (its parser; `--task` is accepted and the depth probe runs whatever it says), same
config files (read as plain Python; only DepthEncoderDecoder configs are accepted), same backbones (the ViT wrapper,
optionally with `--load-distilled-model-from`, optionally under the `--load-denoiser-from` Denoiser).  The probe: a frozen
backbone behind CenterPadding read with the final norm and the cls token, the BNHead bin-classification head (256 depth
bins, upsample x4), SigLoss + GradientLoss on the prediction resized to the ground truth, AdamW with gradient clipping,
cosine LR with linear warmup and OneCycle momentum, whole-image evaluation with flip test-time augmentation and the nine
NYU metrics (a1, a2, a3, abs_rel, rmse, log_10, rmse_log, silog, sq_rel) averaged over images.  The head's upsampled
map, the loss resize and the evaluation run on sm_90a kernels (dvt/dense_eval/depth_ops.py).

Outputs in the work dir: `iter_<n>.pth` every checkpoint_config.interval iterations and at the end (the newest
max_keep_ckpts kept), `latest.pth` pointing at the newest, `best_<save_best>_iter_<n>.pth` (the best evaluation so far,
the previous one removed) and `<timestamp>.log.json` (decode.loss_depth, decode.loss_grad and loss every
log_config.interval iterations; the nine metrics of every evaluation).

Launch: `--launcher none` runs one process; `--launcher pytorch` (the default) runs under torchrun, one process per GPU,
with DDP over NCCL and each rank evaluating a disjoint share of the images."""
import os
import os.path as osp
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "denoising-vit_b200"))
sys.path.insert(0, ROOT)

from evaluate_dense_tasks import parse_args  # noqa: E402
from dvt.dense_eval import check_supported_depth  # noqa: E402
from dvt.dense_eval.launch import finish_run, init_run, load_run_config  # noqa: E402


def main(args):
    cfg, resume_from = load_run_config(args, check_supported_depth)
    rank, world, device, seed, timestamp = init_run(args, cfg, "depth probe")
    from dvt.dense_eval import depth
    from dvt.dense_eval.model import build_backbone
    backbone = build_backbone(args.backbone_type, args.load_distilled_model_from, args.load_denoiser_from, args.num_blocks,
                              device)
    out = depth.train(cfg, backbone, cfg["work_dir"], seed, device, validate=not args.no_validate,
                      resume_from=resume_from or None, timestamp=timestamp, exp_name=osp.basename(args.config))
    finish_run(world)
    return out


if __name__ == "__main__":
    main(parse_args())
