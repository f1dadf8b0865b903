"""Dense-task linear probe on H100 -- drop-in for the reference's evaluate_dense_tasks.py (semantic segmentation).

Same flags (reference evaluate_dense_tasks.py:34-124), same config files (evaluation/configs/vitb_voc2012_linear_config.py,
vitb_ade20k_linear_config.py, read as plain Python: no mmcv), same backbones (:177-214: the ViT wrapper at stride = patch,
optionally with `--load-distilled-model-from`, optionally under the `--load-denoiser-from` Denoiser), same probe (frozen
backbone behind CenterPadding, BNHead on the `in_index` features, cross-entropy of the bilinearly upsampled logits,
AdamW + poly schedule with linear warmup, slide inference, mIoU / mAcc / aAcc).  Only the layers `in_index` selects are
computed.  The full-resolution loss and slide inference run on sm_90a kernels (dvt/dense_eval), and so does mmseg's
multi-scale + flip test (e.g. `--cfg-options data.val.pipeline.1.img_ratios=[0.5,0.75,1.0,1.25,1.5,1.75]
data.val.pipeline.1.flip=True`).

Outputs in the work dir: `iter_<n>.pth` every checkpoint_config.interval iterations and at the end ({"state_dict":
decode_head.* weights, "optimizer", "iter"}), `latest.pth` pointing at the newest, and `<timestamp>.log.json` (one JSON
object per line: training losses every log_config.interval iterations, and mIoU, mAcc, aAcc, per-class IoU / Acc of
every evaluation, as fractions).  `--task depth` is refused: the NYU depth probe is evaluate_depth.py.

Launch: `--launcher none` runs one process; `--launcher pytorch` (the default, as in the reference) runs under torchrun,
one process per GPU, with SyncBatchNorm in the head and DDP over NCCL."""
import argparse
import os
import os.path as osp
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "denoising-vit_b200"))

from dvt.dense_eval import DictAction, check_supported  # noqa: E402
from dvt.dense_eval.launch import finish_run, init_run, load_run_config  # noqa: E402


def parse_args(argv=None):
    parser = argparse.ArgumentParser("Linear Evaluation", add_help=False)
    parser.add_argument("config", help="train config file path")
    parser.add_argument("--work-dir", help="the dir to save logs and models")
    parser.add_argument("--load-denoiser-from", help="the checkpoint file to load weights from")
    parser.add_argument("--load-distilled-model-from", help="the checkpoint file to load weights from")
    parser.add_argument("--num_blocks", type=int, default=1)
    parser.add_argument("--resume-from", help="the checkpoint file to resume from")
    parser.add_argument("--backbone-type", default="vit_small_patch14_dinov2.lvd142m", help="timm model type")
    parser.add_argument("--task", type=str, default="segmentation", choices=["segmentation", "depth"], help="task to train")
    parser.add_argument("--no-validate", action="store_true", help="whether not to evaluate the checkpoint during training")
    parser.add_argument("--seed", type=int, default=None, help="random seed")
    parser.add_argument("--diff_seed", action="store_true", help="Whether or not set different seeds for different ranks")
    parser.add_argument("--deterministic", action="store_true",
                        help="torch.use_deterministic_algorithms(True): a rerun from the same seed on the same GPU model "
                             "gives bit-identical head weights and metrics")
    parser.add_argument("--options", nargs="+", action=DictAction,
                        help="deprecated alias of --cfg-options (merged after it)")
    parser.add_argument("--cfg-options", nargs="+", action=DictAction,
                        help="override settings of the config: key=value pairs with dotted keys, e.g. "
                             "model.decode_head.num_classes=150 or runner.max_iters=1000; lists as key=[a,b] or key=a,b")
    parser.add_argument("--launcher", choices=["none", "pytorch", "slurm", "mpi"], default="pytorch", help="job launcher")
    parser.add_argument("--local-rank", type=int, default=0)
    parser.add_argument("--auto-resume", action="store_true", help="resume from the latest checkpoint automatically.")
    args = parser.parse_args(argv)
    if "LOCAL_RANK" not in os.environ:
        os.environ["LOCAL_RANK"] = str(args.local_rank)
    return args


def main(args):
    if args.task == "depth":
        raise NotImplementedError("--task depth: evaluate_dense_tasks.py runs the segmentation probe only; the NYU depth "
                                  "probe is evaluate_depth.py (same flags and config files)")
    cfg, resume_from = load_run_config(args, check_supported)
    rank, world, device, seed, timestamp = init_run(args, cfg, "segmentation probe")
    from dvt.dense_eval.model import build_backbone
    from dvt.dense_eval.trainer import train
    backbone = build_backbone(args.backbone_type, args.load_distilled_model_from, args.load_denoiser_from, args.num_blocks,
                              device)
    out = train(cfg, backbone, cfg["work_dir"], seed, device, validate=not args.no_validate, resume_from=resume_from,
                timestamp=timestamp, exp_name=osp.basename(args.config))
    finish_run(world)
    return out


if __name__ == "__main__":
    main(parse_args())
