"""Config files of the reference's dense-task evaluation (evaluation/configs/*_linear_config.py) without mmcv.

Those files are self-contained Python: `load_config` executes one and returns its top-level names as a plain dict tree,
which is what mmcv's `Config.fromfile` gives for them.  Inheritance (`_base_`) is not supported.  `DictAction` parses
`--cfg-options key=value` like mmcv's (ints, floats, true / false, None, strings; `[a,b]`, `a,b` and `(a,b)` lists and
tuples, nested), and `merge_options` applies dotted keys, list indices included (`data.train.pipeline.2.prob=0.3`).
`check_supported` refuses, with the name of what is missing, any model, dataset, pipeline or schedule element that
`dvt.dense_eval` does not implement."""
from __future__ import annotations

import argparse
import copy
import types
from typing import Any, Dict


class ConfigError(NotImplementedError):
    pass


def load_config(path: str) -> Dict[str, Any]:
    with open(path) as fh:
        src = fh.read()
    ns: Dict[str, Any] = {"__file__": path, "__name__": "__dense_eval_config__"}
    exec(compile(src, path, "exec"), ns)
    cfg = {k: v for k, v in ns.items() if not k.startswith("__")
           and not isinstance(v, (types.ModuleType, types.FunctionType, type))}
    if "_base_" in cfg:
        raise ConfigError(f"{path}: `_base_` (config inheritance) is not supported; write the config out in full")
    return cfg


def _scalar(v: str):
    for cast in (int, float):
        try:
            return cast(v)
        except ValueError:
            pass
    if v.lower() in ("true", "false"):
        return v.lower() == "true"
    if v == "None":
        return None
    return v


def _next_comma(s: str) -> int:
    depth = 0
    for i, ch in enumerate(s):
        if ch in "([":
            depth += 1
        elif ch in ")]":
            depth -= 1
        elif ch == "," and depth == 0:
            return i
    return len(s)


def parse_value(val: str):
    """mmcv DictAction._parse_iterable."""
    val = val.strip("'\"").replace(" ", "")
    is_tuple = False
    if val.startswith("(") and val.endswith(")"):
        is_tuple, val = True, val[1:-1]
    elif val.startswith("[") and val.endswith("]"):
        val = val[1:-1]
    elif "," not in val:
        return _scalar(val)
    out = []
    while val:
        i = _next_comma(val)
        out.append(parse_value(val[:i]))
        val = val[i + 1:]
    return tuple(out) if is_tuple else out


class DictAction(argparse.Action):
    """argparse action of `--cfg-options a.b=1 c=[x,y]`: a dict of dotted keys to parsed values."""

    def __call__(self, parser, namespace, values, option_string=None):
        options = copy.copy(getattr(namespace, self.dest, None) or {})
        for kv in values:
            key, val = kv.split("=", maxsplit=1)
            options[key] = parse_value(val)
        setattr(namespace, self.dest, options)


def merge_options(cfg: Dict[str, Any], options: Dict[str, Any]) -> Dict[str, Any]:
    for key, val in options.items():
        node = cfg
        parts = key.split(".")
        for p in parts[:-1]:
            if isinstance(node, list):
                node = node[int(p)]
            else:
                node = node.setdefault(p, {})
        if isinstance(node, list):
            node[int(parts[-1])] = val
        else:
            node[parts[-1]] = val
    return cfg


TRAIN_PIPELINE = ("LoadImageFromFile", "LoadAnnotations", "Resize", "RandomCrop", "RandomFlip", "PhotoMetricDistortion",
                  "Normalize", "Pad", "DefaultFormatBundle", "Collect")
TEST_PIPELINE = ("LoadImageFromFile", "MultiScaleFlipAug", "Resize", "RandomFlip", "Normalize", "ImageToTensor", "Collect")
DATASETS = ("PascalVOCDataset", "ADE20KDataset")


def _require(cond: bool, msg: str):
    if not cond:
        raise ConfigError(msg)


def check_supported(cfg: Dict[str, Any]) -> None:
    model = cfg.get("model", {})
    _require(model.get("type") == "EncoderDecoder", f"model type {model.get('type')!r}: only EncoderDecoder is implemented")
    head = model.get("decode_head", {})
    _require(head.get("type") == "BNHead", f"decode_head type {head.get('type')!r}: only the linear BNHead is implemented")
    _require(head.get("input_transform") == "resize_concat",
             f"BNHead input_transform {head.get('input_transform')!r}: only resize_concat is implemented")
    _require(not head.get("align_corners", False), "BNHead align_corners=True is not implemented")
    _require(head.get("resize_factors") is None, "BNHead resize_factors is not implemented")
    _require(not head.get("dropout_ratio", 0), "BNHead dropout is not implemented (the linear configs use dropout_ratio=0)")
    loss = head.get("loss_decode", {"type": "CrossEntropyLoss"})
    _require(loss.get("type") == "CrossEntropyLoss" and not loss.get("use_sigmoid", False)
             and loss.get("loss_weight", 1.0) == 1.0 and not loss.get("avg_non_ignore", False)
             and loss.get("class_weight") is None,
             f"loss_decode {loss}: only softmax CrossEntropyLoss, weight 1, mean over all pixels, is implemented")
    test_cfg = model.get("test_cfg", cfg.get("test_cfg", {})) or {}
    _require(test_cfg.get("mode") == "slide", f"test_cfg mode {test_cfg.get('mode')!r}: only slide inference is implemented")
    opt = cfg.get("optimizer", {})
    _require(opt.get("type") == "AdamW", f"optimizer {opt.get('type')!r}: only AdamW is implemented")
    _require(not opt.get("paramwise_cfg"), "optimizer paramwise_cfg is not implemented")
    lr = cfg.get("lr_config", {})
    _require(lr.get("policy") == "poly" and not lr.get("by_epoch", False),
             f"lr_config policy {lr.get('policy')!r}: only the iteration-based poly schedule is implemented")
    _require(lr.get("warmup") in (None, "linear"), f"lr_config warmup {lr.get('warmup')!r}: only linear warmup is implemented")
    _require(cfg.get("runner", {}).get("type") == "IterBasedRunner", "runner: only IterBasedRunner is implemented")
    _require(len(cfg.get("workflow", [("train", 1)])) == 1, "workflow: only [('train', 1)] is implemented")
    oc = cfg.get("optimizer_config", {}) or {}
    _require(oc.get("grad_clip") is None and not oc.get("use_fp16", False) and oc.get("update_interval", 1) == 1,
             "optimizer_config: gradient clipping, fp16 and accumulation are not implemented")
    data = cfg.get("data", {})
    for split in ("train", "val"):
        ds = data.get(split, {})
        _require(ds.get("type") in DATASETS, f"data.{split} type {ds.get('type')!r}: implemented: {', '.join(DATASETS)}")
        allowed = TRAIN_PIPELINE if split == "train" else TEST_PIPELINE
        steps = list(ds.get("pipeline", []))
        for step in list(steps):
            steps.extend(step.get("transforms", []))
        for step in steps:
            _require(step.get("type") in allowed, f"data.{split} pipeline step {step.get('type')!r} is not implemented")


DEPTH_TRAIN_PIPELINE = ("LoadImageFromFile", "DepthLoadAnnotations", "NYUCrop", "RandomRotate", "RandomFlip", "RandomCrop",
                        "ColorAug", "Normalize", "DefaultFormatBundle", "Collect")
DEPTH_TEST_PIPELINE = ("LoadImageFromFile", "MultiScaleFlipAug", "RandomFlip", "Normalize", "ImageToTensor", "Collect")
MAX_DEPTH_BINS = 256


def check_supported_depth(cfg: Dict[str, Any]) -> None:
    """The NYU depth probe (vitb_nyu_linear_config.py): refuses, naming it, what `dvt.dense_eval.depth` does not
    implement."""
    model = cfg.get("model", {})
    _require(model.get("type") == "DepthEncoderDecoder",
             f"model type {model.get('type')!r}: the depth probe implements DepthEncoderDecoder")
    bb = model.get("backbone", {})
    _require(bb.get("output_cls_token", True),
             "backbone output_cls_token=False is not implemented (the reference's format_output would then index the batch)")
    head = model.get("decode_head", {})
    _require(head.get("type") == "BNHead", f"decode_head type {head.get('type')!r}: only the linear BNHead is implemented")
    _require(head.get("classify", False), "BNHead classify=False (direct regression) is not implemented")
    _require(head.get("bins_strategy", "UD") == "UD", f"BNHead bins_strategy {head.get('bins_strategy')!r}: only UD is "
             f"implemented (SID is not)")
    _require(head.get("norm_strategy", "linear") == "linear",
             f"BNHead norm_strategy {head.get('norm_strategy')!r}: only linear is implemented")
    _require(int(head.get("n_bins", 256)) <= MAX_DEPTH_BINS,
             f"BNHead n_bins {head.get('n_bins')}: at most {MAX_DEPTH_BINS} bins are implemented")
    _require(head.get("input_transform") == "resize_concat",
             f"BNHead input_transform {head.get('input_transform')!r}: only resize_concat is implemented")
    _require(not head.get("align_corners", False), "BNHead align_corners=True is not implemented")
    _require(not head.get("scale_up", False), "BNHead scale_up is not implemented")
    losses = head.get("loss_decode", [])
    losses = [losses] if isinstance(losses, dict) else list(losses)
    kinds = [(l.get("type"), l.get("valid_mask", True), l.get("max_depth")) for l in losses]
    _require(sorted(k[0] for k in kinds) == ["GradientLoss", "SigLoss"] and all(k[1] and k[2] is None for k in kinds),
             f"loss_decode {losses}: only SigLoss + GradientLoss with valid_mask and no max_depth are implemented")
    test_cfg = model.get("test_cfg", cfg.get("test_cfg", {})) or {}
    _require(test_cfg.get("mode") == "whole", f"test_cfg mode {test_cfg.get('mode')!r}: only whole inference is implemented")
    opt = cfg.get("optimizer", {})
    _require(opt.get("type") == "AdamW", f"optimizer {opt.get('type')!r}: only AdamW is implemented")
    pw = opt.get("paramwise_cfg") or {}
    _require(set(pw) <= {"custom_keys"}, f"optimizer paramwise_cfg {sorted(pw)}: only custom_keys is implemented")
    lr = cfg.get("lr_config", {})
    _require(lr.get("policy") == "CosineAnnealing" and not lr.get("by_epoch", False) and "min_lr" not in lr,
             f"lr_config policy {lr.get('policy')!r}: only the iteration-based CosineAnnealing schedule with min_lr_ratio "
             f"is implemented")
    _require(lr.get("warmup") in (None, "linear"), f"lr_config warmup {lr.get('warmup')!r}: only linear warmup is implemented")
    mom = cfg.get("momentum_config")
    _require(mom is None or mom.get("policy") == "OneCycle",
             f"momentum_config policy {(mom or {}).get('policy')!r}: only OneCycle is implemented")
    _require(cfg.get("runner", {}).get("type") == "IterBasedRunner", "runner: only IterBasedRunner is implemented")
    _require(len(cfg.get("workflow", [("train", 1)])) == 1, "workflow: only [('train', 1)] is implemented")
    oc = cfg.get("optimizer_config", {}) or {}
    clip = oc.get("grad_clip")
    _require((clip is None or clip.get("norm_type", 2) == 2) and not oc.get("use_fp16", False)
             and oc.get("update_interval", 1) == 1,
             "optimizer_config: only L2 gradient clipping, without fp16 or accumulation, is implemented")
    ev = cfg.get("evaluation", {})
    _require(ev.get("rule", "less") in ("less", "greater"), f"evaluation rule {ev.get('rule')!r} is not implemented")
    data = cfg.get("data", {})
    for split in ("train", "val"):
        ds = data.get(split, {})
        _require(ds.get("type") == "NYUDataset", f"data.{split} type {ds.get('type')!r}: only NYUDataset is implemented")
        _require(ds.get("split") is not None, f"data.{split}: a split file is required (as in the reference)")
        allowed = DEPTH_TRAIN_PIPELINE if split == "train" else DEPTH_TEST_PIPELINE
        steps = list(ds.get("pipeline", []))
        for step in list(steps):
            steps.extend(step.get("transforms", []))
        for step in steps:
            _require(step.get("type") in allowed, f"data.{split} pipeline step {step.get('type')!r} is not implemented")
