"""Generates the goldens of the segmentation probe from the reference sources:

- tests/golden/cli_flags_dense_eval.json: every `add_argument` of /root/reference/evaluate_dense_tasks.py:34-124 with its
  `type`, `default`, `action`, `nargs` and `choices` expressions, read with `ast` by `make_cli_golden.flags` (the module
  imports mmcv / mmseg and cannot be executed here);
- tests/golden/dense_eval_configs.json: the top-level names of the two linear configs
  (evaluation/configs/vitb_voc2012_linear_config.py, vitb_ade20k_linear_config.py) as executed by Python, in JSON form
  (tuples and ranges as lists).  They are self-contained Python files, so executing them is what mmcv's
  Config.fromfile does for them.

tests/test_dense_eval_cpu.py checks evaluate_dense_tasks.py and dvt.dense_eval.load_config against them.

Run in the build container (needs /root/reference):  python tests/golden/make_dense_eval_golden.py"""
import json
import os
import runpy
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_cli_golden import flags  # noqa: E402

REF = "/root/reference"
CONFIGS = ("vitb_voc2012_linear_config.py", "vitb_ade20k_linear_config.py")


def jsonable(v):
    if isinstance(v, dict):
        return {k: jsonable(x) for k, x in v.items()}
    if isinstance(v, (list, tuple, range)):
        return [jsonable(x) for x in v]
    return v


if __name__ == "__main__":
    gold = {"evaluate_dense_tasks.py": flags(os.path.join(REF, "evaluate_dense_tasks.py"))}
    with open(os.path.join(HERE, "cli_flags_dense_eval.json"), "w") as fh:
        json.dump(gold, fh, indent=1, sort_keys=True)
    cfgs = {}
    for name in CONFIGS:
        ns = runpy.run_path(os.path.join(REF, "evaluation", "configs", name))
        cfgs[name] = jsonable({k: v for k, v in ns.items() if not k.startswith("__")})
    with open(os.path.join(HERE, "dense_eval_configs.json"), "w") as fh:
        json.dump(cfgs, fh, indent=1, sort_keys=True)
    print({k: len(v) for k, v in gold.items()}, {k: len(v) for k, v in cfgs.items()})
