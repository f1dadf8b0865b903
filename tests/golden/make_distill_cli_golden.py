"""Generates tests/golden/cli_flags_distillation.json: every `add_argument` of the reference's stage-3 CLI
(/root/reference/main_distillation.py:26-80) with its `type`, `default`, `action`, `nargs` and `choices` expressions, read
from the source with `ast` by `make_cli_golden.flags` (the module itself imports imageio / timm and cannot be executed
here).  tests/test_distill_cpu.py checks that main_distillation.py accepts the same flags.

Run in the build container (needs /root/reference):  python tests/golden/make_distill_cli_golden.py"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_cli_golden import flags  # noqa: E402

if __name__ == "__main__":
    gold = {"main_distillation.py": flags("/root/reference/main_distillation.py")}
    with open(os.path.join(HERE, "cli_flags_distillation.json"), "w") as fh:
        json.dump(gold, fh, indent=1, sort_keys=True)
    print({k: len(v) for k, v in gold.items()})
