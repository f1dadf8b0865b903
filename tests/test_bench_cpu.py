"""bench.py contract on the CPU: the reference arm (`--impl reference`) prints ONE JSON line with the keys the driver reads,
the same `config` as the H100 arm, and ranks other than 0 exit without work.  (The H100 arm needs a GPU.)"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(extra_env=None, *flags):
    env = dict(os.environ, **(extra_env or {}))
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", *flags],
                          capture_output=True, text=True, env=env, timeout=900, cwd=ROOT)


def test_reference_arm_prints_the_contract_line():
    r = _run(None, "--steps", "1", "--warmup", "0")
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "impl", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["unit"] == "images/s" and d["higher_is_better"] is True
    assert d["vs_baseline"] is None and d["n_gpus"] == 1 and d["steps"] == 1
    assert d["config"]["workload"] == "stage1_vitb14_518_768views_2000iters" and d["config"]["views_per_image"] == 769
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["sample"]
    assert d["cpu_baseline"]["value"] == d["value"] == d["e2e"]["value"] and d["value"] > 0
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert abs(d["ms_per_step"] * d["value"] - 1000.0) < 1e-6

    # the config both arms print is one function of the flags: the GPU arm's line (tests/golden) carries the same dict
    with open(os.path.join(ROOT, "tests", "golden", "bench_gpu_line.json")) as fh:
        ours = json.load(fh)
    same = {k: v for k, v in ours["config"].items() if k != "images_per_gpu"}
    assert same == {k: v for k, v in d["config"].items() if k != "images_per_gpu"}
    assert ours["metric"] == d["metric"] and ours["unit"] == d["unit"]


def test_reference_arm_other_ranks_do_no_work():
    r = _run({"RANK": "1", "WORLD_SIZE": "2", "LOCAL_RANK": "1"}, "--gpus", "2", "--steps", "1", "--warmup", "0")
    assert r.returncode == 0 and r.stdout.strip() == ""
