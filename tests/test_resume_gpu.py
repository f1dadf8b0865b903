"""Resuming stages 2 and 3 bit for bit: under `--deterministic`, a run resumed from the checkpoint of step 3 ends with the
checkpoint of the uninterrupted 8-step run (weights, both AdamW moments and step `torch.equal`) and logs the same losses
for steps 4-7.  It depends on the sampler entering the sample stream at the resumed step and, in stage 3, on the replay
of the DataLoader workers' flip draws (dvt/dataset/resume.py); without them the resumed run trains on other samples."""
import os
import re
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


def _ckpt_equal(a, b):
    assert a.keys() == b.keys() and a["step"] == b["step"]
    model_key = "model" if "model" in a else "denoiser"
    assert a[model_key].keys() == b[model_key].keys()
    for k in a[model_key]:
        assert torch.equal(a[model_key][k], b[model_key][k]), k
    sa, sb = a["optimizer"]["state"], b["optimizer"]["state"]
    assert sa.keys() == sb.keys() and len(sa) > 0
    for i in sa:
        for k in ("exp_avg", "exp_avg_sq", "step"):
            assert torch.equal(sa[i][k], sb[i][k]), (i, k)


def _losses(out):
    """step -> the logged 'loss: .. l2_loss: .. cosine_similarity_loss: ..' (log_freq 1: one step per line)."""
    got = {}
    for ln in out.splitlines():
        m = re.match(r"Train \[\s*(\d+)/\d+\].*?(loss: .*) data_time:", ln)
        if m:
            got[int(m.group(1))] = m.group(2)
    return got


def _run_and_resume(M, argv, work, capsys):
    """An uninterrupted 8-step run 'a' (checkpoints at 0, 3, 6, 7), then run 'b' resumed from a's step-3 checkpoint."""
    M.main(M.get_args(argv + ["--run_name", "a"]))
    full = _losses(capsys.readouterr().out)
    a_dir = work / "denosing-vit" / "a" / "checkpoints"
    M.main(M.get_args(argv + ["--run_name", "b", "--resume", str(a_dir / "ckpt_000003.pth")]))
    out = capsys.readouterr().out
    assert "Resumed from" in out and "at step 4" in out
    resumed = _losses(out)
    assert sorted(full) == list(range(8)) and sorted(resumed) == [4, 5, 6, 7]
    assert {s: full[s] for s in resumed} == resumed
    b_dir = work / "denosing-vit" / "b" / "checkpoints"
    assert sorted(os.listdir(b_dir)) == ["ckpt_000006.pth", "ckpt_000007.pth", "latest.pth"]
    _ckpt_equal(torch.load(str(a_dir / "ckpt_000007.pth"), map_location="cpu"),
                torch.load(str(b_dir / "ckpt_000007.pth"), map_location="cpu"))


def test_stage2_resume_continues_the_uninterrupted_run(det, tmp_path, capsys):
    from argparse import Namespace
    sys.path.insert(0, ROOT)
    import main_denoiser as M
    from dvt.store import FeatureStoreWriter
    from dvt.utils import misc
    model = "vit_small_patch14_dinov2.lvd142m"
    h = w = 5
    data_root = str(tmp_path / "data") + "/"
    sargs = Namespace(data_root=data_root, save_root=str(tmp_path / "feats"), model=model)
    g = torch.Generator().manual_seed(0)
    wr = FeatureStoreWriter()
    rels = [f"img/{i}.jpg" for i in range(6)]            # 6 samples, batch 4: step 4 enters the stream at sample 16 % 6
    for rel in rels:
        clean = torch.randn(h, w, 384, generator=g)
        wr.submit(*misc.feature_paths(sargs, os.path.join(data_root, rel)), clean + 0.3 * torch.randn(h, w, 384, generator=g),
                  clean[None])
    wr.close()
    lst = tmp_path / "list.txt"
    lst.write_text("".join(f"{r} 0\n" for r in rels))
    argv = ["--model", model, "--input_size", "70", "--stride_size", "14", "--data_root", data_root, "--feat_root",
            f"{sargs.save_root}/denoised_features/{model}/", "--data_list_path", str(lst), "--batch_size", "4",
            "--num_iterations", "8", "--blr", "0.02", "--output_root", str(tmp_path / "work"), "--save_freq", "3",
            "--num_workers", "2", "--log_freq", "1", "--deterministic"]
    _run_and_resume(M, argv, tmp_path / "work", capsys)


@pytest.mark.parametrize("grad_ckpt", [False, True], ids=["plain", "grad-checkpointing"])
def test_stage3_resume_continues_the_uninterrupted_run(det, tmp_path, capsys, monkeypatch, grad_ckpt):
    from PIL import Image
    import dvt.models as DVT
    from dvt.models import vit_wrapper as VW
    sys.path.insert(0, ROOT)
    import main_distillation as M
    ident = "vit_small_patch14_reg4_dinov2.lvd142m"
    rs = np.random.RandomState(0)
    for i in range(10):                                  # 10 images, batch 4: step 4 enters the stream at 16 % 10
        d = tmp_path / "data" / f"class{i % 2}"
        d.mkdir(parents=True, exist_ok=True)
        Image.fromarray(rs.randint(0, 255, (70, 70, 3), dtype=np.uint8)).save(d / f"{i}.png")
    torch.manual_seed(0)
    vit = VW.B200VisionTransformer(ident, 14, VW.ARCHS[ident])
    wdir = tmp_path / "weights"
    wdir.mkdir()
    torch.save(vit.state_dict(), wdir / f"{ident}.pth")
    monkeypatch.setenv("DVT_WEIGHTS_DIR", str(wdir))
    den = DVT.Denoiser(9, 9, 384, vit=None, num_blocks=1)
    torch.save({"denoiser": den.state_dict(), "optimizer": {}, "step": 0}, tmp_path / "denoiser.pth")
    argv = ["--model", ident, "--denoiser_ckpt", str(tmp_path / "denoiser.pth"), "--input_size", "70", "--stride_size", "7",
            "--data_root", str(tmp_path / "data"), "--batch_size", "4", "--num_iterations", "8", "--blr", "0.002",
            "--output_root", str(tmp_path / "work"), "--save_freq", "3", "--num_workers", "2", "--log_freq", "1",
            "--deterministic"] + (["--grad_checkpointing"] if grad_ckpt else [])
    _run_and_resume(M, argv, tmp_path / "work", capsys)
