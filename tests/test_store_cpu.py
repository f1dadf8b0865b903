"""CPU: the host-side contract around the hot paths against goldens minted from the reference's own dvt/utils/misc.py
(tests/golden/make_store_golden.py): `.npy` feature-store paths / resume check (SURVEY 8(f-3)), the LR schedule (8a-4),
and the files the stage-1 driver writes (main_img_denoising.py:131-146: raw (h, w, C) and denoised (1, h, w, C), float32)."""
import json
import os
import sys
from argparse import Namespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "store_and_schedule.json")))


def test_feature_store_paths_match_reference():
    from dvt.utils import misc
    for c in GOLD["paths"]:
        args = Namespace(data_root=c["data_root"], save_root=c["save_root"], model=c["model"])
        assert misc.feature_paths(args, c["filename"]) == (c["raw"], c["denoised"])


def test_lr_schedule_matches_reference():
    from dvt.utils import misc
    from oracle import fit as OF
    for s in GOLD["schedules"]:
        a = Namespace(lr=s["lr"], min_lr=s["min_lr"], warmup_iters=s["warmup_iters"], num_iters=s["num_iters"])

        class Opt:
            param_groups = [{"lr": None}, {"lr": None, "lr_scale": 0.5}]
        for it, ref in zip(s["iterations"], s["values"]):
            o = Opt()
            got = misc.adjust_learning_rate(o, it, a)
            assert abs(got - ref) <= 1e-15 * max(1.0, abs(ref)) + 1e-18, (s, it, got, ref)
            assert o.param_groups[0]["lr"] == got and o.param_groups[1]["lr"] == got * 0.5
            assert abs(OF.lr_at(it, s["lr"], s["min_lr"], s["warmup_iters"], s["num_iters"]) - ref) <= 1e-15


def test_feature_store_writer_writes_the_reference_store(tmp_path):
    """`dvt.store.FeatureStoreWriter` (what the drop-in CLI hands every image's maps to): file locations, dtypes and shapes
    of the store (main_img_denoising.py:131-146), NPY v1, atomic rename, and the resume check that makes a second run skip
    the image."""
    from dvt.store import FeatureStoreWriter, load_pair
    from dvt.utils import misc
    h, w, C = 4, 5, 32
    data_root = str(tmp_path / "imgs")
    args = Namespace(data_root=data_root, save_root=str(tmp_path / "store"), model="vit_base_patch14_dinov2.lvd142m")
    img = os.path.join(data_root, "sub", "x.jpg")
    assert not misc.check_if_file_exists(args, img)
    raw_t = torch.arange(h * w * C, dtype=torch.float32).reshape(h, w, C)
    den_t = torch.ones(1, h, w, C)
    raw_p, den_p = misc.feature_paths(args, img)
    wr = FeatureStoreWriter(max_pending=2)
    for k in range(5):                                   # more submissions than staging slots: back-pressure, buffer reuse
        wr.submit(raw_p.replace("x.npy", f"x{k}.npy"), den_p.replace("x.npy", f"x{k}.npy"), raw_t + k, den_t * k)
    wr.submit(raw_p, den_p, raw_t, den_t)
    wr.close()
    assert len(wr.written) == 6
    # (the doubled slash is the reference's: data_root without a trailing slash is replaced by a directory with one)
    assert os.path.normpath(raw_p).endswith("store/raw_features/vit_base_patch14_dinov2.lvd142m/sub/x.npy")
    raw, den = np.load(raw_p), np.load(den_p)
    assert raw.dtype == np.float32 and raw.shape == (h, w, C) and np.array_equal(raw, raw_t.numpy())
    assert den.dtype == np.float32 and den.shape == (1, h, w, C)
    assert np.array_equal(np.load(raw_p.replace("x.npy", "x3.npy")), (raw_t + 3).numpy())
    with open(raw_p, "rb") as f:
        assert f.read(8) == bytes([0x93]) + b"NUMPY" + bytes([1, 0])          # NPY format version 1.0
    assert not [n for n in os.listdir(os.path.dirname(raw_p)) if ".tmp." in n]
    assert misc.check_if_file_exists(args, img)
    r2, d2 = load_pair(den_p)
    assert r2.shape == (h, w, C) and d2.shape == (h, w, C)
    bad = FeatureStoreWriter()
    bad.submit("/proc/definitely/not/writable/r.npy", "/proc/definitely/not/writable/d.npy", raw_t, den_t)
    try:
        bad.close()
        raise AssertionError("write error was swallowed")
    except RuntimeError as e:
        assert "feature store write failed" in str(e)


def test_store_reads_back_through_the_reference_dataset(tmp_path):
    """The store written here, read the way the REFERENCE's stage-2 dataset reads it (dvt/dataset/paired_list_dataset.py:27-43):
    tests/golden/store_reference_reads.json records, per list entry, the files that dataset opens relative to the store's
    root (denoised first, then raw) and the shapes it returns after np.load(...).squeeze()."""
    import json
    from dvt.store import FeatureStoreWriter
    from dvt.utils import misc
    with open(os.path.join(ROOT, "tests", "golden", "store_reference_reads.json")) as f:
        gold = json.load(f)
    h, w, C = gold["feature_shape"]
    data_root = str(tmp_path / "data") + "/"
    args = Namespace(data_root=data_root, save_root=str(tmp_path / "feats"), model=gold["model"])
    rels = [it["entry"] for it in gold["items"]]
    assert len(rels) == gold["length"] == 2
    wr = FeatureStoreWriter()
    maps = {}
    for k, rel in enumerate(rels):
        g = torch.Generator().manual_seed(k)
        maps[rel] = (torch.randn(h, w, C, generator=g), torch.randn(1, h, w, C, generator=g))
        wr.submit(*misc.feature_paths(args, os.path.join(data_root, rel)), *maps[rel])
    wr.close()
    for it in gold["items"]:
        den_rel, raw_rel = it["opened"]
        denoised = np.load(os.path.join(args.save_root, den_rel)).squeeze()
        original = np.load(os.path.join(args.save_root, raw_rel)).squeeze()
        assert list(original.shape) == it["original_shape"] and list(denoised.shape) == it["denoised_shape"]
        assert np.array_equal(original, maps[it["entry"]][0].numpy())
        assert np.array_equal(denoised, maps[it["entry"]][1][0].numpy())


def test_sampling_stream_is_the_references_rng_stream():
    """`draw_sampling_stream` (one int32 draw for all steps, plus the visualisation draw of every vis_freq-th image) leaves
    the global numpy RNG exactly where the reference's per-step int64 draws do (main_img_denoising.py:73,102)."""
    sys.path.insert(0, ROOT)
    import main_img_denoising as M
    args = Namespace(num_iters=7, pixel_bsz=16, vis_freq=2, num_views=5, num_vis_samples=3)
    n_rows = 6 * 37 * 37
    np.random.seed(11)
    got = [M.draw_sampling_stream(args, n_rows, i) for i in range(3)]
    tail = np.random.randint(0, 1 << 30, 4)
    np.random.seed(11)
    for i in range(3):
        ref = np.stack([np.random.randint(0, n_rows, args.pixel_bsz) for _ in range(args.num_iters)])
        if i % args.vis_freq == 0:
            np.random.randint(0, args.num_views + 1, args.num_vis_samples)
        assert got[i].dtype == np.int32 and np.array_equal(got[i], ref)
    assert np.array_equal(tail, np.random.randint(0, 1 << 30, 4))


def test_stage2_schedule_and_samplers_match_reference():
    """Stage-2 host logic against goldens minted from the reference's own CosineScheduler (dvt/utils/misc.py:211-241) and
    samplers (dvt/dataset/sampler.py:7-45): learning rate per iteration (incl. past the end), index streams per rank."""
    import itertools
    from dvt import dataset
    from dvt.utils import misc
    from oracle import train as OT
    for s in GOLD["stage2_schedules"]:
        kw = dict(base_value=s["base_value"], final_value=s["final_value"], total_iters=s["total_iters"],
                  warmup_iters=s["warmup_iters"], start_warmup_value=0)
        for it, ref in enumerate(s["values"]):
            assert abs(misc.cosine_schedule(it, **kw) - ref) <= 1e-18 + 1e-14 * abs(ref), (s["total_iters"], it)
        assert np.allclose(OT.cosine_schedule(**kw), s["values"][:s["total_iters"]], rtol=1e-14, atol=0)
    smp = GOLD["samplers"]
    assert list(itertools.islice(iter(dataset.InfiniteSampler(range(5))), 12)) == smp["infinite_n5_first12"]
    for world in (2, 3):
        for rank in range(world):
            d = dataset.DistributedInfiniteSampler(range(11), num_replicas=world, rank=rank)
            assert [int(i) for i in itertools.islice(iter(d), 14)] == smp[f"distributed_n11_w{world}_r{rank}_first14"]
            assert len(d) == smp[f"distributed_n11_w{world}_r{rank}_len"]


def test_feature_store_dataset_reads_pairs_and_skips_missing(tmp_path):
    from dvt.dataset import FeatureStoreDataset
    from dvt.store import FeatureStoreWriter
    from dvt.utils import misc
    h, w, C = 3, 4, 8
    data_root = str(tmp_path / "d") + "/"
    model = "vit_small_patch14_dinov2.lvd142m"
    args = Namespace(data_root=data_root, save_root=str(tmp_path / "f"), model=model)
    wr = FeatureStoreWriter()
    raw, den = torch.arange(h * w * C, dtype=torch.float32).reshape(h, w, C), torch.ones(1, h, w, C)
    wr.submit(*misc.feature_paths(args, data_root + "a/x.jpg"), raw, den)
    wr.close()
    lst = tmp_path / "l.txt"
    lst.write_text("a/x.jpg 3\na/missing.jpg 1\n")
    ds = FeatureStoreDataset(data_root, str(lst), f"{args.save_root}/denoised_features/{model}/")
    assert len(ds) == 2
    for i in range(2):                                   # the missing image falls back to an existing one
        item = ds[i]
        assert np.array_equal(item["original_feats"], raw.numpy()) and item["denoised_feats"].shape == (h, w, C)
        assert "image" not in item


def test_cli_flags_match_the_reference():
    """Drop-in boundary (SURVEY 8(b)): both stage CLIs accept every flag of the reference's parsers with the same type,
    default, action, nargs and choices (golden: tests/golden/make_cli_golden.py reads the reference sources with ast)."""
    import ast
    import json
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "tests", "golden"))
    try:
        from make_cli_golden import KEYS, flags
    finally:
        sys.path.pop(0)
    assert KEYS and ast
    with open(os.path.join(root, "tests", "golden", "cli_flags.json")) as fh:
        gold = json.load(fh)
    for cli, ref in gold.items():
        ours = flags(os.path.join(root, cli))
        assert len(ref) >= 20
        for name, spec in ref.items():
            assert name in ours, f"{cli}: flag {name} of the reference is missing"
            assert ours[name] == spec, f"{cli} {name}: {ours[name]} != reference {spec}"


def test_model_api_signatures_match_the_reference():
    """Drop-in boundary (SURVEY 8(b)): `dvt.models` mirrors the reference's classes -- same public methods, same positional
    parameters in the same order with the same defaults, same MODEL_LIST (extra keyword-only parameters are allowed)."""
    import json
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "tests", "golden"))
    try:
        from make_cli_golden import signatures
    finally:
        sys.path.pop(0)
    with open(os.path.join(root, "tests", "golden", "api_signatures.json")) as fh:
        gold = json.load(fh)
    n = 0
    for fname, ref in gold.items():
        ours = signatures(os.path.join(root, "denoising-vit_b200", "dvt", "models", fname))
        for name, spec in ref.items():
            assert name in ours, f"{fname}: {name} of the reference is missing"
            assert ours[name] == spec, f"{fname} {name}: {ours[name]} != reference {spec}"
            n += 1
    assert n >= 16
