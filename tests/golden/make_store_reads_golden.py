"""Writes tests/golden/store_reference_reads.json: the files the REFERENCE's stage-2 dataset
(dvt/dataset/paired_list_dataset.py:27-43, imported unmodified) opens for two list entries of a feature store, relative
to the store's root, and the image / array shapes it returns.  Run from the repository root with the reference checkout
given as the first argument:  python tests/golden/make_store_reads_golden.py <reference-root>"""
import importlib.util
import json
import os
import sys
import tempfile

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "store_reference_reads.json")


def main(ref_root):
    spec = importlib.util.spec_from_file_location("ref_paired", os.path.join(ref_root, "dvt/dataset/paired_list_dataset.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    from PIL import Image
    h, w, C = 3, 4, 16
    model = "vit_small_patch14_dinov2.lvd142m"
    rels = ["a/one.jpg", "b/two.png"]
    with tempfile.TemporaryDirectory() as tmp:
        data_root = os.path.join(tmp, "data") + "/"
        save_root = os.path.join(tmp, "feats")
        feat_root = f"{save_root}/denoised_features/{model}/"
        for k, rel in enumerate(rels):
            os.makedirs(os.path.dirname(os.path.join(data_root, rel)), exist_ok=True)
            Image.fromarray(np.full((8, 8, 3), 40 * k, np.uint8)).save(os.path.join(data_root, rel))
            for kind, shape in (("raw_features", (h, w, C)), ("denoised_features", (1, h, w, C))):
                p = os.path.join(save_root, kind, model, os.path.splitext(rel)[0] + ".npy")
                os.makedirs(os.path.dirname(p), exist_ok=True)
                np.save(p, np.zeros(shape, np.float32))
        lst = os.path.join(tmp, "list.txt")
        with open(lst, "w") as f:
            f.write("".join(f"{r} 0\n" for r in rels))
        opened = []
        real_load = np.load
        ref.np.load = lambda p, *a, **k: (opened.append(os.path.relpath(p, save_root)), real_load(p, *a, **k))[1]
        ds = ref.PairedListDataset(data_root=data_root, data_list=lst, feat_root=feat_root, transform=lambda im: im.size)
        items = []
        for k, rel in enumerate(rels):
            opened.clear()
            it = ds[k]
            items.append({"entry": rel, "opened": list(opened), "image": list(it["image"]),
                          "original_shape": list(it["original_feats"].shape),
                          "denoised_shape": list(it["denoised_feats"].shape)})
        ref.np.load = real_load
    with open(OUT, "w") as f:
        json.dump({"model": model, "feature_shape": [h, w, C], "length": len(ds), "items": items}, f, indent=1)
    print("wrote", OUT)


if __name__ == "__main__":
    main(sys.argv[1])
