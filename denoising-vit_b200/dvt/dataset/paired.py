"""Stage-2 data: pairs (raw ViT feature map, per-image denoised map) produced by stage 1.

`FeatureStoreDataset` reads the `.npy` store (layout: dvt/store.py; reference reader dvt/dataset/paired_list_dataset.py:
9-43): one list line per image, `<feat_root>/<rel>.npy` holds the denoised map (1, h, w, C), the raw map sits beside it with
`denoised_features` -> `raw_features` in the path; an image whose files are missing is replaced by a random other one.
The denoiser trained by main_denoiser.py never looks at the pixels (`Denoiser(vit=None)`), so the image is only decoded
when `load_images=True` (the reference always decodes it, for its visualisation).

`InMemoryPairs` serves the same items from the tensors stage 1 gathered with its NCCL all-gather (`--collate_out`), i.e.
without the disk round trip.  The two samplers reproduce the reference's index streams (dvt/dataset/sampler.py:7-45)."""
from __future__ import annotations

import math
import os
from typing import Callable, Dict, Iterator, Optional

import numpy as np
import torch


class FeatureStoreDataset(torch.utils.data.Dataset):
    def __init__(self, data_root: str, data_list: str, feat_root: str, transform: Optional[Callable] = None,
                 load_images: bool = False):
        self.data_root, self.feat_root, self.transform, self.load_images = data_root, feat_root, transform, load_images
        with open(data_list) as fh:
            self.img_paths = [ln.strip().split(" ")[0] for ln in fh if ln.strip()]

    def __len__(self) -> int:
        return len(self.img_paths)

    def paths(self, index: int):
        rel = self.img_paths[index]
        den = os.path.join(self.feat_root, os.path.splitext(rel)[0] + ".npy")
        return rel, den, den.replace("denoised_features", "raw_features")

    def __getitem__(self, index: int) -> Dict[str, object]:
        for _ in range(1000):
            rel, den, raw = self.paths(index)
            if os.path.exists(den):
                break
            index = int(np.random.randint(len(self.img_paths)))     # stage 1 has not (yet) produced this image
        else:
            raise FileNotFoundError(f"no denoised feature file found under {self.feat_root}")
        item = {"original_feats": np.load(raw).squeeze(), "denoised_feats": np.load(den).squeeze()}
        if self.load_images:
            from torchvision.datasets.folder import default_loader
            img = default_loader(os.path.join(self.data_root, rel))
            item["image"] = self.transform(img) if self.transform is not None else img
        return item


class InMemoryPairs(torch.utils.data.Dataset):
    """Items straight from the stacks stage 1 collated on every rank: raw [n, h, w, C] and denoised [n, h, w, C]."""

    def __init__(self, raw: torch.Tensor, denoised: torch.Tensor):
        assert raw.shape == denoised.shape and raw.dim() == 4
        self.raw, self.denoised = raw, denoised

    def __len__(self) -> int:
        return self.raw.shape[0]

    def __getitem__(self, index: int):
        return {"original_feats": self.raw[index], "denoised_feats": self.denoised[index]}


class InfiniteSampler(torch.utils.data.Sampler):
    """0, 1, ..., n-1, 0, 1, ... for ever (single-process training).  `start` is the number of indices already consumed
    (a resumed run): the stream is entered at that position, without walking through the consumed part."""

    def __init__(self, data_source, start: int = 0):
        self.n, self.start = len(data_source), int(start)

    def __iter__(self) -> Iterator[int]:
        i = self.start % self.n
        while True:
            yield i
            i = (i + 1) % self.n


class DistributedInfiniteSampler(torch.utils.data.Sampler):
    """Rank r owns the indices r, r + world, ...; it shuffles them once (numpy default_rng seeded with the epoch) and then
    cycles through that order for ever.  `start` is the number of indices this rank has already consumed: the same
    shuffled order is entered at `start` modulo the length of the rank's shard (which is `num_samples`, or one less on
    the trailing ranks when world does not divide n)."""

    def __init__(self, data_source, num_replicas: int, rank: int, start: int = 0):
        self.n, self.num_replicas, self.rank, self.epoch = len(data_source), num_replicas, rank, 0
        self.num_samples = math.ceil(self.n / num_replicas)
        self.start = int(start)

    def set_epoch(self, epoch: int):
        self.epoch = epoch

    def __len__(self) -> int:
        return self.num_samples

    def __iter__(self) -> Iterator[int]:
        rng = np.random.default_rng(self.epoch)
        shards = [list(range(self.n))[i::self.num_replicas] for i in range(self.num_replicas)]
        mine = shards[self.rank]
        rng.shuffle(mine)
        if mine:
            yield from mine[self.start % len(mine):]
        while True:
            yield from mine
