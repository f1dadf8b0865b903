"""Resuming stages 2 and 3 without a GPU: the samplers entered at a start position yield the unstarted stream from that
position on (arithmetically, also at 10^8), and a DataLoader resumed at batch k with `dvt.dataset.resumed_iter` flips
exactly the samples that the uninterrupted loader flips in batches k, k+1, ... (no workers, and two workers)."""
import itertools
import time

import numpy as np
import pytest
import torch
import torchvision.transforms as transforms
from PIL import Image


def _take(sampler, k):
    return list(itertools.islice(iter(sampler), k))


@pytest.mark.parametrize("n", [7, 10])
@pytest.mark.parametrize("world", [1, 2, 3])
def test_started_sampler_continues_the_stream(n, world):
    from dvt import dataset
    K = 25
    starts = [0, 1, 2, n // world - 1, n // world, n // world + 1, n - 1, n, n + 3, 2 * n + 5, 7 * n + 2]
    for rank in range(world):
        full = _take(dataset.DistributedInfiniteSampler(range(n), num_replicas=world, rank=rank), max(starts) + K)
        for s in starts:
            got = _take(dataset.DistributedInfiniteSampler(range(n), num_replicas=world, rank=rank, start=s), K)
            assert got == full[s:s + K], (n, world, rank, s)
    if world == 1:
        full = _take(dataset.InfiniteSampler(range(n)), max(starts) + K)
        for s in starts:
            assert _take(dataset.InfiniteSampler(range(n), start=s), K) == full[s:s + K], (n, s)


def test_started_sampler_is_immediate_far_into_the_stream():
    from dvt import dataset
    n, pos = 1000, 10 ** 8
    cycles = {}
    for world, rank in ((1, 0), (3, 0), (3, 2)):
        cycle = _take(dataset.DistributedInfiniteSampler(range(n), num_replicas=world, rank=rank), len(range(rank, n, world)))
        cycles[(world, rank)] = cycle
    t0 = time.perf_counter()
    got_inf = _take(dataset.InfiniteSampler(range(n), start=pos), 5)
    got = {k: _take(dataset.DistributedInfiniteSampler(range(n), num_replicas=k[0], rank=k[1], start=pos), 5)
           for k in cycles}
    assert time.perf_counter() - t0 < 0.5
    assert got_inf == [(pos + i) % n for i in range(5)]
    for k, cycle in cycles.items():
        assert got[k] == [cycle[(pos + i) % len(cycle)] for i in range(5)], k


def test_horizontal_flip_draws_one_rand_per_sample():
    """The replay of the stage-3 flip stream assumes that the installed torchvision's RandomHorizontalFlip makes exactly
    one torch.rand(1) draw per sample, and that the rest of main_distillation.py's transform draws nothing."""
    img = Image.fromarray(np.random.RandomState(0).randint(0, 255, (20, 24, 3), dtype=np.uint8))
    tf = transforms.Compose([transforms.Resize([14, 14], interpolation=Image.BICUBIC, antialias=True),
                             transforms.RandomHorizontalFlip(), transforms.ToTensor(),
                             transforms.Normalize((0.5, 0.5, 0.5), (0.2, 0.2, 0.2))])
    for m in (1, 2, 9):
        torch.manual_seed(3)
        for _ in range(m):
            tf(img)
        after = torch.rand(4)
        torch.manual_seed(3)
        torch.rand(m)
        assert torch.equal(torch.rand(4), after), m


def test_skip_torch_draws_equals_single_draws():
    from dvt.dataset import resume
    for n in (0, 1, 5, 300):
        torch.manual_seed(11)
        for _ in range(n):
            torch.rand(1)
        a = torch.rand(3)
        torch.manual_seed(11)
        resume.skip_torch_draws(n)
        assert torch.equal(torch.rand(3), a), n
    n = resume._CHUNK + 7                                   # across a chunk boundary
    torch.manual_seed(12)
    torch.rand(n)
    a = torch.rand(3)
    torch.manual_seed(12)
    resume.skip_torch_draws(n)
    assert torch.equal(torch.rand(3), a)


@pytest.fixture(scope="module")
def flip_folder(tmp_path_factory):
    """An ImageFolder of 7 tiny images: left half bright, right half dark, the index in the green channel; after the
    transform a sample tells which image it is and whether it was flipped."""
    root = tmp_path_factory.mktemp("flips")
    for i in range(7):
        d = root / f"class{i % 2}"
        d.mkdir(exist_ok=True)
        a = np.zeros((4, 6, 3), dtype=np.uint8)
        a[:, :3, 0] = 255
        a[:, :, 1] = 20 * i
        Image.fromarray(a).save(d / f"{i}.png")
    return str(root)


def _loader(root, start_batch, batch, workers):
    from torchvision.datasets import ImageFolder
    from dvt import dataset
    ds = ImageFolder(root, transform=transforms.Compose([transforms.RandomHorizontalFlip(), transforms.ToTensor()]))
    sampler = dataset.InfiniteSampler(ds, start=start_batch * batch)
    return torch.utils.data.DataLoader(ds, batch_size=batch, sampler=sampler, num_workers=workers)


def _decode(batch):
    x = batch[0]
    ident = torch.round(x[:, 1, 0, 0] * 255 / 20).long().tolist()
    flipped = (x[:, 0, 0, 0] < 0.5).tolist()
    return list(zip(ident, flipped))


@pytest.mark.parametrize("workers", [0, 2])
@pytest.mark.parametrize("start_batch", [1, 2, 5])
def test_resumed_loader_flips_like_the_uninterrupted_one(flip_folder, workers, start_batch):
    from dvt import dataset
    batch, K = 3, 6
    torch.manual_seed(0)
    it = iter(_loader(flip_folder, 0, batch, workers))
    full = [_decode(next(it)) for _ in range(start_batch + K)]
    del it
    assert any(f for b in full for _, f in b) and not all(f for b in full for _, f in b)
    torch.manual_seed(0)
    it = dataset.resumed_iter(_loader(flip_folder, start_batch, batch, workers), start_batch)
    assert [_decode(next(it)) for _ in range(K)] == full[start_batch:]
    del it
    # without the replay the resumed loader visits the same images but flips others
    torch.manual_seed(0)
    it = iter(_loader(flip_folder, start_batch, batch, workers))
    naive = [_decode(next(it)) for _ in range(K)]
    assert [[i for i, _ in b] for b in naive] == [[i for i, _ in b] for b in full[start_batch:]]
    assert naive != full[start_batch:]
