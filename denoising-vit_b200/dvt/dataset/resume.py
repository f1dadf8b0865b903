"""Resuming the torch random streams of a DataLoader, so that a run resumed at batch k draws the random numbers of batches
k, k+1, ... that an uninterrupted run draws (stage 3: `RandomHorizontalFlip`, one `torch.rand(1)` per sample).

How a DataLoader draws, in torch's `_BaseDataLoaderIter` / `_worker_loop`:
- `iter(loader)` takes `base_seed` from the main process's default generator.  A resumed run reaches that call in the
  same generator state as the uninterrupted one when the same seed and code path precede it (the checkpoint load draws
  nothing), so it gets the same `base_seed`.
- Worker w seeds its torch generator with `base_seed + w`, and the workers take the batches in turn: batch j of an
  iterator goes to worker j mod W.  In the resumed iterator, worker w therefore takes the batches that worker
  (k + w) mod W took in the uninterrupted run, and `worker_init_fn` reseeds it as that worker and skips the draws that
  worker made for its batches before k.
- With no workers the samples are drawn in the main process, right after `iter(loader)`: its generator is advanced by
  the draws of the first k batches.

Only torch's generator is replayed (Python's `random` and numpy's are seeded by the DataLoader but not advanced).  The
number of draws to skip is computed, not counted; they are then made in chunks of 4 M (a few ms per million on a CPU)."""
from __future__ import annotations

import torch

_CHUNK = 1 << 22


def skip_torch_draws(n: int) -> None:
    """Advance the default torch generator by n `torch.rand(1)` draws (`torch.rand(m)` consumes what m of them do)."""
    while n > 0:
        m = min(n, _CHUNK)
        torch.rand(m)
        n -= m


class SkipWorkerDraws:
    """`worker_init_fn` of a DataLoader resumed at batch `start_batch`: worker w becomes worker (start_batch + w) mod W of
    the uninterrupted loader, advanced past the `draws_per_batch` draws of each of its batches before `start_batch`."""

    def __init__(self, start_batch: int, draws_per_batch: int, num_workers: int):
        self.start_batch, self.draws_per_batch, self.num_workers = start_batch, draws_per_batch, num_workers

    def __call__(self, worker_id: int) -> None:
        info = torch.utils.data.get_worker_info()
        assert info.num_workers == self.num_workers and info.id == worker_id
        orig = (self.start_batch + worker_id) % self.num_workers
        torch.manual_seed(info.seed - worker_id + orig)        # info.seed is base_seed + worker_id
        done = (self.start_batch - orig + self.num_workers - 1) // self.num_workers   # its batches before start_batch
        skip_torch_draws(done * self.draws_per_batch)


def resumed_iter(loader: torch.utils.data.DataLoader, start_batch: int):
    """`iter(loader)` for a run resumed at batch `start_batch` whose dataset makes one torch draw per sample; the loader's
    sampler must already start at sample `start_batch * batch_size`.  At `start_batch` 0 this is `iter(loader)`.  With
    workers, it installs `SkipWorkerDraws` as the loader's `worker_init_fn`."""
    if start_batch == 0:
        return iter(loader)
    if loader.num_workers == 0:
        it = iter(loader)              # draws base_seed first, as the uninterrupted run did
        skip_torch_draws(start_batch * loader.batch_size)
        return it
    assert loader.worker_init_fn is None, "resumed_iter installs its own worker_init_fn"
    loader.worker_init_fn = SkipWorkerDraws(start_batch, loader.batch_size, loader.num_workers)
    return iter(loader)
