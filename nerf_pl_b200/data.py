"""Device-resident training batches: the reference's ``DataLoader(train_dataset, shuffle=True, num_workers=4,
batch_size=1024, pin_memory=True)`` (train.py:89-94) without the host.  The rays and colours live on the GPU; every
epoch draws one permutation there and each batch is one gather.

The host-side arithmetic (how many batches an epoch has, which indices a rank gets) is kept in plain functions so it
can be checked without a GPU; ``CapturedTrainStep`` (training.py) shares it.
"""
from __future__ import annotations

from typing import Dict, Iterator, Optional, Tuple

import torch

__all__ = ["DeviceRayBatches", "num_batches", "shard_size", "shard_indices", "epoch_position", "next_step_schedule",
           "default_seed"]


def num_batches(n: int, batch_size: int, drop_last: bool) -> int:
    """``len(DataLoader)`` over ``n`` samples: full batches, plus a partial one unless ``drop_last``."""
    return n // batch_size if drop_last else (n + batch_size - 1) // batch_size


def shard_size(n: int, world_size: int) -> int:
    """Samples per rank under ``DistributedSampler(drop_last=False)``: the epoch is padded to a multiple of
    ``world_size`` by repeating its first indices, so every rank gets ceil(n / world_size)."""
    return (n + world_size - 1) // world_size


def shard_indices(perm: torch.Tensor, rank: int, world_size: int) -> torch.Tensor:
    """This rank's part of the epoch permutation ``perm`` (``DistributedSampler``'s semantics): pad ``perm`` to
    ``shard_size(n, world_size) * world_size`` with its own leading entries (repeated as often as needed), then take
    every ``world_size``-th entry from ``rank``.  The ranks' parts are disjoint apart from the padding, cover ``perm``
    and have equal length."""
    if not 0 <= rank < world_size:
        raise ValueError(f"rank {rank} outside world_size {world_size}")
    n = perm.shape[0]
    total = shard_size(n, world_size) * world_size
    if total > n:
        reps = (total - n + n - 1) // n
        perm = torch.cat([perm] + [perm] * reps)[:total]
    return perm[rank:total:world_size]


def epoch_position(step: int, batches_per_epoch: int) -> Tuple[int, int]:
    """(epoch, batch within the epoch) of the ``step``-th batch (0-based) of a run of full epochs."""
    if batches_per_epoch <= 0:
        raise ValueError("an epoch needs at least one batch")
    return divmod(step, batches_per_epoch)


def next_step_schedule(steps_done: int, batches_per_epoch: int) -> Tuple[bool, int, int]:
    """``CapturedTrainStep.step()``'s host-side schedule for the step that follows ``steps_done`` steps of full
    batches: (draw the next epoch's permutation first?, its epoch, its batch within the epoch).  The permutation of
    epoch 0 is drawn when the step is built, so a redraw happens exactly before the first step of every later
    epoch; the device offset of the step is ``batch * batch_size``."""
    epoch, batch = epoch_position(steps_done, batches_per_epoch)
    return batch == 0 and epoch > 0, epoch, batch


def default_seed(seed: Optional[int], world_size: int) -> int:
    """The seed of the epoch permutations.  Given: itself.  Under DDP (``world_size > 1``) every rank must draw the
    same permutation, and ``torch.initial_seed()`` differs between processes that were not seeded, so the default is
    0, as ``DistributedSampler``'s.  Single process: ``torch.initial_seed()`` (follows ``torch.manual_seed``)."""
    if seed is not None:
        return int(seed)
    return 0 if world_size > 1 else int(torch.initial_seed())


def _dist_rank_world() -> Tuple[int, int]:
    dist = torch.distributed
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


class DeviceRayBatches:
    """Shuffled ``{'rays': (B, 8), 'rgbs': (B, 3)}`` batches drawn on the GPU, the keys ``NeRFSystem.decode_batch``
    reads.  A drop-in for the training ``DataLoader``: ``iter()`` runs one epoch, ``len()`` is its number of
    batches (``drop_last`` as ``DataLoader`` defines it).

    ``rays`` (N, 8) and ``rgbs`` (N, 3), e.g. ``train_dataset.all_rays`` / ``all_rgbs``, are copied to the device
    once as float32: 44 B per ray, so a 100-view 800x800 Blender set holds 2.8 GB of device memory.  Every epoch
    draws a fresh permutation with ``torch.randperm`` on the device from this object's own generator, seeded with
    ``seed`` (default: ``default_seed``: ``torch.initial_seed()`` in one process, 0 under DDP), so the same seed
    repeats the same epochs.  The permutations have
    ``RandomSampler``'s distribution (uniform over all orders) but are not the ones the CPU ``DataLoader`` draws
    from the same seed.  ``shuffle=False`` yields the rays in order.

    Under DDP each rank takes its part of the same epoch permutation (``shard_indices``: ``DistributedSampler``'s
    semantics, padded to equal length); ``rank`` / ``world_size`` default to the initialised process group.  The
    ranks draw the same permutation as long as they pass the same ``seed`` or none (the DDP default is
    rank-independent, as ``DistributedSampler``'s).  The gather is a plain ``index_select`` (44 B per ray)."""

    def __init__(self, rays: torch.Tensor, rgbs: torch.Tensor, batch_size: int = 1024, shuffle: bool = True,
                 drop_last: bool = False, seed: Optional[int] = None, rank: Optional[int] = None,
                 world_size: Optional[int] = None, device: Optional[torch.device] = None):
        if rays.dim() != 2 or rays.shape[1] != 8 or rgbs.dim() != 2 or rgbs.shape[1] != 3 \
                or rays.shape[0] != rgbs.shape[0]:
            raise ValueError("rays must be (N, 8) and rgbs (N, 3)")
        if rays.shape[0] == 0 or batch_size <= 0:
            raise ValueError("an empty dataset or a batch size < 1")
        if device is None:
            device = rays.device if rays.is_cuda else torch.device("cuda", torch.cuda.current_device())
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("DeviceRayBatches keeps the dataset on a CUDA device (no CPU fallback)")
        if rank is None or world_size is None:
            r, w = _dist_rank_world()
            rank = r if rank is None else rank
            world_size = w if world_size is None else world_size
        if not 0 <= rank < world_size:
            raise ValueError(f"rank {rank} outside world_size {world_size}")
        self.rays = rays.detach().to(device=device, dtype=torch.float32).contiguous()
        self.rgbs = rgbs.detach().to(device=device, dtype=torch.float32).contiguous()
        self.batch_size = int(batch_size)
        self.shuffle = bool(shuffle)
        self.drop_last = bool(drop_last)
        self.rank, self.world_size = int(rank), int(world_size)
        self.device = device
        self.seed = default_seed(seed, self.world_size)
        self.generator = torch.Generator(device=device)
        self.generator.manual_seed(self.seed)
        self.epoch = 0              # epochs started so far

    @property
    def n_rays(self) -> int:
        return self.rays.shape[0]

    @property
    def samples_per_rank(self) -> int:
        return shard_size(self.n_rays, self.world_size)

    def __len__(self) -> int:
        return num_batches(self.samples_per_rank, self.batch_size, self.drop_last)

    def next_permutation(self) -> torch.Tensor:
        """This rank's indices of the next epoch, (samples_per_rank,) int64 on the device."""
        n = self.n_rays
        if self.shuffle:
            perm = torch.randperm(n, device=self.device, generator=self.generator)
        else:
            perm = torch.arange(n, device=self.device)
        self.epoch += 1
        if self.world_size == 1:
            return perm
        return shard_indices(perm, self.rank, self.world_size)

    def gather(self, idx: torch.Tensor) -> Dict[str, torch.Tensor]:
        return {"rays": self.rays.index_select(0, idx), "rgbs": self.rgbs.index_select(0, idx)}

    def __iter__(self) -> Iterator[Dict[str, torch.Tensor]]:
        perm = self.next_permutation()
        B = self.batch_size
        for i in range(len(self)):
            yield self.gather(perm[i * B:(i + 1) * B])
