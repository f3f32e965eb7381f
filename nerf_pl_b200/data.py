"""Device-resident training batches: the reference's ``DataLoader(train_dataset, shuffle=True, num_workers=4,
batch_size=1024, pin_memory=True)`` (train.py:89-94) without the host.  The rays and colours live on the GPU; every
epoch draws one permutation there and each batch is one gather.  ``DeviceViewBatches`` keeps the views (uint8
images and poses) instead and makes each batch's rays and colours on the device.

The host-side arithmetic (how many batches an epoch has, which indices a rank gets) is kept in plain functions so it
can be checked without a GPU; ``CapturedTrainStep`` (training.py) shares it.
"""
from __future__ import annotations

from typing import Dict, Iterator, Optional, Tuple

import torch

from . import _lib

__all__ = ["DeviceRayBatches", "DeviceViewBatches", "num_batches", "shard_size", "shard_indices", "epoch_position",
           "next_step_schedule", "default_seed"]


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


def _cuda_device(device, like: torch.Tensor, who: str) -> torch.device:
    if device is None:
        device = like.device if like.is_cuda else torch.device("cuda", torch.cuda.current_device())
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError(f"{who} keeps the dataset on a CUDA device (no CPU fallback)")
    return device


class _EpochBatches:
    """What every device-resident batch source shares: ``n_rays`` samples, shuffled per epoch on the device from
    this object's own generator, sharded over DDP ranks, cut into ``batch_size`` batches; ``gather(idx)`` (the
    subclass's) turns one batch of sample indices into ``{'rays', 'rgbs'}``.  ``CapturedTrainStep`` accepts any
    subclass."""

    def __init__(self, n_rays: int, batch_size: int, shuffle: bool, drop_last: bool, seed: Optional[int],
                 rank: Optional[int], world_size: Optional[int], device: torch.device):
        if rank is None or world_size is None:
            r, w = _dist_rank_world()
            rank = r if rank is None else rank
            world_size = w if world_size is None else world_size
        if not 0 <= rank < world_size:
            raise ValueError(f"rank {rank} outside world_size {world_size}")
        self._n_rays = int(n_rays)
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
        return self._n_rays

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
        raise NotImplementedError

    def __iter__(self) -> Iterator[Dict[str, torch.Tensor]]:
        perm = self.next_permutation()
        B = self.batch_size
        for i in range(len(self)):
            yield self.gather(perm[i * B:(i + 1) * B])


class DeviceRayBatches(_EpochBatches):
    """Shuffled ``{'rays': (B, 8), 'rgbs': (B, 3)}`` batches drawn on the GPU, the keys ``NeRFSystem.decode_batch``
    reads.  A drop-in for the training ``DataLoader``: ``iter()`` runs one epoch, ``len()`` is its number of
    batches (``drop_last`` as ``DataLoader`` defines it).

    ``rays`` (N, 8) and ``rgbs`` (N, 3), e.g. ``train_dataset.all_rays`` / ``all_rgbs``, are copied to the device
    once as float32: 44 B per ray, so a 100-view 800x800 Blender set holds 2.8 GB of device memory
    (``DeviceViewBatches`` holds the views instead: 4 B per pixel).  Every epoch
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
        device = _cuda_device(device, rays, "DeviceRayBatches")
        super().__init__(rays.shape[0], batch_size, shuffle, drop_last, seed, rank, world_size, device)
        self.rays = rays.detach().to(device=device, dtype=torch.float32).contiguous()
        self.rgbs = rgbs.detach().to(device=device, dtype=torch.float32).contiguous()

    def gather(self, idx: torch.Tensor) -> Dict[str, torch.Tensor]:
        return {"rays": self.rays.index_select(0, idx), "rgbs": self.rgbs.index_select(0, idx)}


class DeviceViewBatches(_EpochBatches):
    """``DeviceRayBatches`` that keeps the views instead of the rays: the uint8 images and one pose per view live on
    the GPU (3 or 4 B per pixel plus 48 B per view), and every batch's rays and colours are made there, in one
    launch, from the pixel ids the epoch permutation selects.

    ``images``: (V, H, W, 3) RGB or (V, H, W, 4) RGBA uint8 (``read_llff_views`` / ``read_blender_views``);
    ``c2w``: (V, 3, 4) poses (cast to float32, as the reference's ``torch.FloatTensor(pose)``); ``focal``, ``near``,
    ``far``, ``ndc``: as ``generate_rays`` takes them.  Sample ``p`` is pixel ``(j, i)`` of view ``v`` with
    ``p = (v * H + j) * W + i``, the order in which the reference concatenates ``all_rays`` / ``all_rgbs``, and its
    ray and colour are bit for bit what ``generate_rays`` gives for that view and what ``T.ToTensor()`` (and, for
    RGBA, blender.py:58's ``rgb * a + (1 - a)``) gives for that pixel.  So with the same ``seed`` this object yields
    the batches a ``DeviceRayBatches`` built from those rays and colours yields; the epoch permutation, ``len()``,
    seeding and DDP sharding are the same code.  ``view(v)`` returns one whole view for validation and testing."""

    def __init__(self, images, c2w, focal: float, near: float, far: float, ndc: bool = False, batch_size: int = 1024,
                 shuffle: bool = True, drop_last: bool = False, seed: Optional[int] = None, rank: Optional[int] = None,
                 world_size: Optional[int] = None, device: Optional[torch.device] = None):
        images = torch.as_tensor(images)
        c2w = torch.as_tensor(c2w)
        if images.dtype != torch.uint8 or images.dim() != 4 or images.shape[3] not in (3, 4):
            raise ValueError("images must be uint8 of shape (V, H, W, 3) or (V, H, W, 4)")
        V, H, W, C = images.shape
        if c2w.shape != (V, 3, 4):
            raise ValueError(f"c2w must be ({V}, 3, 4), one pose per view")
        if V * H * W == 0 or batch_size <= 0:
            raise ValueError("an empty dataset or a batch size < 1")
        if H >= 2 ** 31 or W >= 2 ** 31:
            raise ValueError("H and W must be < 2**31")
        if not float(focal) > 0:
            raise ValueError("focal must be > 0")
        device = _cuda_device(device, images, "DeviceViewBatches")
        super().__init__(V * H * W, batch_size, shuffle, drop_last, seed, rank, world_size, device)
        self.images = images.detach().to(device=device).contiguous()
        self.c2w = c2w.detach().to(device=device, dtype=torch.float32).contiguous()
        self.shape = (int(V), int(H), int(W), int(C))
        self.focal, self.near, self.far, self.ndc = float(focal), float(near), float(far), bool(ndc)

    def gather(self, idx: torch.Tensor) -> Dict[str, torch.Tensor]:
        """The rays and colours of the pixel ids ``idx`` (int64, on this object's device): one launch."""
        idx = idx.to(torch.int64).contiguous()
        n = idx.shape[0]
        rays = torch.empty(n, 8, dtype=torch.float32, device=self.device)
        rgbs = torch.empty(n, 3, dtype=torch.float32, device=self.device)
        V, H, W, C = self.shape
        _lib.call("nerfb200_view_batch", self.device, self.images.data_ptr(), V, H, W, C, self.c2w.data_ptr(),
                  self.focal, self.near, self.far, int(self.ndc), idx.data_ptr(), n, rays.data_ptr(), rgbs.data_ptr())
        return {"rays": rays, "rgbs": rgbs}

    def view(self, v: int) -> Dict[str, torch.Tensor]:
        """View ``v`` whole, as the reference's val / test ``__getitem__`` gives it (blender.py:88-108,
        llff.py:259-292): ``rays`` (H W, 8), ``rgbs`` (H W, 3) and, for RGBA, ``valid_mask`` (H W,) = alpha > 0."""
        V, H, W, C = self.shape
        if not 0 <= v < V:
            raise IndexError(f"view {v} outside [0, {V})")
        out = self.gather(torch.arange(v * H * W, (v + 1) * H * W, device=self.device))
        if C == 4:
            out["valid_mask"] = (self.images[v, ..., 3] > 0).reshape(-1)
        return out
