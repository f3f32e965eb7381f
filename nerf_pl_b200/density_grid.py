"""An occupancy grid kept current during training (DESIGN.md "Keeping the grid current during training").

``nb.occupancy_grid`` builds a grid once, from sigma at the N^3 lattice points.  ``DensityGrid`` keeps one up to
date instead: each cell holds a density that decays by ``decay`` at every ``update`` and is raised to sigma at one
jittered point of the cell (the scheme of Instant-NGP-style occupancy grids), and a cell is occupied while its
density is above ``sigma_threshold``.  ``grid`` is an ``OccupancyGrid`` over the same bits tensor, so every consumer
of a grid (``render_rays_culled``, ``skip="samples"``, ``render_rays_loss(occupancy=)``, ``CapturedTrainStep``)
takes it as is.  An update is a fixed sequence of sm_90a launches with no host synchronisation and no allocation
after the first call (csrc/density_kernels.cuh, include/nerf_pl_b200.h), so a CUDA graph can capture it;
``CapturedTrainStep(occupancy=grid, update_every=R)`` does.

A fresh or reset grid has density 0 and every cell occupied: it skips nothing until its first update.

``levels = L > 1`` keeps a cascade current (``OccupancyGrid``; DESIGN.md §10h): every level is updated as above on
its own box, for its non-inner cells only, with the jitter of level k drawn as element ``3 k + a``; inner cells
keep density 0 and bit 0.
"""
from __future__ import annotations

import ctypes
import math
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib
from .culling import OccupancyGrid, _check_levels, inner_cells
from .nerf import packed_weights


def _seed_word(seed: int) -> int:
    s = int(seed) & 0xFFFFFFFFFFFFFFFF
    return s - (1 << 64) if s >= 1 << 63 else s          # the same 64 bits as an int64


class DensityGrid:
    """A decaying density per cell of an ``N``-point grid over ``x_range x y_range x z_range`` and the occupancy bits
    it implies (``OccupancyGrid``'s conventions: ``M = N - 1`` cells per axis, x fastest).

    ``update(model)`` runs, for every cell c: three uniforms from the render kernel's Philox generator (key
    ``key``, ray c, stream 2), the point ``lo + (cell + u) * (hi - lo) / M`` in float64 rounded to float32, sigma of
    ``model`` there, ``density[c] = max(float32(decay * density[c]), max(sigma, 0))`` (NaN sigma counts as 0),
    occupied iff ``density[c] > sigma_threshold``, the set dilated by ``dilate`` cells and packed; then the key
    advances by one on the device.  ``seed=None`` takes ``torch.initial_seed()``.  ``chunk`` cells are evaluated
    per MLP launch; the results do not depend on it.  ``levels = L > 1``: a cascade (module docstring)."""

    def __init__(self, N: int, x_range, y_range, z_range, sigma_threshold: float = 1.0, decay: float = 0.95,
                 dilate: int = 1, seed: Optional[int] = None, device="cuda", chunk: int = 1 << 21, levels: int = 1):
        N = int(N)
        if not 2 <= N <= 1625:
            raise ValueError(f"DensityGrid: N = {N} outside [2, 1625]")
        levels = _check_levels(levels, "DensityGrid")
        thr = float(sigma_threshold)
        if math.isnan(thr):
            raise ValueError("DensityGrid: sigma_threshold is NaN")
        dec = float(np.float32(decay))
        if not 0.0 <= dec <= 1.0:
            raise ValueError(f"DensityGrid: decay = {decay} must be in [0, 1]")
        if int(dilate) != dilate or int(dilate) < 0:
            raise ValueError(f"DensityGrid: dilate = {dilate} must be an int >= 0")
        if int(chunk) != chunk or int(chunk) < 1:
            raise ValueError(f"DensityGrid: chunk = {chunk} must be an int >= 1")
        ranges = tuple(_lib.ranges_host(x_range, y_range, z_range))
        if not all(math.isfinite(v) for v in ranges) or any(ranges[2 * a] == ranges[2 * a + 1] for a in range(3)):
            raise ValueError("DensityGrid: every range needs finite min != max")
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("DensityGrid: the grid lives on a CUDA device (nerf_pl_b200 has no CPU fallback)")
        self.N, self.ranges, self.levels = N, ranges, levels
        self.sigma_threshold, self.decay, self.dilate, self.chunk = thr, dec, int(dilate), int(chunk)
        self.seed = torch.initial_seed() if seed is None else int(seed)
        M = N - 1
        self._density = torch.zeros(levels * M ** 3, dtype=torch.float32, device=device)
        bits = torch.empty(levels * ((M ** 3 + 31) // 32), dtype=torch.int32, device=device)
        self.grid = OccupancyGrid(bits, N, ranges[0:2], ranges[2:4], ranges[4:6], self.dilate, levels)
        self.key = torch.zeros((), dtype=torch.int64, device=device)
        self._ws = None
        self.reset()

    @property
    def device(self) -> torch.device:
        return self._density.device

    @property
    def bits(self) -> torch.Tensor:
        """The bit field, ``grid.bits`` itself."""
        return self.grid.bits

    @property
    def density(self) -> torch.Tensor:
        """(M, M, M) float32 view indexed ``[cx, cy, cz]``, as ``OccupancyGrid.to_dense``; (L, M, M, M) for a
        cascade."""
        M = self.N - 1
        d = self._density.view(self.levels, M, M, M).permute(0, 3, 2, 1)
        return d[0] if self.levels == 1 else d

    @torch.no_grad()
    def reset(self) -> None:
        """Density 0, every cell occupied (but the inner cells of a cascade), the key back to the seed."""
        M = self.N - 1
        occ = np.ones((self.levels, M, M, M), bool)            # [level, cz, cy, cx]: cell order
        for k in range(1, self.levels):
            a, b = inner_cells(self.N, k)
            occ[k, a:b, a:b, a:b] = False
        flat = occ.reshape(self.levels, -1)
        pad = np.zeros((self.levels, (-M ** 3) % 32), bool)    # the bits past the last cell are 0
        words = np.packbits(np.concatenate([flat, pad], 1), axis=1, bitorder="little").reshape(-1).view("<u4")
        self._density.zero_()
        self.bits.copy_(torch.from_numpy(words.view(np.int32).copy()))
        self.key.fill_(_seed_word(self.seed))

    def _workspace(self) -> torch.Tensor:
        if self._ws is None:
            nbytes = _lib.load().nerfb200_density_workspace_bytes(self.N, self.chunk)
            self._ws = _lib.workspace(nbytes, self.device)
            self._ranges_c = (ctypes.c_double * 6)(*self.ranges)
        return self._ws

    @torch.no_grad()
    def update(self, model: torch.nn.Module) -> None:
        """One update from ``model`` (the network that decides the picture: the fine one).  Stream-ordered, no
        synchronisation; after the first call it allocates nothing (the packed image is ``packed_weights``')."""
        packed = packed_weights(model)
        if packed.device != self.device:
            raise ValueError(f"the model is on {packed.device}, the density grid on {self.device}")
        ws = self._workspace()
        _lib.call("nerfb200_density_update", self.device, packed.data_ptr(), self.grid.grid_n(), self._ranges_c, self.sigma_threshold, self.decay, self.dilate, self.chunk, self.key.data_ptr(),
                  self._density.data_ptr(), self.bits.data_ptr(), ws.data_ptr(), ws.numel())

    @torch.no_grad()
    def points(self, start: int = 0, count: Optional[int] = None, level: int = 0) -> torch.Tensor:
        """(count, 3) float32: the points the next update evaluates for cells [start, start + count) (of a cascade
        level, its non-inner cells in cell order)."""
        level = int(level)
        if not 0 <= level < self.levels:
            raise ValueError(f"points: level = {level} outside [0, {self.levels})")
        cells = [(self.N - 1) ** 3 - (b - a) ** 3 for a, b in (inner_cells(self.N, k) for k in range(self.levels))]
        count = cells[level] - int(start) if count is None else int(count)
        if int(start) < 0 or count < 0 or int(start) + count > cells[level]:
            raise ValueError(f"points: cells [start, start + count) outside the grid (level {level} evaluates "
                             f"{cells[level]})")
        xyz = torch.empty(max(count, 0), 3, dtype=torch.float32, device=self.device)
        # the entry numbers the evaluated cells of all levels in turn
        _lib.call("nerfb200_density_points", self.device, self.grid.grid_n(), (ctypes.c_double * 6)(*self.ranges),
                  self.key.data_ptr(), sum(cells[:level]) + int(start), count, xyz.data_ptr())
        return xyz

    def state_dict(self) -> Dict[str, object]:
        """The grid's state; ``levels`` only for a cascade, so a one-level grid saves what it always saved."""
        st = {"density": self._density.detach().cpu(), "bits": self.bits.detach().cpu(),
              "key": int(self.key.item()), "seed": self.seed, "N": self.N, "ranges": tuple(self.ranges),
              "sigma_threshold": self.sigma_threshold, "decay": self.decay, "dilate": self.dilate,
              "chunk": self.chunk}
        if self.levels > 1:
            st["levels"] = self.levels
        return st

    @torch.no_grad()
    def load_state_dict(self, state: Dict[str, object]) -> "DensityGrid":
        """Restore a ``state_dict()`` of a grid of the same ``N``, ranges, threshold, decay and dilate into this
        grid's own tensors (so a graph that captured them keeps working)."""
        got = (int(state["N"]), tuple(float(v) for v in state["ranges"]), float(state["sigma_threshold"]),
               float(state["decay"]), int(state["dilate"]))
        have = (self.N, tuple(self.ranges), self.sigma_threshold, self.decay, self.dilate)
        if got != have:
            raise ValueError(f"load_state_dict: the state is of a grid with (N, ranges, sigma_threshold, decay, "
                             f"dilate) = {got}, this grid has {have}")
        if int(state.get("levels", 1)) != self.levels:
            raise ValueError(f"load_state_dict: the state is of a grid with {state.get('levels', 1)} levels, this "
                             f"grid has {self.levels}")
        self._density.copy_(torch.as_tensor(state["density"]).reshape(-1))
        self.bits.copy_(torch.as_tensor(state["bits"]).reshape(-1).view(torch.int32))
        self.key.fill_(int(state["key"]))
        self.seed = int(state.get("seed", self.seed))
        return self

    @classmethod
    def from_state_dict(cls, state: Dict[str, object], device="cuda") -> "DensityGrid":
        """The grid of a ``state_dict()`` saved beside a checkpoint, on ``device``; its next update is the one the
        saved grid would have made."""
        r = tuple(state["ranges"])
        g = cls(state["N"], r[0:2], r[2:4], r[4:6], state["sigma_threshold"], state["decay"], state["dilate"],
                seed=state.get("seed", 0), device=device, chunk=state.get("chunk", 1 << 21),
                levels=state.get("levels", 1))
        return g.load_state_dict(state)
