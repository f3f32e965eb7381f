"""Baked volumes: rgb and sigma on a lattice, stored in sparse bricks and rendered without the MLP (DESIGN.md §10j).

extract_mesh.ipynb bakes ``[sigmoid rgb, raw sigma]`` on an N^3 lattice with the view direction 0 and the Unity
project ray-marches that volume.  ``bake_volume`` makes the same lattice on the device through an occupancy grid,
keeping only the 8^3-point bricks of the sparse marching cubes' plan (§10i); ``render_baked`` renders rays from it
in one launch (csrc/baked_kernels.cuh), and ``to_dense`` gives back ``rgb_sigma_grid(..., occupancy=)`` bit for bit,
so ``pack_volume`` / ``write_vol`` write the Unity file from a bake.

``bake_volume(..., view_dependent=True)`` bakes the view-dependent kind instead (DESIGN.md §10k): per point raw sigma
and the degree-2 spherical-harmonic coefficients of the colour, fitted over 64 fixed directions in the MLP's epilogue
(``query_rgb_sh``); ``render_baked`` evaluates them at each ray's direction.
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional

import torch

from . import _lib
from .culling import OccupancyGrid
from .mesh import _check_occupancy, _cuda, _device_of
from .nerf import packed_weights

BAKED_MAX_N = 2048
DENSE_MAX_N = 1625
SH_MAX_N = 1024             # bake, render, from_grid and to_dense of the view-dependent kind
SH_CHANNELS = 28


def _check_n(N, what: str, top: int = BAKED_MAX_N) -> int:
    N = int(N)
    if not 2 <= N <= top:
        raise ValueError(f"{what}: N = {N} outside [2, {top}]")
    return N


class BakedVolume:
    """[sigmoid rgb, raw sigma] on the N^3 lattice of ``rgb_sigma_grid`` over ``ranges``, stored per brick of 8^3
    points: ``data`` is one uint8 CUDA buffer of ``bricks`` bricks of 9^3 float4 points (the +1 apron copied from the
    neighbours) and the int32 map of the ceil(N / 8)^3 bricks (include/nerf_pl_b200_baked.h).  A point outside the
    stored bricks holds (0, 0, 0, 0).

    With ``view_dependent`` a point is the 28 floats of ``query_rgb_sh`` (7 float4: (c_r0, c_g0, c_b0, sigma), then
    the coefficients of m = 1..8; include/nerf_pl_b200_baked_sh.h), N <= 1024."""

    def __init__(self, data: torch.Tensor, N: int, x_range, y_range, z_range, bricks: int,
                 view_dependent: bool = False):
        self.view_dependent = bool(view_dependent)
        self.N = _check_n(N, "BakedVolume", SH_MAX_N if self.view_dependent else BAKED_MAX_N)
        self.ranges = tuple(_lib.ranges_host(x_range, y_range, z_range))
        self.bricks = int(bricks)
        nbytes = getattr(_lib.load(), self._api("bytes"))(self.N, self.bricks)
        if nbytes == 0:
            raise ValueError(f"BakedVolume: bricks = {bricks} outside [0, ceil(N / 8)^3]")
        if not isinstance(data, torch.Tensor) or not data.is_cuda:
            raise RuntimeError("BakedVolume: data must be a CUDA tensor (nerf_pl_b200 has no CPU fallback)")
        if data.dtype != torch.uint8 or data.numel() != nbytes:
            raise ValueError(f"BakedVolume: data must be {nbytes} bytes (uint8)")
        self.data = data.contiguous().reshape(-1)

    def _api(self, what: str) -> str:
        return ("nerfb200_baked_sh_" if self.view_dependent else "nerfb200_baked_") + what

    @property
    def channels(self) -> int:
        """Floats per point: 4, or 28 for the view-dependent kind."""
        return SH_CHANNELS if self.view_dependent else 4

    @property
    def device(self) -> torch.device:
        return self.data.device

    @property
    def nbytes(self) -> int:
        """Bytes of the stored volume: 11,664 per brick (81,648 for the view-dependent kind) plus 4 per brick of the
        map."""
        return self.data.numel()

    def _ranges_host(self):
        return (ctypes.c_double * 6)(*self.ranges)

    @classmethod
    @torch.no_grad()
    def from_grid(cls, rgbsigma: torch.Tensor, x_range, y_range, z_range) -> "BakedVolume":
        """The volume of a dense CUDA (N, N, N, 4) grid in ``rgb_sigma_grid``'s layout (raw sigma), or of an
        (N, N, N, 28) grid of ``query_rgb_sh`` points (the view-dependent kind, N <= 1024): the bricks whose 9^3
        points hold a sigma with ``max(sigma, 0)`` non-zero or non-finite are stored, each with the grid's values.
        Every other cell has alpha = 0, so this volume renders what a bake of the same grid renders.  N <= 1625."""
        g = _cuda(rgbsigma, "rgbsigma").detach().to(torch.float32).contiguous()
        if g.dim() != 4 or g.shape[3] not in (4, SH_CHANNELS) or not (g.shape[0] == g.shape[1] == g.shape[2]):
            raise ValueError("rgbsigma must be (N, N, N, 4) or (N, N, N, 28)")
        vd = g.shape[3] == SH_CHANNELS
        N = _check_n(g.shape[0], "BakedVolume.from_grid", SH_MAX_N if vd else DENSE_MAX_N)
        api = "nerfb200_baked_sh_" if vd else "nerfb200_baked_"
        lib = _lib.load()
        plan = _lib.workspace(lib.nerfb200_sparse_mc_plan_workspace_bytes(N), g.device)
        bricks = (ctypes.c_int64 * 1)()
        _lib.call(api + "from_grid_count", g.device, g.data_ptr(), N, plan.data_ptr(), plan.numel(), bricks)
        data = torch.empty(getattr(lib, api + "bytes")(N, bricks[0]), dtype=torch.uint8, device=g.device)
        _lib.call(api + "from_grid", g.device, g.data_ptr(), N, plan.data_ptr(), plan.numel(), bricks[0],
                  data.data_ptr(), data.numel())
        r = _lib.ranges_host(x_range, y_range, z_range)
        return cls(data, N, r[0:2], r[2:4], r[4:6], bricks[0], view_dependent=vd)

    @torch.no_grad()
    def to_dense(self) -> torch.Tensor:
        """(N, N, N, channels) fp32, 0 outside the stored bricks: ``rgb_sigma_grid``'s layout, N <= 1625, as for
        ``pack_volume``; or the 28 floats per point of the view-dependent kind, N <= 1024."""
        _check_n(self.N, "BakedVolume.to_dense", SH_MAX_N if self.view_dependent else DENSE_MAX_N)
        out = torch.empty(self.N, self.N, self.N, self.channels, dtype=torch.float32, device=self.device)
        _lib.call(self._api("to_dense"), self.device, self.data.data_ptr(), self.data.numel(), self.N, self.bricks,
                  out.data_ptr())
        return out

    def state_dict(self) -> Dict[str, object]:
        st = {"data": self.data.detach().cpu(), "N": self.N, "ranges": tuple(self.ranges), "bricks": self.bricks}
        if self.view_dependent:
            st["view_dependent"] = True
        return st

    @classmethod
    def from_state_dict(cls, state: Dict[str, object], device="cuda") -> "BakedVolume":
        """The volume of a ``state_dict()``, on ``device``."""
        r = tuple(state["ranges"])
        return cls(torch.as_tensor(state["data"]).to(device), state["N"], r[0:2], r[2:4], r[4:6], state["bricks"],
                   view_dependent=bool(state.get("view_dependent", False)))


@torch.no_grad()
def bake_volume(model: torch.nn.Module, N: int, x_range, y_range, z_range, *,
                occupancy: OccupancyGrid, view_dependent: bool = False) -> BakedVolume:
    """Bake ``model`` (direction 0) on the N^3 lattice of ``rgb_sigma_grid`` through ``occupancy``, N in [2, 2048]:
    the lattice points the grid evaluates (the rule of ``sigma_grid(..., occupancy=)``) go through the rgb + sigma
    query, one MLP pass each, and the bricks of the sparse marching cubes' plan that can hold a non-empty sample are
    stored.  ``bake_volume(...).to_dense()`` equals ``rgb_sigma_grid(..., occupancy=occupancy)`` bit for bit.  It
    synchronises (the plan's counts size the volume).

    ``view_dependent=True``: the same points and bricks go through ``query_rgb_sh`` instead, N in [2, 1024]; the
    sigma channel of ``to_dense()`` is the direction-0 bake's bit for bit."""
    dev = _device_of(model)
    occ = _check_occupancy(occupancy, dev)
    vd = bool(view_dependent)
    N = _check_n(N, "bake_volume", SH_MAX_N if vd else BAKED_MAX_N)
    api = "nerfb200_baked_sh_" if vd else "nerfb200_baked_"
    lib = _lib.load()
    ranges = _lib.ranges_host(x_range, y_range, z_range)
    occ_ranges = (ctypes.c_double * 6)(*occ.ranges)
    plan = _lib.workspace(lib.nerfb200_sparse_mc_plan_workspace_bytes(N), dev)
    bricks = (ctypes.c_int64 * 2)()
    _lib.call("nerfb200_sparse_mc_plan", dev, N, ranges, occ.bits.data_ptr(), occ.grid_n(), occ_ranges,
              plan.data_ptr(), plan.numel(), bricks)
    ws = _lib.workspace(getattr(lib, api + "workspace_bytes")(N, bricks[0], bricks[1]), dev)
    data = torch.empty(getattr(lib, api + "bytes")(N, bricks[1]), dtype=torch.uint8, device=dev)
    _lib.call(api + "bake", dev, packed_weights(model).data_ptr(), N, ranges, occ.bits.data_ptr(),
              occ.grid_n(), occ_ranges, plan.data_ptr(), plan.numel(), bricks, ws.data_ptr(), ws.numel(),
              data.data_ptr(), data.numel())
    return BakedVolume(data, N, ranges[0:2], ranges[2:4], ranges[4:6], bricks[1], view_dependent=vd)


def default_step(volume: BakedVolume) -> float:
    """One sample per cell: the smallest cell edge, ``min_a |max_a - min_a| / (N - 1)``."""
    r = volume.ranges
    return min(abs(r[2 * a + 1] - r[2 * a]) for a in range(3)) / (volume.N - 1)


@torch.no_grad()
def render_baked(volume: BakedVolume, rays: torch.Tensor, step: Optional[float] = None, white_back: bool = False,
                 early_stop: float = 0.0) -> Dict[str, torch.Tensor]:
    """Render the CUDA rays (n, 8) ``[o, d, near, far]`` through ``volume``: {"rgb": (n, 3), "depth": (n,),
    "opacity": (n,)} fp32 (DESIGN.md §10j).  Samples every ``step`` world units (default ``default_step``) from
    ``near``, trilinear rgb and ``max(sigma, 0)``, composited in sample order; ``early_stop = eps`` ends a ray after
    the first sample where its transmittance drops below eps.  One launch, no host synchronisation and no workspace,
    so it can be captured in a CUDA graph.  A view-dependent volume's colour is ``clamp(sum_m c_m Y_m(d / |d|), 0, 1)``
    of the trilinear coefficients at the ray's direction (DESIGN.md §10k)."""
    r = _cuda(rays, "rays")
    if r.dtype != torch.float32 or r.dim() != 2 or r.shape[1] != 8:
        raise ValueError("rays must be a float32 (n, 8) tensor [o, d, near, far]")
    if r.device != volume.device:
        raise RuntimeError(f"the rays are on {r.device}, the volume on {volume.device}")
    r = r.contiguous()
    s = default_step(volume) if step is None else float(step)
    n = r.shape[0]
    rgb = torch.empty(n, 3, dtype=torch.float32, device=r.device)
    depth = torch.empty(n, dtype=torch.float32, device=r.device)
    opacity = torch.empty(n, dtype=torch.float32, device=r.device)
    _lib.call(volume._api("render"), r.device, volume.data.data_ptr(), volume.data.numel(), volume.N,
              volume._ranges_host(), volume.bricks, r.data_ptr(), n, s, int(bool(white_back)), float(early_stop),
              rgb.data_ptr(), depth.data_ptr(), opacity.data_ptr())
    return {"rgb": rgb, "depth": depth, "opacity": opacity}
