"""Empty-space skipping at render time (DESIGN.md "Empty-space skipping").

``occupancy_grid`` turns a trained network into a bit field of occupied cells; ``cull_rays`` classifies rays
against it and compacts the live ones; ``render_rays_culled`` renders only those with the ordinary fused kernel and
scatters the results back over the value a ray through vacuum renders.  Every stage is an sm_90a kernel of
``libnerf_pl_b200.so`` (csrc/occupancy_kernels.cuh, include/nerf_pl_b200.h); the render kernel is not
touched.  The reference has no counterpart: it evaluates every sample of every ray.

``skip="samples"`` (``render_rays_culled``, ``batched_inference``, ``render_image``) goes one step further: inside a
live ray, a sample whose point lies in no occupied cell gets sigma = 0 and is not evaluated
(csrc/sample_skip_kernels.cuh, include/nerf_pl_b200.h; DESIGN.md "Skipping empty samples").  The evaluated
samples have the fused kernel's sigma and rgb bit for bit, and a ray with nothing to skip renders bit for bit as
``render_rays`` renders it; a ray with skipped samples is an approximation, like a culled ray.

What it guarantees.  A live ray is rendered by the same kernel on an ordinary ``(n_live, 8)`` tensor, and with
``perturb = noise_std = 0`` a ray's result does not depend on its row: live pixels are bit-identical to the
unculled render.  A culled pixel is *approximated* by the vacuum value.  The cell walk is exact and the dilation
adds a margin, but sigma is only sampled at the grid points and the trained sigma of empty space is small, not
zero: the error of a culled pixel is an empirical bound governed by ``N``, ``sigma_threshold`` and ``dilate``, not
a proof.  Space outside the grid's box counts as empty.  Culling is for inference only: training must see the
background rays to learn that they are empty.

``levels = L > 1`` makes the grid a cascade (DESIGN.md §10h): level 0 is the given box and level k has the same
centre and ``2^k`` times its half-extent, each with the same ``N``.  A point belongs to the smallest level whose box
holds it, so a 360° scene keeps fine cells on the object and coarse ones over the background it would otherwise
lose; only space outside the last level counts as empty.  Every consumer takes the grid as it is.
"""
from __future__ import annotations

import ctypes
import math
from typing import Callable, Dict, List, Optional, Sequence

import torch

from . import _lib
from .nerf import packed_weights
from .rendering import _seed_fields, render_rays

RESULT_KEYS = ("rgb_coarse", "depth_coarse", "opacity_coarse", "rgb_fine", "depth_fine", "opacity_fine")
MAX_LEVELS = 8


def level_ranges(x_range, y_range, z_range, level: int):
    """The (x_range, y_range, z_range) of cascade level ``level``: the ranges as given at level 0; for k >= 1, with
    ``c = 0.5 (lo + hi)`` and ``h = 0.5 (hi - lo)`` in float64, ``(c - 2^k h, c + 2^k h)`` per axis."""
    r = tuple(_lib.ranges_host(x_range, y_range, z_range))
    if level == 0:
        return r[0:2], r[2:4], r[4:6]
    out = []
    for a in range(3):
        lo, hi = r[2 * a], r[2 * a + 1]
        c, h = 0.5 * (lo + hi), 0.5 * (hi - lo)
        e = math.ldexp(h, int(level))
        out.append((c - e, c + e))
    return tuple(out)


def inner_cells(N: int, level: int):
    """The inner cell indices ``[a, b)`` of one axis of a level: a cell of level k >= 1 whose indices all lie in
    it is inside level k - 1's box, never looked up and always empty.  ``(0, 0)`` at level 0."""
    M = int(N) - 1
    if level == 0:
        return 0, 0
    a = (M + 3) // 4
    return a, max(3 * M // 4, a)


def _check_levels(levels, who: str) -> int:
    if int(levels) != levels or not 1 <= int(levels) <= MAX_LEVELS:
        raise ValueError(f"{who}: levels = {levels!r} must be an int in [1, {MAX_LEVELS}]")
    return int(levels)


class OccupancyGrid:
    """The occupied cells of a ``N``-point grid over ``x_range x y_range x z_range``: ``bits`` is a CUDA tensor of
    ``ceil((N-1)^3 / 32)`` uint32 words (stored as int32), one bit per cell, x fastest.  Cell ``(cx, cy, cz)`` spans
    ``[x_cx, x_cx+1] x [y_cy, y_cy+1] x [z_cz, z_cz+1]`` of ``np.linspace(*range, N)``; note that ``nb.sigma_grid``
    indexes ``[y, x, z]``, and this object does not.

    ``levels = L > 1``: a cascade (module docstring) of L such bit fields, level k's words after level k - 1's, each
    over ``level_ranges(..., k)``; the inner cells of levels k >= 1 (``inner_cells``) are 0."""

    def __init__(self, bits: torch.Tensor, N: int, x_range, y_range, z_range, dilate: int = 0, levels: int = 1):
        N = int(N)
        if not 2 <= N <= 1625:
            raise ValueError(f"OccupancyGrid: N = {N} outside [2, 1625]")
        levels = _check_levels(levels, "OccupancyGrid")
        words = ((N - 1) ** 3 + 31) // 32
        if not isinstance(bits, torch.Tensor) or not bits.is_cuda:
            raise RuntimeError("OccupancyGrid: bits must be a CUDA tensor (nerf_pl_b200 has no CPU fallback)")
        if bits.dtype not in (torch.int32, torch.uint32) or bits.numel() != words * levels:
            raise ValueError(f"OccupancyGrid: bits must hold {words * levels} 32-bit words")
        self.bits = bits.contiguous().view(torch.int32).reshape(-1)
        self.N = N
        self.ranges = tuple(_lib.ranges_host(x_range, y_range, z_range))
        if any(self.ranges[2 * a] == self.ranges[2 * a + 1] for a in range(3)):
            raise ValueError("OccupancyGrid: every range needs min != max")
        self.dilate = int(dilate)
        self.levels = levels

    @property
    def device(self) -> torch.device:
        return self.bits.device

    def grid_n(self) -> int:
        """The grid size argument of the C entries (``_lib.grid_n``): N, with the level count above it."""
        return _lib.grid_n(self.N, self.levels)

    def n_cells(self) -> int:
        """The cells a point can be looked up in: every cell of level 0, the non-inner ones of the other levels."""
        a, b = inner_cells(self.N, 1)
        return self.levels * (self.N - 1) ** 3 - (self.levels - 1) * (b - a) ** 3

    def occupied_fraction(self) -> float:
        """Occupied cells over ``n_cells()`` (a popcount reduction on the device)."""
        count = torch.empty(1, dtype=torch.int64, device=self.device)
        _lib.call("nerfb200_occupancy_popcount", self.device, self.bits.data_ptr(), self.grid_n(), count.data_ptr())
        return int(count.item()) / self.n_cells()

    def to_dense(self) -> torch.Tensor:
        """(N-1, N-1, N-1) bool, indexed ``[cx, cy, cz]`` (for tests and inspection); a cascade has a leading level
        axis, (L, N-1, N-1, N-1)."""
        M = self.N - 1
        shifts = torch.arange(32, dtype=torch.int32, device=self.device)
        words = self.bits.view(self.levels, -1)
        flat = ((words[:, :, None] >> shifts) & 1).reshape(self.levels, -1)[:, :M ** 3].bool()
        dense = flat.view(self.levels, M, M, M).permute(0, 3, 2, 1).contiguous()
        return dense[0] if self.levels == 1 else dense

    def state_dict(self) -> Dict[str, object]:
        """The grid's state; ``levels`` only for a cascade, so a one-level grid saves what it always saved."""
        st = {"bits": self.bits.detach().cpu(), "N": self.N, "ranges": tuple(self.ranges), "dilate": self.dilate}
        if self.levels > 1:
            st["levels"] = self.levels
        return st

    def load_state_dict(self, state: Dict[str, object]) -> "OccupancyGrid":
        self.__dict__.update(OccupancyGrid.from_state_dict(state, self.device).__dict__)
        return self

    @classmethod
    def from_state_dict(cls, state: Dict[str, object], device="cuda") -> "OccupancyGrid":
        """The grid of a ``state_dict()`` saved beside a checkpoint, on ``device``."""
        r = tuple(state["ranges"])
        return cls(torch.as_tensor(state["bits"]).to(device), state["N"], r[0:2], r[2:4], r[4:6], state["dilate"],
                   state.get("levels", 1))


@torch.no_grad()
def pack_occupancy(sigma: torch.Tensor, x_range, y_range, z_range, sigma_threshold: float,
                   dilate: int = 1, levels: int = 1) -> OccupancyGrid:
    """The occupancy grid of a CUDA (N, N, N) sigma grid in ``nb.sigma_grid``'s order (``sigma[i, j, k] =
    sigma(x_j, y_i, z_k)``): a cell is occupied iff the largest sigma of its 8 corners is ``> sigma_threshold``; the
    set is dilated by ``dilate`` cells in Chebyshev distance and packed.

    ``levels = L > 1``: sigma is (L, N, N, N), level k's grid over ``level_ranges(..., k)``; each level is marked
    with its inner cells empty, dilated within the level and packed with its inner cells cleared."""
    levels = _check_levels(levels, "pack_occupancy")
    if not isinstance(sigma, torch.Tensor) or not sigma.is_cuda:
        raise RuntimeError("pack_occupancy: sigma must be a CUDA tensor (nerf_pl_b200 has no CPU fallback)")
    cube = sigma.shape[-3:]
    if sigma.dim() != (3 if levels == 1 else 4) or not (cube[0] == cube[1] == cube[2]) or \
            (levels > 1 and sigma.shape[0] != levels):
        raise ValueError("sigma must be (N, N, N)" if levels == 1 else f"sigma must be ({levels}, N, N, N)")
    s = sigma.detach().to(torch.float32).contiguous()
    N = s.shape[-1]
    nbytes = _lib.load().nerfb200_occupancy_workspace_bytes(N)
    if nbytes == 0:
        raise ValueError(f"pack_occupancy: N = {N} outside [2, 1625]")
    ws = _lib.workspace(nbytes, s.device)
    bits = torch.empty(levels * (((N - 1) ** 3 + 31) // 32), dtype=torch.int32, device=s.device)
    _lib.call("nerfb200_occupancy_pack", s.device, s.data_ptr(), _lib.grid_n(N, levels), float(sigma_threshold),
              int(dilate), ws.data_ptr(), ws.numel(), bits.data_ptr())
    return OccupancyGrid(bits, N, x_range, y_range, z_range, dilate, levels)


@torch.no_grad()
def occupancy_grid(model: torch.nn.Module, N: int, x_range, y_range, z_range, sigma_threshold: float, dilate: int = 1,
                   chunk: int = 1 << 21) -> OccupancyGrid:
    """The occupancy grid of ``model`` (the network that decides the picture: the fine one): ``nb.sigma_grid`` on N^3
    points, with ``N`` and the ranges as for mesh extraction, then ``pack_occupancy``.  The float sigma grid is
    transient.  A ray that only crosses unoccupied cells will be given the vacuum value, so choose
    ``sigma_threshold`` well below the density of anything visible (see the module docstring for what is and is
    not guaranteed).  ``occupancy_cascade`` builds a cascade."""
    return occupancy_cascade(model, N, x_range, y_range, z_range, sigma_threshold, 1, dilate, chunk)


@torch.no_grad()
def occupancy_cascade(model: torch.nn.Module, N: int, x_range, y_range, z_range, sigma_threshold: float, levels: int,
                      dilate: int = 1, chunk: int = 1 << 21) -> OccupancyGrid:
    """``occupancy_grid`` with ``levels`` cascade levels (module docstring) around the box of ``x_range x y_range x
    z_range``: ``nb.sigma_grid`` on each level's box (``level_ranges``), L N^3 points, then
    ``pack_occupancy(..., levels=levels)``.  ``levels = 1`` is ``occupancy_grid``."""
    from .mesh import sigma_grid     # mesh imports inference, which imports this module
    levels = _check_levels(levels, "occupancy_cascade")
    if levels == 1:
        sigma = sigma_grid(model, int(N), x_range, y_range, z_range, chunk)
    else:
        sigma = torch.stack([sigma_grid(model, int(N), *level_ranges(x_range, y_range, z_range, k), chunk)
                             for k in range(levels)])
    grid = pack_occupancy(sigma, x_range, y_range, z_range, sigma_threshold, dilate, levels)
    del sigma
    return grid


def _check_rays(rays: torch.Tensor, occupancy: OccupancyGrid) -> torch.Tensor:
    if not isinstance(occupancy, OccupancyGrid):
        raise ValueError("occupancy must be a nerf_pl_b200.OccupancyGrid")
    if not isinstance(rays, torch.Tensor) or not rays.is_cuda:
        raise RuntimeError("rays must be a CUDA tensor (nerf_pl_b200 has no CPU fallback)")
    if rays.dim() != 2 or rays.shape[1] != 8:
        raise ValueError("rays must be (n, 8) [o, d, near, far]")
    if rays.device != occupancy.device:
        raise ValueError("rays and the occupancy grid must be on the same device")
    return rays.detach().to(torch.float32).contiguous()


@torch.no_grad()
def cull_rays(rays: torch.Tensor, occupancy: OccupancyGrid, return_flag: bool = False):
    """(live_idx (n_live) int64, increasing; live_rays (n_live, 8) = rays[live_idx]) of the rays whose segment
    ``o + t d, t in [near, far]`` crosses an occupied cell.  The rays are taken as given: for NDC rays use a grid
    built over NDC coordinates.  A ray with a non-finite value or ``far <= near`` is live.  ``return_flag`` adds
    the per-ray uint8 flag.  Synchronises (the number of live rays sizes the outputs)."""
    r = _check_rays(rays, occupancy)
    dev, n = r.device, r.shape[0]
    ws = _lib.workspace(_lib.load().nerfb200_cull_workspace_bytes(n), dev)
    flag = torch.empty(n, dtype=torch.uint8, device=dev)
    n_live = ctypes.c_int64()
    _lib.call("nerfb200_cull_count", dev, r.data_ptr(), n, occupancy.bits.data_ptr(), occupancy.grid_n(),
              (ctypes.c_double * 6)(*occupancy.ranges), ws.data_ptr(), ws.numel(), flag.data_ptr(), ctypes.byref(n_live))
    live_idx = torch.empty(n_live.value, dtype=torch.int64, device=dev)
    live_rays = torch.empty(n_live.value, 8, dtype=torch.float32, device=dev)
    if n_live.value:
        _lib.call("nerfb200_cull_emit", dev, r.data_ptr(), n, flag.data_ptr(), ws.data_ptr(), ws.numel(),
                  live_idx.data_ptr(), live_rays.data_ptr())
    return (live_idx, live_rays, flag) if return_flag else (live_idx, live_rays)


def result_keys(N_importance: int, test_time: bool) -> List[str]:
    keys = ["opacity_coarse"] if test_time else ["rgb_coarse", "depth_coarse", "opacity_coarse"]
    return keys + (["rgb_fine", "depth_fine", "opacity_fine"] if N_importance > 0 else [])


@torch.no_grad()
def scatter_results(compact: Optional[Dict[str, torch.Tensor]], live_idx: torch.Tensor, n_rays: int, white_back: bool,
                    keys: Optional[Sequence[str]] = None) -> Dict[str, torch.Tensor]:
    """Full-size results of a render of compacted rays, in one launch: row ``live_idx[r]`` of every key is row r of
    ``compact``; every other ray gets the vacuum value (opacity 0, depth 0, rgb 1 if ``white_back`` else 0).
    ``keys`` names the results when there is no live ray (``compact`` may then be None)."""
    dev = live_idx.device
    n_live = live_idx.shape[0]
    keys = list(compact) if keys is None else list(keys)
    if not keys or any(k not in RESULT_KEYS for k in keys):
        raise ValueError(f"scatter_results: keys must be among {RESULT_KEYS}")
    src = {k: compact[k].detach().to(torch.float32).contiguous() for k in keys} if n_live else {}
    out = {k: torch.empty((n_rays, 3) if k.startswith("rgb") else (n_rays,), dtype=torch.float32, device=dev)
           for k in keys}
    for k in src:
        if src[k].shape != (n_live,) + tuple(out[k].shape[1:]) or src[k].device != dev:
            raise ValueError(f"scatter_results: {k} must be {(n_live,) + tuple(out[k].shape[1:])} on {dev}")
    ptrs = lambda d: (ctypes.c_void_p * 6)(*[d[k].data_ptr() if k in d else None for k in RESULT_KEYS])  # noqa: E731
    idx = live_idx.to(torch.int64).contiguous()
    _lib.call("nerfb200_scatter_results", dev, ptrs(src), ptrs(out), idx.data_ptr() if n_live else None, n_live,
              int(n_rays), int(bool(white_back)))
    return out


def render_culled(render_fn: Callable[[torch.Tensor], Dict[str, torch.Tensor]], rays: torch.Tensor,
                  occupancy: OccupancyGrid, keys: Sequence[str], white_back: bool) -> Dict[str, torch.Tensor]:
    """cull -> ``render_fn(live_rays)`` -> scatter.  With no live ray there is no render launch."""
    live_idx, live_rays = cull_rays(rays, occupancy)
    compact = render_fn(live_rays) if live_idx.shape[0] else None
    out = scatter_results(compact, live_idx, rays.shape[0], white_back, keys)
    out["live"] = int(live_idx.shape[0])
    out["live_idx"] = live_idx
    return out


# Rays per nerfb200_render_samples call: the workspace is about 6.4 KB per ray at 64 + 128 samples (210 MB per
# chunk), and each chunk costs two read-backs of a sample count.  Tests lower it to show that results do not depend
# on it.
_SAMPLE_CHUNK = 1 << 15

SKIP_MODES = ("rays", "samples")


def check_skip(skip: str, occupancy) -> None:
    """``skip`` must name a mode, and ``"samples"`` needs a grid."""
    if skip not in SKIP_MODES:
        raise ValueError(f"skip must be one of {SKIP_MODES}, got {skip!r}")
    if skip == "samples" and occupancy is None:
        raise ValueError("skip='samples' needs an occupancy grid")


def check_early_stop(early_stop: float, samples: bool, N_importance: int, perturb: float = 0.0,
                     noise_std: float = 0.0) -> float:
    """``early_stop`` (DESIGN.md §10f) as a float; ``samples`` is whether empty samples are skipped.  A ValueError for
    anything the coarse-only termination does not support."""
    eps = float(early_stop)
    if not 0.0 <= eps <= 1.0:
        raise ValueError(f"early_stop must be in [0, 1], got {early_stop!r}")
    if eps > 0.0:
        if not samples:
            raise ValueError("early_stop > 0 needs skip='samples' (occupancy= for fuse_vertex_colors)")
        if int(N_importance) > 0:
            raise ValueError("early_stop > 0 needs N_importance = 0: with importance samples at most about 5 % of the "
                             "evaluated fine samples lie behind the cut (DESIGN.md §10f), and cutting the coarse pass "
                             "would change z_vals_fine")
        if float(perturb) != 0.0 or float(noise_std) != 0.0:
            raise ValueError("early_stop > 0 needs perturb = 0 and noise_std = 0")
    return eps


@torch.no_grad()
def render_samples(models: Sequence[torch.nn.Module], rays: torch.Tensor, occupancy: OccupancyGrid, N_samples: int,
                   use_disp: bool, N_importance: int, white_back: bool, test_time: bool,
                   live_flag: Optional[torch.Tensor] = None, extras: bool = False,
                   per_sample: bool = False, perturb: float = 0.0, noise_std: float = 0.0,
                   randoms=(None, None, None, None), rng_seed=None, *,
                   early_stop: float = 0.0) -> Dict[str, torch.Tensor]:
    """Render every ray of ``rays`` (n, 8) with empty samples skipped (module docstring), in chunks of
    ``_SAMPLE_CHUNK`` rays.  Returns ``render_rays``' keys for ``test_time`` / ``N_importance``, ``extras`` as
    ``render_rays`` gives them, and ``'live_samples'``: (evaluated coarse samples, evaluated fine samples).
    ``live_flag`` (n) uint8: a ray whose flag is 0 has every sample skipped.  ``per_sample`` adds
    ``'samples_coarse'`` / ``'samples_fine'`` (n, S, 4: rgb and sigma, 0 where skipped) and ``'mask_coarse'`` /
    ``'mask_fine'`` (n, 6) int32 (bit b of word w: sample 32 w + b evaluated).  Synchronises twice per chunk.

    ``perturb`` / ``noise_std`` > 0 render as the training step does (``render_rays(..., occupancy=)``'s graph path,
    the same values bit for bit): ``randoms`` = (perturb_rand, noise_coarse, u_rand, noise_fine), rows of ``rays``
    (None where not used), and ``rng_seed`` an in-kernel seed as ``rendering._resolve_randoms`` returns it, under
    which a ray draws by its index in ``rays`` whatever the chunk.

    ``early_stop`` = eps > 0 (``N_importance = 0``, ``perturb = noise_std = 0``) stops each ray once it is opaque
    (DESIGN.md §10f): the coarse samples are evaluated in rounds of one 32-sample mask word, and a ray whose float64
    transmittance falls below eps after a word has its later words treated as empty.  Weights up to the end of the
    cut word are bit-identical to ``early_stop = 0``, later ones are 0, a ray never cut is bit-identical in every
    output, and |d opacity|, |d rgb| are at most ``T_cut (1 + S 1e-10) + 4e-6`` (|d depth| that times the ray's
    largest depth).  ``'live_samples'`` counts what was evaluated; ``per_sample`` also returns ``'cut_coarse'`` (n)
    int32, the word each ray was cut after or -1, and the masks without the dropped words.  With ``N_samples = 32``
    there is one word and nothing to drop: the render takes the path without termination.  It synchronises once per
    word of each chunk."""
    S_c, K = int(N_samples), int(N_importance)
    S_f = S_c + K
    eps = check_early_stop(early_stop, True, K, perturb, noise_std)
    if K > 0 and len(models) < 2:
        raise ValueError("N_importance > 0 needs a fine model (models[1])")
    lib = _lib.load()
    rays = rays.detach().to(torch.float32).contiguous()
    dev, n = rays.device, rays.shape[0]
    chunk = max(1, min(int(_SAMPLE_CHUNK), n))
    nbytes = lib.nerfb200_samples_workspace_bytes(chunk, S_c, K)
    if nbytes == 0:
        raise ValueError("skip='samples' supports N_samples in {32, 64, 128} and N_importance a multiple of 32 with "
                         "N_samples + N_importance <= 192")
    f32 = dict(dtype=torch.float32, device=dev)
    out = {k: torch.empty((n, 3) if k.startswith("rgb") else (n,), **f32) for k in result_keys(K, bool(test_time))}
    opt = {}
    if extras:
        opt["weights_coarse"] = torch.empty(n, S_c, **f32)
        if K > 0:
            opt["z_fine"] = torch.empty(n, S_f, **f32)
            opt["weights_fine"] = torch.empty(n, S_f, **f32)
    if per_sample:
        opt["samples_coarse"] = torch.empty(n, S_c, 4, **f32)
        opt["mask_coarse"] = torch.empty(n, 6, dtype=torch.int32, device=dev)
        if K > 0:
            opt["samples_fine"] = torch.empty(n, S_f, 4, **f32)
            opt["mask_fine"] = torch.empty(n, 6, dtype=torch.int32, device=dev)
        if eps > 0.0:
            opt["cut_coarse"] = torch.empty(n, dtype=torch.int32, device=dev)
    flag = None if live_flag is None else live_flag.to(torch.uint8).contiguous()
    pr, nc, ur, nf = [None if t is None else t.detach().to(torch.float32).contiguous() for t in randoms]
    for name, t, cols in (("perturb_rand", pr, S_c), ("noise_coarse", nc, S_c), ("u_rand", ur, K),
                          ("noise_fine", nf, S_f)):
        if t is not None and (tuple(t.shape) != (n, cols) or t.device != dev):
            raise ValueError(f"{name} must be ({n}, {cols}) on {dev}, got {tuple(t.shape)} on {t.device}")
    rng = _seed_fields(rng_seed)
    packed = (packed_weights(models[0]), packed_weights(models[1]) if K > 0 else None)
    ws = _lib.workspace(nbytes, dev)
    counts = [0, 0]
    got = (ctypes.c_int64 * 2)()
    for lo in range(0, n, chunk):
        m = min(chunk, n - lo)
        ptr = lambda t: None if t is None else t.data_ptr() + lo * t.stride(0) * t.element_size()  # noqa: E731
        args = _lib.SamplesArgs(
            rays=ptr(rays), n_rays=m, live_flag=ptr(flag), packed_coarse=packed[0].data_ptr(),
            packed_fine=None if packed[1] is None else packed[1].data_ptr(), n_samples=S_c, n_importance=K,
            use_disp=int(bool(use_disp)), white_back=int(bool(white_back)), test_time=int(bool(test_time)),
            bits=occupancy.bits.data_ptr(), N=occupancy.N, ranges=_lib.ranges_host(*[occupancy.ranges[2 * a:2 * a + 2]
                                                                                       for a in range(3)]),
            levels=occupancy.levels,
            **{k: ptr(out.get(k)) for k in RESULT_KEYS}, **{k: ptr(t) for k, t in opt.items()},
            perturb=float(perturb), noise_std=float(noise_std), perturb_rand=ptr(pr), noise_coarse=ptr(nc),
            u_rand=ptr(ur), noise_fine=ptr(nf), rng_ray_offset=lo, early_stop=eps, **rng)
        _lib.call("nerfb200_render_samples", dev, ctypes.byref(args), ws.data_ptr(), ws.numel(), got)
        counts[0] += got[0]
        counts[1] += got[1]
    if extras:
        out["weights_coarse"] = opt["weights_coarse"]
        if K > 0:
            out["z_vals_fine"] = opt["z_fine"]
            out["weights_fine"] = opt["weights_fine"]
    if per_sample:
        out.update({k: v for k, v in opt.items() if k.startswith(("samples", "mask", "cut"))})
    out["live_samples"] = tuple(counts)
    return out


def render_culled_samples(models: Sequence[torch.nn.Module], rays: torch.Tensor, occupancy: OccupancyGrid,
                          N_samples: int, use_disp: bool, N_importance: int, white_back: bool, test_time: bool,
                          extras: bool = False, sharded: bool = False, *,
                          early_stop: float = 0.0) -> Dict[str, torch.Tensor]:
    """cull -> ``render_samples(live rays)`` -> scatter, with ``'live'``, ``'live_idx'`` and ``'live_samples'``.
    With ``extras`` every ray goes through ``render_samples``, the culled ones with every sample skipped, so that the
    extra tensors are full size; their results are then the vacuum value as well.  ``sharded`` splits the live rays
    over the ranks (``render_rays_sharded``); ``'live_samples'`` then counts this rank's samples.  ``early_stop``:
    as for ``render_samples``."""
    eps = check_early_stop(early_stop, True, N_importance)
    r = _check_rays(rays, occupancy)
    keys = result_keys(int(N_importance), bool(test_time))
    counts = [0, 0]

    def fn(live, flag=None):
        res = render_samples(models, live, occupancy, N_samples, use_disp, N_importance, white_back, test_time,
                             live_flag=flag, extras=extras, early_stop=eps)
        ls = res.pop("live_samples")
        counts[0] += ls[0]
        counts[1] += ls[1]
        return res

    if extras:
        live_idx, _, flag = cull_rays(r, occupancy, return_flag=True)
        out = fn(r, flag)
    else:
        from .sharded import render_rays_sharded
        run = (lambda x: render_rays_sharded(fn, x)) if sharded else fn
        live_idx, live_rays = cull_rays(r, occupancy)
        compact = run(live_rays) if live_idx.shape[0] else None
        out = scatter_results(compact, live_idx, r.shape[0], white_back, keys)
    out["live"] = int(live_idx.shape[0])
    out["live_idx"] = live_idx
    out["live_samples"] = tuple(counts)
    return out


@torch.no_grad()
def render_rays_culled(models: List[torch.nn.Module], embeddings: List[torch.nn.Module], rays: torch.Tensor,
                       occupancy: OccupancyGrid, N_samples: int = 64, use_disp: bool = False, N_importance: int = 0,
                       white_back: bool = False, test_time: bool = True, *, perturb: float = 0,
                       noise_std: float = 0, skip: str = "rays", extras: bool = False,
                       early_stop: float = 0.0) -> Dict[str, torch.Tensor]:
    """``render_rays`` at inference with empty space skipped: the same keys, shapes and dtypes, plus ``'live'``
    (the number of rays rendered) and ``'live_idx'`` (their indices, int64).  Live rays are bit-identical to
    ``render_rays(..., perturb=0, noise_std=0)``; a culled ray gets the vacuum value, an approximation whose error
    is bounded empirically, not proved (module docstring).  Inference only: ``perturb`` and ``noise_std`` must be
    0 and no gradient is built; anything else is a ValueError, because training must see the background rays to
    learn that they are empty.

    ``skip="samples"`` also skips the empty samples of the live rays (module docstring; DESIGN.md "Skipping empty
    samples"): faster, no longer bit-identical, and the result holds ``'live_samples'`` (evaluated coarse, fine
    samples).  ``extras=True`` (with ``"samples"``) adds ``weights_coarse``, ``weights_fine`` and ``z_vals_fine`` as
    ``render_rays`` does.  It synchronises twice per chunk of ``_SAMPLE_CHUNK`` live rays.

    ``early_stop`` = eps > 0 (``skip="samples"``, ``N_importance = 0``) also stops each live ray once its
    transmittance falls below eps after a 32-sample word, within the bound ``render_samples`` states (DESIGN.md §10f);
    0 renders exactly as without it.  With ``N_samples = 32`` there is one word and nothing to stop."""
    if float(perturb) != 0.0 or float(noise_std) != 0.0:
        raise ValueError("render_rays_culled is inference only (perturb = 0, noise_std = 0): training must see the "
                         "background rays to learn that they are empty")
    check_skip(skip, occupancy)
    eps = check_early_stop(early_stop, skip == "samples", N_importance)
    if extras and skip != "samples":
        raise ValueError("extras=True needs skip='samples' (render_rays(..., extras=True) renders every ray)")
    r = _check_rays(rays, occupancy)
    if skip == "samples":
        from .rendering import _check_render_inputs
        _check_render_inputs("render_rays_culled", models, embeddings, int(N_importance), r)
        return render_culled_samples(list(models), r, occupancy, int(N_samples), use_disp, int(N_importance),
                                     white_back, test_time, extras=extras, early_stop=eps)

    def fn(live):
        return render_rays(list(models), list(embeddings), live, int(N_samples), use_disp, 0, 0, int(N_importance),
                           1024 * 32, white_back, test_time=test_time, match_reference_rng=False)

    return render_culled(fn, r, occupancy, result_keys(int(N_importance), bool(test_time)), bool(white_back))
