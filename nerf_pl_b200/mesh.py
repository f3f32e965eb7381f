"""Coloured mesh extraction on the device (the reference's ``extract_color_mesh.py``, ``README_mesh.md``).

sigma grid -> marching cubes -> index-to-world transform -> largest cluster -> occlusion-aware vertex
colours, every stage an sm_90a kernel of ``libnerf_pl_b200.so`` (csrc/mesh_kernels.cuh); the grid query and
the occlusion renders run the existing fused MLP / render launches.  Replaces PyMCubes
(``mcubes.marching_cubes``), open3d (``cluster_connected_triangles`` + ``remove_unreferenced_vertices``),
``cv2.remap`` and the numpy projection loop; ``write_ply`` writes what plyfile wrote.  Conventions and the
reference's quirks that are kept: DESIGN.md "Coloured mesh extraction".  The ``--use_vertex_normal`` method is
``vertex_normals`` -> ``normal_rays`` -> the fused render of both networks, in one call: ``normal_vertex_colors``.

The Unity volume export of extract_mesh.ipynb is ``rgb_sigma_grid`` -> ``pack_volume`` -> ``write_vol`` (DESIGN.md
"Unity volume").
"""
from __future__ import annotations

import ctypes
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .culling import OccupancyGrid, check_early_stop, render_rays_culled
from .inference import to_uint8
from .nerf import Embedding, packed_weights
from .rendering import render_rays


def _device_of(model: torch.nn.Module) -> torch.device:
    dev = next(model.parameters()).device
    if dev.type != "cuda":
        raise RuntimeError("nerf_pl_b200.mesh runs on CUDA only (no CPU fallback)")
    return dev


def _cuda(t: torch.Tensor, what: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f"{what} must be a CUDA tensor (nerf_pl_b200 has no CPU fallback)")
    return t


@torch.no_grad()
def grid_positions(N: int, x_range, y_range, z_range, start: int = 0, count: Optional[int] = None,
                   device=None) -> torch.Tensor:
    """Points [start, start+count) of ``torch.FloatTensor(np.stack(np.meshgrid(x, y, z), -1).reshape(-1, 3))``
    with ``x = np.linspace(*x_range, N)`` etc. (extract_color_mesh.py:119-123), built on the device."""
    device = torch.device("cuda") if device is None else torch.device(device)
    count = N ** 3 - start if count is None else count
    out = torch.empty(count, 3, dtype=torch.float32, device=device)
    _lib.call("nerfb200_grid_positions", device, N, _lib.ranges_host(x_range, y_range, z_range), start, count,
              out.data_ptr())
    return out


def _check_occupancy(occupancy, dev: torch.device) -> OccupancyGrid:
    if not isinstance(occupancy, OccupancyGrid):
        raise ValueError("occupancy must be a nerf_pl_b200.OccupancyGrid (for a DensityGrid pass its .grid)")
    if occupancy.device != dev:
        raise RuntimeError(f"the occupancy grid is on {occupancy.device}, the model on {dev}")
    return occupancy


def _masked_grid(entry: str, model: torch.nn.Module, N: int, ranges, occupancy, chunk: int, channels: int):
    """The grid of ``entry`` (nerfb200_sigma_grid_masked or nerfb200_rgb_sigma_grid_masked): (grid, evaluated)."""
    dev = _device_of(model)
    occ = _check_occupancy(occupancy, dev)
    out = torch.empty((N, N, N) if channels == 1 else (N, N, N, channels), dtype=torch.float32, device=dev)
    blob = packed_weights(model)
    chunk = int(min(chunk, N ** 3))
    nbytes = _lib.load().nerfb200_masked_grid_workspace_bytes(chunk)
    if nbytes == 0:
        raise ValueError(f"chunk = {chunk} must be >= 1")
    ws = _lib.workspace(nbytes, dev)
    evaluated = ctypes.c_int64()
    _lib.call(entry, dev, blob.data_ptr(), N, ranges, occ.bits.data_ptr(), occ.grid_n(),
              (ctypes.c_double * 6)(*occ.ranges), chunk, ws.data_ptr(), ws.numel(), out.data_ptr(),
              ctypes.byref(evaluated))
    return out, int(evaluated.value)


@torch.no_grad()
def sigma_grid(model: torch.nn.Module, N: int, x_range, y_range, z_range, chunk: int = 1 << 21, *,
               occupancy: Optional[OccupancyGrid] = None, return_evaluated: bool = False):
    """(N, N, N) fp32 ``max(sigma, 0)`` of ``model`` on the reference's grid (extract_color_mesh.py:113-140):
    ``sigma[i, j, k] = max(sigma(x_j, y_i, z_k), 0)`` (np.meshgrid's 'xy' indexing).  ``chunk`` points are
    queried per launch; the scratch is their positions only.

    ``occupancy`` (an ``OccupancyGrid``; for a ``DensityGrid`` its ``.grid``) evaluates only the lattice points that
    lie in the closed box of an occupied cell, the rule of ``skip="samples"``: those get the value above bit for bit,
    every other point gets +0.0 (DESIGN.md "Grids through an occupancy grid").  Its N and box are independent of the
    mesh grid's.  It synchronises once per chunk.  ``return_evaluated`` returns (grid, number of evaluated points;
    N^3 without a grid)."""
    if occupancy is not None:
        out, evaluated = _masked_grid("nerfb200_sigma_grid_masked", model, int(N),
                                      _lib.ranges_host(x_range, y_range, z_range), occupancy, chunk, 1)
        return (out, evaluated) if return_evaluated else out
    dev = _device_of(model)
    out = torch.empty(N, N, N, dtype=torch.float32, device=dev)
    blob = packed_weights(model)
    chunk = int(min(chunk, N ** 3))
    ws = _lib.workspace(_lib.load().nerfb200_sigma_grid_workspace_bytes(chunk), dev)
    _lib.call("nerfb200_sigma_grid", dev, blob.data_ptr(), N, _lib.ranges_host(x_range, y_range, z_range), chunk,
              ws.data_ptr(), ws.numel(), out.data_ptr())
    return (out, N ** 3) if return_evaluated else out


@torch.no_grad()
def marching_cubes(sigma: torch.Tensor, threshold: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """Drop-in for ``mcubes.marching_cubes(sigma, threshold)`` on a CUDA (n0, n1, n2) grid: index-space
    vertices (V, 3) float64 and triangles (T, 3) int32, on the device.  Inside is ``sigma > threshold``;
    normals point from inside to outside; the order is fixed (DESIGN.md)."""
    s = _cuda(sigma, "sigma").detach().to(torch.float32).contiguous()
    if s.dim() != 3:
        raise ValueError("sigma must be a 3-D grid")
    n0, n1, n2 = s.shape
    nbytes = _lib.load().nerfb200_mc_workspace_bytes(n0, n1, n2)
    if nbytes == 0:
        raise ValueError(f"marching_cubes: unsupported grid shape {tuple(s.shape)}")
    ws = _lib.workspace(nbytes, s.device)
    counts = (ctypes.c_int64 * 2)()
    _lib.call("nerfb200_mc_count", s.device, s.data_ptr(), n0, n1, n2, float(threshold), ws.data_ptr(), ws.numel(),
              counts)
    verts = torch.empty(counts[0], 3, dtype=torch.float64, device=s.device)
    tris = torch.empty(counts[1], 3, dtype=torch.int32, device=s.device)
    _lib.call("nerfb200_mc_emit", s.device, s.data_ptr(), n0, n1, n2, float(threshold), ws.data_ptr(), ws.numel(),
              verts.data_ptr() if counts[0] else None, tris.data_ptr() if counts[1] else None)
    return verts, tris


SPARSE_MC_MAX_N = 2048


@torch.no_grad()
def sparse_marching_cubes(model: torch.nn.Module, N: int, x_range, y_range, z_range, threshold: float, *,
                          occupancy: OccupancyGrid) -> Tuple[torch.Tensor, torch.Tensor]:
    """``marching_cubes(sigma_grid(model, N, x_range, y_range, z_range, occupancy=occupancy), threshold)`` without the
    dense N^3 grid, for N in [2, 2048]: the same index-space vertices (V, 3) float64 and triangles (T, 3) int32, bit
    for bit and in the same order (DESIGN.md §10i).  Only the 8^3-point bricks that hold a point the grid evaluates
    (and their lower neighbours) are queried, stored and marched, so memory follows the occupied volume."""
    dev = _device_of(model)
    occ = _check_occupancy(occupancy, dev)
    N = int(N)
    if not 2 <= N <= SPARSE_MC_MAX_N:
        raise ValueError(f"sparse_marching_cubes: N = {N} outside [2, {SPARSE_MC_MAX_N}]")
    lib = _lib.load()
    ranges = _lib.ranges_host(x_range, y_range, z_range)
    occ_ranges = (ctypes.c_double * 6)(*occ.ranges)
    plan = _lib.workspace(lib.nerfb200_sparse_mc_plan_workspace_bytes(N), dev)
    bricks = (ctypes.c_int64 * 2)()
    _lib.call("nerfb200_sparse_mc_plan", dev, N, ranges, occ.bits.data_ptr(), occ.grid_n(), occ_ranges,
              plan.data_ptr(), plan.numel(), bricks)
    ws = _lib.workspace(lib.nerfb200_sparse_mc_workspace_bytes(N, bricks[0], bricks[1]), dev)
    counts = (ctypes.c_int64 * 2)()
    _lib.call("nerfb200_sparse_mc_count", dev, packed_weights(model).data_ptr(), N, ranges, occ.bits.data_ptr(),
              occ.grid_n(), occ_ranges, float(threshold), plan.data_ptr(), plan.numel(), bricks, ws.data_ptr(),
              ws.numel(), counts)
    verts = torch.empty(counts[0], 3, dtype=torch.float64, device=dev)
    tris = torch.empty(counts[1], 3, dtype=torch.int32, device=dev)
    emit = _lib.workspace(lib.nerfb200_sparse_mc_emit_workspace_bytes(counts[0], counts[1]), dev)
    _lib.call("nerfb200_sparse_mc_emit", dev, N, float(threshold), plan.data_ptr(), plan.numel(), bricks,
              ws.data_ptr(), ws.numel(), counts, emit.data_ptr(), emit.numel(),
              verts.data_ptr() if counts[0] else None, tris.data_ptr() if counts[1] else None)
    return verts, tris


@torch.no_grad()
def to_world(vertices: torch.Tensor, N: int, x_range, y_range, z_range) -> torch.Tensor:
    """extract_color_mesh.py:148-154 on the device, quirks included: divides by N (not N - 1) and swaps the
    x / y ranges (x takes y_range)."""
    v = _cuda(vertices, "vertices").detach().to(torch.float64).contiguous()
    out = torch.empty(v.shape[0], 3, dtype=torch.float32, device=v.device)
    _lib.call("nerfb200_mesh_to_world", v.device, v.data_ptr(), v.shape[0], N,
              _lib.ranges_host(x_range, y_range, z_range), out.data_ptr())
    return out


@torch.no_grad()
def keep_largest_cluster(vertices: torch.Tensor, triangles: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """extract_color_mesh.py:163-171: the edge-connected component with the most triangles (ties: the one
    holding the lowest-indexed triangle), unreferenced vertices removed, order kept."""
    v = _cuda(vertices, "vertices").detach().to(torch.float32).contiguous()
    t = _cuda(triangles, "triangles").detach().to(torch.int32).contiguous()
    if t.shape[0] == 0:
        return v[:0], t[:0]
    ws = _lib.workspace(_lib.load().nerfb200_mesh_cluster_workspace_bytes(v.shape[0], t.shape[0]), v.device)
    counts = (ctypes.c_int64 * 2)()
    _lib.call("nerfb200_mesh_cluster_count", v.device, t.data_ptr(), t.shape[0], v.shape[0], ws.data_ptr(), ws.numel(),
              counts)
    vo = torch.empty(counts[0], 3, dtype=torch.float32, device=v.device)
    to = torch.empty(counts[1], 3, dtype=torch.int32, device=v.device)
    _lib.call("nerfb200_mesh_cluster_emit", v.device, v.data_ptr(), t.data_ptr(), t.shape[0], v.shape[0], ws.data_ptr(),
              ws.numel(), vo.data_ptr(), to.data_ptr())
    return vo, to


@torch.no_grad()
def extract_mesh(model: torch.nn.Module, N_grid: int, x_range, y_range, z_range, sigma_threshold: float,
                 keep_largest: bool = True, *,
                 occupancy: Optional[OccupancyGrid] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """extract_color_mesh.py:113-171: world vertices (V, 3) fp32 and triangles (T, 3) int32 on the device.
    ``occupancy``: the mesh is ``marching_cubes(sigma_grid(..., occupancy=occupancy), sigma_threshold)``, so density
    the grid calls empty never reaches marching cubes; it is computed by ``sparse_marching_cubes``, which never builds
    the dense grid, so N_grid may go up to 2048."""
    if occupancy is not None:
        vidx, tris = sparse_marching_cubes(model, N_grid, x_range, y_range, z_range, sigma_threshold,
                                           occupancy=occupancy)
    else:
        sigma = sigma_grid(model, N_grid, x_range, y_range, z_range)
        vidx, tris = marching_cubes(sigma, sigma_threshold)
        del sigma
    verts = to_world(vidx, N_grid, x_range, y_range, z_range)
    if keep_largest:
        verts, tris = keep_largest_cluster(verts, tris)
    return verts, tris


@torch.no_grad()
def remap_bilinear(image: torch.Tensor, xy: torch.Tensor) -> torch.Tensor:
    """``cv2.remap(image, xy[:, 0], xy[:, 1], cv2.INTER_LINEAR)`` (constant 0 border) of a CUDA (H, W, 3) uint8
    image at (n, 2) fp32 points -> (n, 3) uint8."""
    img = _cuda(image, "image").contiguous()
    if img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] != 3:
        raise ValueError("image must be (H, W, 3) uint8")
    p = _cuda(xy, "xy").detach().to(torch.float32).contiguous()
    out = torch.empty(p.shape[0], 3, dtype=torch.uint8, device=img.device)
    _lib.call("nerfb200_remap_bilinear", img.device, img.data_ptr(), img.shape[0], img.shape[1], p.data_ptr(),
              p.shape[0], out.data_ptr())
    return out


def w2c_of(pose) -> np.ndarray:
    """extract_color_mesh.py:220-221: ``np.linalg.inv([[c2w], [0, 0, 0, 1]])[:3]`` in float64."""
    c2w = np.asarray(pose.detach().cpu().numpy() if isinstance(pose, torch.Tensor) else pose, dtype=np.float64)
    return np.linalg.inv(np.concatenate([c2w.reshape(3, 4), np.array([[0, 0, 0, 1.0]])], 0))[:3]


@torch.no_grad()
def project_view(vertices: torch.Tensor, image: torch.Tensor, pose, focal: float, near: float):
    """One view of extract_color_mesh.py:215-262: (colours (V, 3) uint8, depth (V) fp64, occlusion rays (V, 8))."""
    v = _cuda(vertices, "vertices")
    H, W = image.shape[0], image.shape[1]
    c2w = np.asarray(pose.detach().cpu().numpy() if isinstance(pose, torch.Tensor) else pose, dtype=np.float64)
    w2c = (ctypes.c_double * 12)(*w2c_of(c2w).reshape(-1).tolist())
    origin = (ctypes.c_float * 3)(*np.asarray(c2w.reshape(3, 4)[:, 3], dtype=np.float32).tolist())
    n = v.shape[0]
    colors = torch.empty(n, 3, dtype=torch.uint8, device=v.device)
    depth = torch.empty(n, dtype=torch.float64, device=v.device)
    rays = torch.empty(n, 8, dtype=torch.float32, device=v.device)
    _lib.call("nerfb200_color_project", v.device, v.data_ptr(), n, w2c, origin, float(focal), W, H, image.data_ptr(),
              float(near), colors.data_ptr(), depth.data_ptr(), rays.data_ptr())
    return colors, depth, rays


@torch.no_grad()
def fuse_vertex_colors(model: torch.nn.Module, vertices: torch.Tensor, images: torch.Tensor, poses: Sequence,
                       focal: float, near: float, N_samples: int = 64, occ_threshold: float = 0.2,
                       white_back: bool = False, return_opacities: bool = False, *,
                       occupancy: Optional[OccupancyGrid] = None, early_stop: float = 0.0):
    """extract_color_mesh.py:206-284 (the default colour-averaging method) on the device.

    vertices (V, 3) fp32 world; images (n_views, H, W, 3) uint8 CUDA; poses: n_views (3, 4) camera-to-world;
    focal: the dataset focal (K is float32 with principal point (W/2, H/2)); near: ``dataset.bounds.min()``.
    Per view: project + bilinear sample + occlusion rays, the fused ``render_rays`` with ``model`` as the only
    network (N_importance = 0, test_time), and a float64 accumulation in view order.  Returns (V, 3) uint8
    (and the per-view opacities (n_views, V) when ``return_opacities``).

    ``occupancy``: each view's occlusion rays are rendered by ``render_rays_culled(..., skip="samples")`` on that grid
    instead, so density in cells it calls empty does not occlude a vertex.

    ``early_stop`` = eps > 0 (needs ``occupancy``) stops each occlusion ray once it is opaque (DESIGN.md §10f).  A cut
    ray has T_cut < eps, so its terminated and its full opacity both exceed ``1 - eps - 4e-6``: for
    ``eps <= 1 - occ_threshold - 1e-5`` no ``opacity < occ_threshold`` decision changes and the colours are
    bit-identical to ``early_stop = 0``; the opacities move by at most ``T_cut (1 + N_samples 1e-10) + 4e-6``.
    With ``N_samples = 32`` there is nothing to stop."""
    eps = check_early_stop(early_stop, occupancy is not None, 0)
    v = _cuda(vertices, "vertices").detach().to(torch.float32).contiguous()
    if occupancy is not None:
        _check_occupancy(occupancy, _device_of(model))
    imgs = _cuda(images, "images").contiguous()
    if imgs.dtype != torch.uint8 or imgs.dim() != 4 or imgs.shape[3] != 3:
        raise ValueError("images must be (n_views, H, W, 3) uint8")
    if len(poses) != imgs.shape[0]:
        raise ValueError("one pose per image")
    n = v.shape[0]
    sum4 = torch.zeros(n, 4, dtype=torch.float64, device=v.device)
    emb = [Embedding(3, 10), Embedding(3, 4)]
    opac = []
    for idx in range(imgs.shape[0]):
        colors, depth, rays = project_view(v, imgs[idx], poses[idx], focal, near)
        if occupancy is None:
            res = render_rays([model], emb, rays, N_samples, False, 0, 0, 0, 1024 * 32, white_back, test_time=True,
                              match_reference_rng=False)
        else:
            res = render_rays_culled([model], emb, rays, occupancy, N_samples, False, 0, white_back, True,
                                     skip="samples", early_stop=eps)
        opacity = res["opacity_coarse"].contiguous()
        if return_opacities:
            opac.append(opacity)
        _lib.call("nerfb200_color_accumulate", v.device, colors.data_ptr(), depth.data_ptr(), opacity.data_ptr(), n,
                  float(np.float32(occ_threshold)), sum4.data_ptr())
    out = torch.empty(n, 3, dtype=torch.uint8, device=v.device)
    _lib.call("nerfb200_color_finalize", v.device, sum4.data_ptr(), n, out.data_ptr())
    if return_opacities:
        return out, (torch.stack(opac) if opac else torch.empty(0, n, device=v.device))
    return out


def _mesh_vertices(vertices: torch.Tensor) -> torch.Tensor:
    v = _cuda(vertices, "vertices")
    if v.dim() != 2 or v.shape[1] != 3 or not v.is_floating_point():
        raise ValueError("vertices must be (V, 3) floating point")
    return v.detach().to(torch.float32).contiguous()


@torch.no_grad()
def vertex_normals(vertices: torch.Tensor, triangles: torch.Tensor) -> torch.Tensor:
    """Drop-in for ``np.asarray(mesh.compute_vertex_normals().vertex_normals)`` (extract_color_mesh.py:189-190) on a
    mesh without normals: (V, 3) float64 on the device, open3d's definition bit for bit (DESIGN.md "Vertex-normal
    colours").  vertices (V, 3) are taken in float32, the precision the reference's PLY round trip leaves them in;
    triangles (T, 3) integer.  An index outside [0, V) raises ValueError."""
    v = _mesh_vertices(vertices)
    t = _cuda(triangles, "triangles")
    if t.dim() != 2 or t.shape[1] != 3 or t.is_floating_point() or t.is_complex() or t.dtype == torch.bool:
        raise ValueError("triangles must be (T, 3) integer")
    if t.device != v.device:
        raise ValueError("vertices and triangles must be on the same device")
    n_v, n_t = v.shape[0], t.shape[0]
    if t.dtype != torch.int32:
        # an index beyond int32 stays out of range through the cast
        t = t.to(torch.int64).clamp(-1, n_v)
    t = t.detach().to(torch.int32).contiguous()
    nbytes = _lib.load().nerfb200_vertex_normals_workspace_bytes(n_v, n_t)
    if nbytes == 0:
        raise ValueError(f"vertex_normals: unsupported mesh size (V = {n_v}, T = {n_t})")
    out = torch.empty(n_v, 3, dtype=torch.float64, device=v.device)
    ws = _lib.workspace(nbytes, v.device)
    _lib.call("nerfb200_vertex_normals", v.device, v.data_ptr(), n_v, t.data_ptr(), n_t, ws.data_ptr(), ws.numel(),
              out.data_ptr())
    return out


@torch.no_grad()
def normal_rays(vertices: torch.Tensor, normals: torch.Tensor, near: float, far: float,
                near_t: float = 1.0) -> torch.Tensor:
    """extract_color_mesh.py:190-193 on the device: (V, 8) float32 rays ``[v - d * near * near_t, d, near, far]`` with
    ``d = float32(normals)``, bit for bit the reference's CPU torch expression (``near``, ``far`` and ``near_t``
    rounded to float32 as torch rounds them)."""
    v = _mesh_vertices(vertices)
    n = _cuda(normals, "normals")
    if n.shape != v.shape or not n.is_floating_point():
        raise ValueError("normals must be floating point and shaped like vertices (V, 3)")
    n = n.detach().to(torch.float64).contiguous()
    rays = torch.empty(v.shape[0], 8, dtype=torch.float32, device=v.device)
    _lib.call("nerfb200_normal_rays", v.device, v.data_ptr(), n.data_ptr(), v.shape[0], float(np.float32(near)),
              float(np.float32(far)), float(np.float32(near_t)), rays.data_ptr())
    return rays


@torch.no_grad()
def normal_vertex_colors(nerf_coarse: torch.nn.Module, nerf_fine: torch.nn.Module, vertices: torch.Tensor,
                         triangles: torch.Tensor, near: float, far: float, N_samples: int = 64,
                         N_importance: int = 64, near_t: float = 1.0, white_back: bool = False, *,
                         occupancy: Optional[OccupancyGrid] = None) -> torch.Tensor:
    """extract_color_mesh.py:187-203 and 280-281 (``--use_vertex_normal``) on the device: (V, 3) uint8 vertex colours
    ``(rgb_fine * 255).astype(uint8)`` of rays that start at ``v - n * near * near_t`` and run along the open3d
    vertex normal n.  One ``vertex_normals``, one ``normal_rays``, one fused ``render_rays`` of all V rays with both
    networks (test_time, perturb 0, noise 0), and ``to_uint8``.  near / far: ``dataset.bounds.min()`` / ``.max()``;
    white_back: ``dataset.white_back``.  ``occupancy``: the rays are rendered by ``render_rays_culled(...,
    skip="samples")`` on that grid instead, so density in cells it calls empty does not tint the colours."""
    dev = _device_of(nerf_coarse)
    _device_of(nerf_fine)
    if occupancy is not None:
        _check_occupancy(occupancy, dev)
    if int(N_importance) <= 0:
        raise ValueError("normal_vertex_colors needs N_importance > 0 (the colours are rgb_fine)")
    normals = vertex_normals(vertices, triangles)
    rays = normal_rays(vertices, normals, near, far, near_t)
    emb = [Embedding(3, 10), Embedding(3, 4)]
    if occupancy is None:
        res = render_rays([nerf_coarse, nerf_fine], emb, rays, int(N_samples), False, 0, 0, int(N_importance),
                          1024 * 32, bool(white_back), test_time=True, match_reference_rng=False)
    else:
        res = render_rays_culled([nerf_coarse, nerf_fine], emb, rays, occupancy, int(N_samples), False,
                                 int(N_importance), bool(white_back), True, skip="samples")
    return to_uint8(res["rgb_fine"])


@torch.no_grad()
def query_rgb_sigma(model: torch.nn.Module, xyz: torch.Tensor) -> torch.Tensor:
    """(n, 4) [sigmoid rgb, raw sigma] of ``model`` at positions xyz (n, 3) with the direction (0, 0, 0), one fused
    launch (encoding in-kernel): ``nerf(cat(embedding_xyz(xyz), embedding_dir(zeros)))`` of extract_mesh.ipynb."""
    x = _cuda(xyz, "xyz").detach().to(torch.float32).contiguous()
    if x.dim() != 2 or x.shape[1] != 3:
        raise ValueError("xyz must be (n, 3)")
    out = torch.empty(x.shape[0], 4, dtype=torch.float32, device=x.device)
    blob = packed_weights(model)
    _lib.call("nerfb200_query_rgb_sigma", x.device, x.data_ptr(), x.shape[0], 3, blob.data_ptr(), out.data_ptr())
    return out


@torch.no_grad()
def query_rgb_sh(model: torch.nn.Module, xyz: torch.Tensor) -> torch.Tensor:
    """(n, 28) fp32 of ``model`` at positions xyz (n, 3), one fused launch after a small table launch (DESIGN.md
    §10k): (c_r0, c_g0, c_b0, sigma), then c_{r,g,b; m} for m = 1..8, the degree-2 spherical-harmonic coefficients
    (PlenOctrees' eval_sh basis) fitted by P = pinv(Y) to the sigmoid rgb at 64 fixed directions; sigma is
    ``query_rgb_sigma``'s bit for bit."""
    x = _cuda(xyz, "xyz").detach().to(torch.float32).contiguous()
    if x.dim() != 2 or x.shape[1] != 3:
        raise ValueError("xyz must be (n, 3)")
    out = torch.empty(x.shape[0], 28, dtype=torch.float32, device=x.device)
    blob = packed_weights(model)
    ws = _lib.workspace(_lib.load().nerfb200_query_rgb_sh_workspace_bytes(), x.device)
    _lib.call("nerfb200_query_rgb_sh", x.device, x.data_ptr(), x.shape[0], 3, blob.data_ptr(), ws.data_ptr(),
              ws.numel(), out.data_ptr())
    return out


@torch.no_grad()
def rgb_sigma_grid(model: torch.nn.Module, N: int, x_range, y_range, z_range, chunk: int = 1 << 21, *,
                   occupancy: Optional[OccupancyGrid] = None, return_evaluated: bool = False):
    """(N, N, N, 4) fp32 [sigmoid rgb, raw sigma] of ``model`` on the grid of ``sigma_grid`` with the direction
    (0, 0, 0): extract_mesh.ipynb's ``rgbsigma`` ("Search for tight bounds"), reshaped.  Raw sigma: no
    ``max(sigma, 0)``.  ``chunk`` points are queried per launch; the scratch is their positions only.

    ``occupancy`` and ``return_evaluated`` as for ``sigma_grid``: an evaluated point gets the four channels above bit
    for bit, every other point (0, 0, 0, 0), which ``pack_volume`` drops (alpha 0)."""
    if occupancy is not None:
        if not 2 <= int(N) <= 1625:
            raise ValueError(f"rgb_sigma_grid: N = {N} outside [2, 1625]")
        out, evaluated = _masked_grid("nerfb200_rgb_sigma_grid_masked", model, int(N),
                                      _lib.ranges_host(x_range, y_range, z_range), occupancy, chunk, 4)
        return (out, evaluated) if return_evaluated else out
    dev = _device_of(model)
    out = torch.empty(N, N, N, 4, dtype=torch.float32, device=dev)
    blob = packed_weights(model)
    chunk = int(min(chunk, N ** 3))
    ws = _lib.workspace(_lib.load().nerfb200_sigma_grid_workspace_bytes(chunk), dev)
    _lib.call("nerfb200_rgb_sigma_grid", dev, blob.data_ptr(), N, _lib.ranges_host(x_range, y_range, z_range), chunk,
              ws.data_ptr(), ws.numel(), out.data_ptr())
    return (out, N ** 3) if return_evaluated else out


@torch.no_grad()
def pack_volume(rgbsigma: torch.Tensor, x_range) -> torch.Tensor:
    """extract_mesh.ipynb "Generate .vol file for volume rendering in Unity" on a CUDA (N, N, N, 4) rgbsigma grid
    (raw sigma): (M, 2) uint32 rows [i, r << 24 + g << 16 + b << 8 + a8] of the points with alpha > 0, in
    increasing flat index i, where a = 1 - exp(float32(-(xmax - xmin) / N) * max(sigma, 0)) (float32, exp
    correctly rounded), a8 = trunc(255 a) and r = trunc(255 rgb).  Only ``x_range`` enters alpha, as in the
    notebook.  N <= 1625 (the indices are uint32)."""
    g = _cuda(rgbsigma, "rgbsigma").detach().to(torch.float32).contiguous()
    if g.dim() == 4 and g.shape[3] == 28:
        raise ValueError("pack_volume: a view-dependent (N, N, N, 28) grid has no .vol form; the Unity file holds the "
                         "direction-0 colour of an (N, N, N, 4) grid")
    if g.dim() != 4 or g.shape[3] != 4 or not (g.shape[0] == g.shape[1] == g.shape[2]):
        raise ValueError("rgbsigma must be (N, N, N, 4)")
    N = g.shape[0]
    xmin, xmax = (float(v) for v in x_range)
    nbytes = _lib.load().nerfb200_volume_workspace_bytes(N)
    if nbytes == 0:
        raise ValueError(f"pack_volume: N = {N} outside [2, 1625]")
    ws = _lib.workspace(nbytes, g.device)
    count = ctypes.c_int64()
    _lib.call("nerfb200_volume_count", g.device, g.data_ptr(), N, xmin, xmax, ws.data_ptr(), ws.numel(),
              ctypes.byref(count))
    # torch has no uint32 arithmetic to speak of; the rows are stored as int32 and viewed as uint32
    out = torch.empty(count.value, 2, dtype=torch.int32, device=g.device)
    if count.value:
        _lib.call("nerfb200_volume_emit", g.device, g.data_ptr(), N, xmin, xmax, ws.data_ptr(), ws.numel(),
                  out.data_ptr())
    return out.view(torch.uint32)


def write_vol(path: str, packed) -> None:
    """The .vol file of extract_mesh.ipynb: the (M, 2) uint32 rows of ``pack_volume`` as little-endian uint32,
    row by row (``res.tobytes()``)."""
    a = packed.detach().cpu().numpy() if isinstance(packed, torch.Tensor) else np.asarray(packed)
    with open(path, "wb") as f:
        f.write(np.ascontiguousarray(a.reshape(-1), dtype="<u4").tobytes())


def write_ply(path: str, vertices, triangles, colors=None) -> None:
    """The binary little-endian PLY plyfile writes at extract_color_mesh.py:286-297: element ``vertex`` with
    float ``x y z`` (and uchar ``red green blue``), element ``face`` with ``list uchar int vertex_indices``."""
    def host(a):
        return a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)

    v = host(vertices).astype(np.float32).reshape(-1, 3)
    t = host(triangles).astype(np.int32).reshape(-1, 3)
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    if colors is not None:
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    vert = np.empty(len(v), dtype=fields)
    vert["x"], vert["y"], vert["z"] = v[:, 0], v[:, 1], v[:, 2]
    if colors is not None:
        c = host(colors).astype(np.uint8).reshape(-1, 3)
        vert["red"], vert["green"], vert["blue"] = c[:, 0], c[:, 1], c[:, 2]
    face = np.empty(len(t), dtype=[("n", "u1"), ("vertex_indices", "<i4", (3,))])
    face["n"] = 3
    face["vertex_indices"] = t
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {len(v)}"]
    head += [f"property float {k}" for k in ("x", "y", "z")]
    if colors is not None:
        head += [f"property uchar {k}" for k in ("red", "green", "blue")]
    head += [f"element face {len(t)}", "property list uchar int vertex_indices", "end_header"]
    with open(path, "wb") as f:
        f.write(("\n".join(head) + "\n").encode("ascii"))
        f.write(vert.tobytes())
        f.write(face.tobytes())
