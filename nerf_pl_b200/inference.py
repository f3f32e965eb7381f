"""Full-image inference driver (SURVEY.md section 8f rows 1-2): on-GPU ray generation, one fused render
launch per image (optionally ray-sharded across ranks), uint8 conversion on the device.

Mirrors the reference's eval path: ``datasets/ray_utils.py`` (get_ray_directions / get_rays /
get_ndc_rays), ``eval.py:58-86`` batched_inference and ``eval.py:119-128`` (reshape + uint8).
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional, Sequence

import torch

from . import _lib
from .culling import OccupancyGrid, check_early_stop, check_skip, render_culled, render_culled_samples, result_keys
from .nerf import packed_weights
from .rendering import render_rays
from .sharded import render_rays_sharded


def generate_rays(H: int, W: int, focal: float, c2w, near: float, far: float, ndc: bool = False,
                  device: Optional[torch.device] = None) -> torch.Tensor:
    """(H*W, 8) rays [o, d, near, far] for a pinhole camera, built on the GPU.
    c2w: (3,4) camera-to-world (any array-like / tensor).  ``ndc=True`` applies the forward-facing
    NDC warp exactly as datasets/llff.py:236-241 does (near plane 1.0, near/far columns 0/1)."""
    device = torch.device("cuda") if device is None else torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("nerf_pl_b200.generate_rays runs on CUDA only (no CPU fallback)")
    c2w_t = torch.as_tensor(c2w, dtype=torch.float32).reshape(-1).cpu()
    if c2w_t.numel() != 12:
        raise ValueError("c2w must be (3, 4)")
    arr = (ctypes.c_float * 12)(*c2w_t.tolist())
    rays = torch.empty(H * W, 8, dtype=torch.float32, device=device)
    _lib.call("nerfb200_generate_rays", device, H, W, float(focal), arr, float(near), float(far), int(bool(ndc)),
              rays.data_ptr())
    return rays


def to_uint8(img: torch.Tensor) -> torch.Tensor:
    """(clip(img, 0, 1) * 255).astype(uint8) on the device (eval.py:126-128)."""
    if not img.is_cuda:
        raise RuntimeError("nerf_pl_b200.to_uint8 runs on CUDA tensors only (no CPU fallback)")
    src = img.detach().to(torch.float32).contiguous()
    dst = torch.empty(src.shape, dtype=torch.uint8, device=src.device)
    _lib.call("nerfb200_to_uint8", src.device, src.data_ptr(), src.numel(), dst.data_ptr())
    return dst


@torch.no_grad()
def batched_inference(models: Sequence[torch.nn.Module], embeddings: Sequence[torch.nn.Module],
                      rays: torch.Tensor, N_samples: int, N_importance: int, use_disp: bool,
                      chunk: int = 1024 * 32, white_back: bool = False, sharded: bool = False, skip: str = "rays", *,
                      early_stop: float = 0.0, occupancy: Optional[OccupancyGrid] = None) -> Dict[str, torch.Tensor]:
    """Drop-in for eval.py:58-86 batched_inference(models, embeddings, rays, N_samples,
    N_importance, use_disp, chunk, white_back): perturb=0, noise_std=0, test_time=True.  The
    reference loops over 32768-ray chunks and concatenates; here the whole image is one launch
    (``chunk`` is ignored).  ``sharded=True`` splits the rays over the ranks of the default process
    group and all-gathers the result (nerf_pl_b200.sharded).  ``occupancy`` (an ``nb.occupancy_grid``; default None:
    every ray is rendered) skips empty space: only the rays that cross an occupied cell are rendered, the others
    get the vacuum value, and the result also holds ``'live'`` and ``'live_idx'`` (nerf_pl_b200.culling, which also
    says what that does and does not guarantee).  With ``sharded`` the live rays are what is split, so the ranks
    get equal work.  ``skip="samples"`` (needs ``occupancy``; pass both by keyword) also skips the empty samples of
    the live rays and adds ``'live_samples'`` (nerf_pl_b200.culling).  ``early_stop`` and ``occupancy`` are
    keyword-only.  ``early_stop`` = eps > 0 (``skip="samples"``, ``N_importance = 0``)
    stops each ray once it is opaque, within a stated bound (``render_rays_culled``; DESIGN.md §10f); with
    ``N_samples = 32`` there is nothing to stop."""
    del chunk
    check_skip(skip, occupancy)
    eps = check_early_stop(early_stop, skip == "samples", N_importance)
    if skip == "samples":
        from .rendering import _check_render_inputs
        _check_render_inputs("batched_inference", models, embeddings, int(N_importance), rays)
        return render_culled_samples(list(models), rays, occupancy, int(N_samples), use_disp, int(N_importance),
                                     white_back, True, sharded=sharded, early_stop=eps)

    def fn(r):
        # eval never consumes the reference's noise draws: do not materialise them for a whole image
        return render_rays(list(models), list(embeddings), r, N_samples, use_disp, 0, 0, N_importance,
                           1024 * 32, white_back, test_time=True, match_reference_rng=False)

    run = (lambda r: render_rays_sharded(fn, r)) if sharded else fn
    if occupancy is None:
        return run(rays)
    return render_culled(run, rays, occupancy, result_keys(int(N_importance), True), bool(white_back))


@torch.no_grad()
def render_image(models, embeddings, H: int, W: int, focal: float, c2w, near: float, far: float,
                 N_samples: int = 64, N_importance: int = 64, use_disp: bool = False, white_back: bool = False,
                 ndc: bool = False, sharded: bool = False, device=None, skip: str = "rays",
                 *, early_stop: float = 0.0, occupancy: Optional[OccupancyGrid] = None) -> Dict[str, torch.Tensor]:
    """Pose -> rays -> fused render -> (H, W, 3) uint8 image + float maps, all on the device
    (test.ipynb cell 2 / eval.py:117-128).  ``occupancy``, ``skip`` and ``early_stop``: as for ``batched_inference``;
    the result then also holds ``'live'`` (and ``'live_samples'`` with ``skip="samples"``)."""
    check_skip(skip, occupancy)
    eps = check_early_stop(early_stop, skip == "samples", N_importance)
    rays = generate_rays(H, W, focal, c2w, near, far, ndc=ndc, device=device)
    res = batched_inference(models, embeddings, rays, N_samples, N_importance, use_disp, 1024 * 32, white_back,
                            sharded=sharded, occupancy=occupancy, skip=skip, early_stop=eps)
    typ = "fine" if N_importance > 0 else "coarse"
    out = {"rays": rays, "opacity": res[f"opacity_{typ}"].view(H, W)}
    if f"rgb_{typ}" in res:
        out["rgb"] = res[f"rgb_{typ}"].view(H, W, 3)
        out["depth"] = res[f"depth_{typ}"].view(H, W)
        out["rgb_uint8"] = to_uint8(out["rgb"])
    if occupancy is not None:
        out["live"] = res["live"]
    if skip == "samples":
        out["live_samples"] = res["live_samples"]
    return out


@torch.no_grad()
def query_sigma(model: torch.nn.Module, xyz: torch.Tensor) -> torch.Tensor:
    """Raw sigma at positions xyz (N,3) with one fused launch (encoding in-kernel, sigma-only MLP).
    Equivalent to extract_color_mesh.py:127-140 `nerf(cat(embedding_xyz(x), embedding_dir(0)))[:, -1]`."""
    if not xyz.is_cuda or xyz.dim() != 2 or xyz.shape[1] != 3:
        raise ValueError("xyz must be a (N, 3) CUDA tensor")
    x = xyz.detach().to(torch.float32).contiguous()
    out = torch.empty(x.shape[0], dtype=torch.float32, device=x.device)
    blob = packed_weights(model)
    _lib.call("nerfb200_query_sigma", x.device, x.data_ptr(), x.shape[0], 3, blob.data_ptr(), out.data_ptr())
    return out


@torch.no_grad()
def mse_psnr(results: Dict[str, torch.Tensor], targets: torch.Tensor) -> Dict[str, torch.Tensor]:
    """losses.py:9-14 MSELoss + metrics.py:12-13 psnr of a render_rays result in one launch.
    Returns {'loss': mse_coarse (+ mse_fine), 'psnr': of rgb_fine if present else rgb_coarse}."""
    rc, rf = results.get("rgb_coarse"), results.get("rgb_fine")
    ref = rf if rf is not None else rc
    if ref is None:
        raise ValueError("results must hold CUDA rgb_coarse and/or rgb_fine")
    # the C entry takes its row count from targets: every shape is checked here, before anything is launched
    if targets.dim() != 2 or targets.shape[1] != 3:
        raise ValueError(f"targets must be (N_rays, 3), got {tuple(targets.shape)}")
    for name, v in (("rgb_coarse", rc), ("rgb_fine", rf)):
        if v is not None and v.shape != targets.shape:
            raise ValueError(f"{name} must have the shape of targets {tuple(targets.shape)}, got {tuple(v.shape)}")
    if not ref.is_cuda:
        raise ValueError("results must hold CUDA rgb_coarse and/or rgb_fine")
    t = targets.detach().to(torch.float32).contiguous()
    out = torch.empty(4, dtype=torch.float32, device=ref.device)
    keep = [None if v is None else v.detach().float().contiguous() for v in (rc, rf)]
    _lib.call("nerfb200_mse_psnr", ref.device, None if keep[0] is None else keep[0].data_ptr(),
              None if keep[1] is None else keep[1].data_ptr(), t.data_ptr(), t.shape[0], out.data_ptr())
    return {"loss": out[2] if rc is not None else out[1], "psnr": out[3], "mse_coarse": out[0], "mse_fine": out[1]}
