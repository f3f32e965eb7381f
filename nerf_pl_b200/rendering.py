"""``render_rays`` with the reference's exact signature and result keys
(reference: models/rendering.py:58-244), executed by one fused sm_90a kernel launch.

Also exposes the pieces the reference exposes or depends on, each through the C ABI:
``sample_pdf`` (models/rendering.py:14-55), ``searchsorted`` (torchsearchsorted
searchsorted.py:20-53), ``volume_render`` (models/rendering.py:143-170).
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional, Sequence

import torch

from . import _lib
from .nerf import nerf_forward_torch, packed_weights

__all__ = ["render_rays", "render_rays_host", "render_rays_loss", "sample_pdf", "searchsorted", "volume_render"]


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _require_fp32(name: str, *tensors) -> None:
    """The kernels compute in fp32 (the reference's dtype, SURVEY App. A.19).  torchsearchsorted also
    accepts float64 and keeps it; silently rounding such inputs would change results, so they are
    rejected instead."""
    for t in tensors:
        if t is not None and t.dtype == torch.float64:
            raise ValueError(f"nerf_pl_b200.{name} computes in float32; got a float64 tensor (convert it explicitly)")


_EMB_OK = set()


def _check_embeddings(embeddings: Sequence) -> None:
    ex, ed = embeddings[0], embeddings[1]
    if (id(ex), id(ed)) in _EMB_OK:          # validated before (reading freq_bands costs a host sync-free but slow .item())
        return
    ok = (getattr(ex, "N_freqs", None) == 10 and getattr(ed, "N_freqs", None) == 4
          and getattr(ex, "in_channels", 3) == 3 and getattr(ed, "in_channels", 3) == 3)
    fb = getattr(ex, "freq_bands", None)
    if ok and fb is not None and len(fb) == 10:
        ok = abs(float(fb[-1]) - 512.0) < 1e-3
    if not ok:
        raise ValueError("nerf_pl_b200.render_rays supports the reference's embeddings "
                         "Embedding(3, 10) / Embedding(3, 4) with logscale=True")
    if len(_EMB_OK) < 64:
        _EMB_OK.add((id(ex), id(ed)))


def _check_render_inputs(name: str, models, embeddings, N_importance: int, rays: Optional[torch.Tensor]) -> None:
    """The argument checks of render_rays, render_rays_loss and render_rays_host (``name``, the public function the
    messages name).  ``rays`` are device rays; None for render_rays_host, which checks its host rays itself."""
    if rays is not None:
        if rays.dim() != 2 or rays.shape[1] != 8:
            raise ValueError("rays must be (N_rays, 8)")
        if not rays.is_cuda:
            raise RuntimeError(f"nerf_pl_b200.{name} runs on CUDA tensors only (no CPU fallback)")
    _check_embeddings(embeddings)
    if N_importance > 0 and len(models) < 2:
        raise ValueError("N_importance > 0 needs a fine model (models[1])")


def searchsorted(a: torch.Tensor, v: torch.Tensor, out: Optional[torch.Tensor] = None,
                 side: str = "left") -> torch.Tensor:
    """Row-wise batched binary search; same contract as torchsearchsorted.searchsorted
    (searchsorted.py:20-53): 2-D inputs, equal row counts or one of them with a single row,
    int64 result of shape (max rows, v columns)."""
    assert len(a.shape) == 2, "input `a` must be 2-D."
    assert len(v.shape) == 2, "input `v` mus(t) be 2-D."
    assert (a.shape[0] == v.shape[0]) or (a.shape[0] == 1) or (v.shape[0] == 1), \
        "`a` and `v` must have the same number of rows or one of them must have only 1 row"
    assert a.device == v.device, "`a` and `v` must be on the same device"
    if side not in ("left", "right"):
        raise ValueError("side must be 'left' or 'right'")
    if not a.is_cuda:
        raise RuntimeError("nerf_pl_b200.searchsorted runs on CUDA tensors only (no CPU fallback)")
    _require_fp32("searchsorted", a, v)
    nrow = max(a.shape[0], v.shape[0])
    if out is None:
        out = torch.empty(nrow, v.shape[1], dtype=torch.long, device=v.device)
    else:
        assert out.shape == (nrow, v.shape[1]) and out.dtype == torch.long and out.is_contiguous()
    ac = a.to(torch.float32).contiguous()
    vc = v.to(torch.float32).contiguous()
    _lib.call("nerfb200_searchsorted", a.device, ac.data_ptr(), vc.data_ptr(), out.data_ptr(), ac.shape[0],
              vc.shape[0], ac.shape[1], vc.shape[1], 1 if side == "right" else 0)
    return out


def sample_pdf(bins: torch.Tensor, weights: torch.Tensor, N_importance: int, det: bool = False,
               eps: float = 1e-5, u: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Inverse-CDF sampling of ``N_importance`` depths per ray (reference models/rendering.py:14-55).
    ``u`` may be given to reproduce a specific random draw."""
    if abs(eps - 1e-5) > 1e-12:
        raise ValueError("nerf_pl_b200.sample_pdf implements the reference default eps=1e-5")
    # the C entry gets only sizes: every shape is checked here, before anything is launched
    if weights.dim() != 2:
        raise ValueError("weights must be (N_rays, N_samples_)")
    n_rays, n_w = weights.shape
    if tuple(bins.shape) != (n_rays, n_w + 1):
        raise ValueError("bins must be (N_rays, N_samples_+1)")
    if u is not None and tuple(u.shape) != (n_rays, N_importance):
        raise ValueError(f"u must be (N_rays, N_importance) = ({n_rays}, {N_importance}), got {tuple(u.shape)}")
    if not bins.is_cuda:
        raise RuntimeError("nerf_pl_b200.sample_pdf runs on CUDA tensors only (no CPU fallback)")
    _require_fp32("sample_pdf", bins, weights, u)
    if u is None:
        if det:
            u = torch.linspace(0, 1, N_importance, device=bins.device).expand(n_rays, N_importance)
        else:
            u = torch.rand(n_rays, N_importance, device=bins.device)
    u = u.to(torch.float32).contiguous()
    out = torch.empty(n_rays, N_importance, dtype=torch.float32, device=bins.device)
    bc, wc = bins.to(torch.float32).contiguous(), weights.detach().to(torch.float32).contiguous()
    _lib.call("nerfb200_sample_pdf", bins.device, bc.data_ptr(), wc.data_ptr(), u.data_ptr(), n_rays, n_w,
              N_importance, out.data_ptr())
    return out


def volume_render(sigmas: torch.Tensor, rgbs: Optional[torch.Tensor], z_vals: torch.Tensor,
                  dirs: torch.Tensor, noise: Optional[torch.Tensor] = None, noise_std: float = 0.0,
                  white_back: bool = False):
    """Alpha-compositing quadrature (reference models/rendering.py:143-170).
    Returns (weights, rgb | None, depth | None, opacity)."""
    # the C entry gets only sizes: every shape is checked here, before anything is launched
    if sigmas.dim() != 2:
        raise ValueError("sigmas must be (N_rays, N_samples)")
    n, S = sigmas.shape
    for name, t, shape in (("rgbs", rgbs, (n, S, 3)), ("z_vals", z_vals, (n, S)), ("dirs", dirs, (n, 3)),
                           ("noise", noise, (n, S))):
        if t is not None and tuple(t.shape) != shape:
            raise ValueError(f"{name} must be {shape} for sigmas of shape {(n, S)}, got {tuple(t.shape)}")
    if not sigmas.is_cuda:
        raise RuntimeError("nerf_pl_b200.volume_render runs on CUDA tensors only (no CPU fallback)")
    _require_fp32("volume_render", sigmas, rgbs, z_vals, dirs, noise)
    dev = sigmas.device
    f32 = dict(dtype=torch.float32, device=dev)
    weights = torch.empty(n, S, **f32)
    opac = torch.empty(n, **f32)
    rgb = torch.empty(n, 3, **f32) if rgbs is not None else None
    depth = torch.empty(n, **f32) if rgbs is not None else None
    keep = [sigmas.float().contiguous(), None if rgbs is None else rgbs.float().contiguous(),
            z_vals.float().contiguous(), dirs.float().contiguous(),
            None if noise is None else noise.float().contiguous()]
    _lib.call("nerfb200_composite", dev, _ptr(keep[0]), _ptr(keep[1]), _ptr(keep[2]), _ptr(keep[3]), _ptr(keep[4]),
              float(noise_std), int(bool(white_back)), n, S, weights.data_ptr(), _ptr(rgb), _ptr(depth), opac.data_ptr())
    return weights, rgb, depth, opac


def _draw_randoms(n: int, S_c: int, K: int, perturb: float, noise_std: float, device, match_rng: bool):
    """Draw the random inputs in the order the reference consumes the global torch RNG
    (models/rendering.py:203 rand, :152 randn, :39 rand, :152 randn) so a seeded run sees the
    same numbers.  With ``match_rng`` the unused randn draws (noise_std == 0) are still made, as
    the reference does."""
    pr = nc = ur = nf = None
    if perturb > 0 and K > 0 and not match_rng and noise_std <= 0:
        # no promise about the draw order: both uniform tensors from ONE generator launch
        flat = torch.rand(n * (S_c + K), device=device)
        return flat[:n * S_c].view(n, S_c), None, flat[n * S_c:].view(n, K), None
    if perturb > 0:
        pr = torch.rand(n, S_c, device=device)
    if noise_std > 0 or match_rng:
        nc = torch.randn(n, S_c, device=device)
    if K > 0:
        if perturb > 0:
            ur = torch.rand(n, K, device=device)
        if noise_std > 0 or match_rng:
            nf = torch.randn(n, S_c + K, device=device)
    if noise_std <= 0:
        nc = nf = None
    return pr, nc, ur, nf


_KERNEL_RNG_CALLS = 0


def _seed_fields(seed) -> Dict[str, int]:
    """The RenderArgs fields of a kernel seed: None (tensor inputs), an int, or a device int64 tensor holding it
    (rng_in_kernel == 2: the kernel reads the key at that address)."""
    if seed is None:
        return dict(rng_seed=0, rng_in_kernel=0)
    if torch.is_tensor(seed):
        return dict(rng_seed=seed.data_ptr(), rng_in_kernel=2)
    return dict(rng_seed=seed, rng_in_kernel=1)


def _render_args(rays, S_c: int, K: int, use_disp, perturb: float, noise_std: float, white_back, test_time,
                 packed, randoms, outs: Dict[str, Optional[torch.Tensor]], seed, workspace=None, target=None,
                 loss_out=None) -> _lib.RenderArgs:
    """The ``nerfb200_render_args`` of one render.  ``packed``: the (coarse, fine | None) weight images; ``randoms``:
    (perturb_rand, noise_coarse, u_rand, noise_fine), each None when not drawn; ``outs``: output tensors keyed by field
    name; ``workspace``: a training workspace.  Every field not given is zero / NULL."""
    pr, nc, ur, nf = randoms
    return _lib.RenderArgs(
        rays=rays.data_ptr(), n_rays=rays.shape[0], ray_stride=rays.stride(0),
        packed_coarse=packed[0].data_ptr(), packed_fine=_ptr(packed[1]),
        n_samples=S_c, n_importance=K, use_disp=int(bool(use_disp)), perturb=perturb, noise_std=noise_std,
        white_back=int(bool(white_back)), test_time=int(bool(test_time)),
        perturb_rand=_ptr(pr), noise_coarse=_ptr(nc), u_rand=_ptr(ur), noise_fine=_ptr(nf),
        train_workspace=None if workspace is None else workspace.buf.data_ptr(), target=_ptr(target),
        loss_out=_ptr(loss_out), **{k: _ptr(t) for k, t in outs.items()}, **_seed_fields(seed))


def _resolve_randoms(randoms, n, S_c, K, perturb, noise_std, dev, match_rng):
    """-> (perturb_rand, noise_coarse, u_rand, noise_fine, kernel_seed | None).

    ``randoms`` is None (draw with torch as the reference does), a dict of pre-drawn tensors, the string
    ``"kernel"`` or ``{"seed": int}``: the two uniform inputs are then generated inside the render kernel
    (Philox4x32-10 keyed by the seed, include/nerf_pl_b200.h ``rng_in_kernel``) - no generator launch, no (N, S)
    tensors.  ``"kernel"`` derives the seed from ``torch.initial_seed()`` and a per-process call counter
    (deterministic under ``torch.manual_seed``).  Because that seed is a host value, ``"kernel"`` is refused while
    a CUDA graph is being captured (a replay would reuse it); there ``{"seed": t}`` with ``t`` a one-element int64
    CUDA tensor keys the numbers from device memory (its 64 bits are the seed; ``CapturedTrainStep`` advances it
    inside the graph).  The Gaussian noise inputs (``noise_std > 0``) are tensors in every mode."""
    global _KERNEL_RNG_CALLS
    seed = None
    if isinstance(randoms, str):
        if randoms != "kernel":
            raise ValueError("randoms must be None, a dict of tensors, {'seed': int} or 'kernel'")
        if torch.cuda.is_initialized() and torch.cuda.is_current_stream_capturing():
            raise ValueError("randoms='kernel' derives its seed on the host, so a captured graph would replay one "
                             "seed: pass {'seed': <int64 CUDA tensor>} or use nerf_pl_b200.CapturedTrainStep")
        _KERNEL_RNG_CALLS += 1
        seed = (torch.initial_seed() * 0x9E3779B97F4A7C15 + _KERNEL_RNG_CALLS * 0xD1B54A32D192ED03) & 0xFFFFFFFFFFFFFFFF
        randoms = {}
    elif randoms is not None and "seed" in randoms:
        seed = randoms["seed"]
        if torch.is_tensor(seed):
            if not (seed.is_cuda and seed.dtype == torch.int64 and seed.numel() == 1 and seed.device == dev):
                raise ValueError("a tensor seed must be a one-element int64 tensor on the rays' device")
        else:
            seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    if randoms is None:
        pr, nc, ur, nf = _draw_randoms(n, S_c, K, perturb, noise_std, dev, match_rng)
    else:
        pr, nc = randoms.get("perturb_rand"), randoms.get("noise_coarse")
        ur, nf = randoms.get("u_rand"), randoms.get("noise_fine")
        if seed is not None:
            pr = ur = None
            if noise_std > 0:
                if nc is None:
                    nc = torch.randn(n, S_c, device=dev)
                if nf is None and K > 0:
                    nf = torch.randn(n, S_c + K, device=dev)
    pr, nc, ur, nf = [t.to(torch.float32).contiguous() if t is not None else None for t in (pr, nc, ur, nf)]
    return pr, nc, ur, nf, seed


def render_rays(models: List[torch.nn.Module],
                embeddings: List[torch.nn.Module],
                rays: torch.Tensor,
                N_samples: int = 64,
                use_disp: bool = False,
                perturb: float = 0,
                noise_std: float = 1,
                N_importance: int = 0,
                chunk: int = 1024 * 32,
                white_back: bool = False,
                test_time: bool = False,
                *,
                randoms: Optional[Dict[str, torch.Tensor]] = None,
                match_reference_rng: bool = True,
                extras: bool = False,
                autograd_impl: str = "fused",
                occupancy=None) -> Dict[str, torch.Tensor]:
    """Render rays with the coarse (and fine) NeRF.  Drop-in for reference
    ``models.rendering.render_rays`` (models/rendering.py:58-244): same positional arguments,
    defaults and result keys/shapes/dtypes:

    * ``test_time=False``: ``rgb_coarse (N,3)``, ``depth_coarse (N)``, ``opacity_coarse (N)``
    * ``test_time=True`` : ``opacity_coarse`` only for the coarse pass
    * ``N_importance>0`` : additionally ``rgb_fine``, ``depth_fine``, ``opacity_fine``

    ``chunk`` is accepted and ignored (nothing is materialised per point, so there is nothing to
    chunk).  Keyword-only extensions: ``randoms`` supplies pre-drawn ``perturb_rand``,
    ``noise_coarse``, ``u_rand``, ``noise_fine`` tensors, or ``"kernel"`` / ``{"seed": s}`` to draw the uniform
    numbers inside the kernel (``_resolve_randoms``); ``extras=True`` adds ``z_vals_fine``,
    ``weights_coarse``, ``weights_fine`` to the result.  When a gradient graph is needed the
    result comes from ``nerf_pl_b200.training.FusedRenderFunction`` (fused forward with activation
    capture + hand-written backward); ``autograd_impl="torch"`` selects the plain torch-op
    evaluation instead (the gradient reference used by the tests).

    ``occupancy`` (a ``nerf_pl_b200.OccupancyGrid``; for a ``DensityGrid`` pass its ``.grid``) skips empty samples
    with ``skip="samples"``'s rule (DESIGN.md "Training with empty samples skipped"): a sample in no occupied cell
    gets sigma = 0 and no noise, is not evaluated, has weight exactly 0 and receives no gradient.  Every ray is
    rendered.  With a gradient graph (``train_skip.render_rays_train_skip``) every returned key is differentiable,
    the values are ``render_rays_loss(..., occupancy=)``'s for the same randoms, and neither the forward nor the
    backward synchronises; it needs ``test_time=False``, ``extras=False``, ``autograd_impl="fused"`` and the shapes
    of ``train_skip.check_shape`` (ValueError otherwise).  Without one (validation, evaluation) the rays go through
    ``culling.render_samples`` with the same randoms, giving the same values bit for bit.
    """
    del chunk
    if autograd_impl not in ("fused", "torch"):
        raise ValueError("autograd_impl must be 'fused' or 'torch'")
    needs_graph = torch.is_grad_enabled() and any(
        p.requires_grad for m in models[:2] for p in m.parameters())
    if occupancy is not None:
        _check_grid_call(occupancy, rays, int(N_samples), int(N_importance), needs_graph, test_time, extras,
                         autograd_impl)
    _check_render_inputs("render_rays", models, embeddings, N_importance, rays)
    if occupancy is not None and rays.shape[0] > 0:
        from .train_skip import check_grid
        check_grid(occupancy, rays)

    dev = rays.device
    n = rays.shape[0]
    S_c, K = int(N_samples), int(N_importance)
    S_f = S_c + K
    rays_c = rays.detach().to(torch.float32).contiguous()
    perturb = float(perturb)
    noise_std = float(noise_std)

    pr, nc, ur, nf, seed = _resolve_randoms(randoms, n, S_c, K, perturb, noise_std, dev, match_reference_rng)
    if seed is not None and needs_graph and (autograd_impl == "torch" or test_time):
        raise ValueError("in-kernel random numbers are not available on the torch-autograd path")
    if occupancy is not None and n > 0:
        return _render_rays_grid(models, rays_c, S_c, K, use_disp, perturb, noise_std, white_back, test_time, extras,
                                 needs_graph, occupancy, (pr, nc, ur, nf), seed)

    if needs_graph and extras:
        raise ValueError("extras=True is an inference-only option (no gradient graph is built for the extra tensors)")
    if needs_graph and autograd_impl == "fused" and not test_time and n > 0:
        from .training import render_rays_train
        return render_rays_train(models, rays_c, S_c, use_disp, perturb, noise_std, K, white_back, pr, nc, ur, nf,
                                 rng_seed=seed)

    f32 = dict(dtype=torch.float32, device=dev)
    coarse_rgb = not test_time
    # one allocation, contiguous (n,3) / (n,) views of it
    flat = torch.empty(10 * n, **f32)
    out = {
        "rgb_coarse": flat[0:3 * n].view(n, 3) if coarse_rgb else None,
        "depth_coarse": flat[3 * n:4 * n] if coarse_rgb else None,
        "opacity_coarse": flat[4 * n:5 * n],
        "rgb_fine": flat[5 * n:8 * n].view(n, 3) if K > 0 else None,
        "depth_fine": flat[8 * n:9 * n] if K > 0 else None,
        "opacity_fine": flat[9 * n:10 * n] if K > 0 else None,
    }
    z_fine = torch.empty(n, S_f, **f32) if ((extras or needs_graph) and K > 0) else None
    w_c = torch.empty(n, S_c, **f32) if extras else None
    w_f = torch.empty(n, S_f, **f32) if (extras and K > 0) else None

    packed = (packed_weights(models[0]), packed_weights(models[1]) if K > 0 else None)
    args = _render_args(rays_c, S_c, K, use_disp, perturb, noise_std, white_back, test_time, packed, (pr, nc, ur, nf),
                        dict(out, z_fine=z_fine, weights_coarse=w_c, weights_fine=w_f), seed)
    _lib.call("nerfb200_render_rays", dev, ctypes.byref(args))

    if needs_graph:
        return _render_with_graph(models, embeddings, rays_c, S_c, K, bool(use_disp), perturb, noise_std,
                                  bool(white_back), bool(test_time), pr, nc, nf, z_fine)

    result = {k: v for k, v in out.items() if v is not None}
    if extras:
        if z_fine is not None:
            result["z_vals_fine"] = z_fine
            result["weights_fine"] = w_f
        result["weights_coarse"] = w_c
    return result


def _check_grid_call(occupancy, rays, S_c: int, K: int, needs_graph: bool, test_time, extras, autograd_impl) -> None:
    """The checks of render_rays(..., occupancy=) that need no device: the grid's type and, with a gradient graph,
    the options and shapes that path supports (ValueError)."""
    from .culling import OccupancyGrid
    from .train_skip import check_shape
    if not isinstance(occupancy, OccupancyGrid):
        raise ValueError("occupancy must be a nerf_pl_b200.OccupancyGrid (for a DensityGrid pass its .grid)")
    if not needs_graph:
        return
    if test_time or extras or autograd_impl != "fused":
        raise ValueError("render_rays(..., occupancy=) with a gradient graph needs test_time=False, extras=False and "
                         "autograd_impl='fused' (render under torch.no_grad() for the others)")
    n = rays.shape[0]
    if n != 0:
        check_shape(n, S_c, K)


def _render_rays_grid(models, rays, S_c: int, K: int, use_disp, perturb: float, noise_std: float, white_back,
                      test_time, extras, needs_graph: bool, occupancy, randoms, seed) -> Dict[str, torch.Tensor]:
    """render_rays(..., occupancy=) of n >= 1 rays: the differentiable skipped step without a loss, or the skipped
    render of every ray.  Returns render_rays' keys."""
    if needs_graph:
        from .train_skip import render_rays_train_skip
        live = torch.empty(2, dtype=torch.int64, device=rays.device)      # the capturable entries: no read-back
        res = render_rays_train_skip(models, rays, S_c, use_disp, perturb, noise_std, K, white_back, *randoms, None,
                                     occupancy, rng_seed=seed, live_samples=live)
    else:
        from .culling import render_samples
        res = render_samples(models, rays, occupancy, S_c, use_disp, K, white_back, test_time, extras=extras,
                             perturb=perturb, noise_std=noise_std, randoms=randoms, rng_seed=seed)
    del res["live_samples"]
    return res


@torch.no_grad()
def render_rays_host(models: List[torch.nn.Module],
                     embeddings: List[torch.nn.Module],
                     rays: torch.Tensor,
                     N_samples: int = 64,
                     use_disp: bool = False,
                     perturb: float = 0,
                     noise_std: float = 1,
                     N_importance: int = 0,
                     chunk: int = 1024 * 32,
                     white_back: bool = False,
                     test_time: bool = False,
                     *,
                     out: Optional[Dict[str, torch.Tensor]] = None,
                     randoms=None,
                     match_reference_rng: bool = False) -> Dict[str, torch.Tensor]:
    """render_rays for rays that live in HOST memory (the reference's eval loop moves every chunk with
    ``.cuda()`` and the results back with ``.cpu()``, eval.py:117-123): ONE call into the C ABI
    (``nerfb200_render_rays_host``) renders them and returns with the results readable on the host.
    ``rays``: (N, 8) float32 CPU tensor.  With pinned rays (and pinned ``out`` tensors, allocated here when
    not supplied) the kernel reads the rays and writes the results over PCIe itself (mapped memory: no staging
    copies); pageable buffers are staged through device memory with cudaMemcpyAsync.  Returns CPU tensors.
    Inference only; the random inputs are drawn on the device."""
    del chunk
    if rays.is_cuda or rays.dim() != 2 or rays.shape[1] != 8 or rays.dtype != torch.float32:
        raise ValueError("rays must be a (N_rays, 8) float32 CPU tensor")
    _check_render_inputs("render_rays_host", models, embeddings, N_importance, None)
    dev = next(models[0].parameters()).device
    if dev.type != "cuda":
        raise RuntimeError("the models must live on a CUDA device (no CPU fallback)")
    n, S_c, K = rays.shape[0], int(N_samples), int(N_importance)
    if rays.stride(1) != 1 or rays.stride(0) < 8:
        rays = rays.contiguous()          # a row stride (column slice of a wider tensor) is passed through
    pinned = rays.is_pinned()       # results then come back in pinned memory too: the C entry's zero-copy path
    perturb, noise_std = float(perturb), float(noise_std)
    pr, nc, ur, nf, seed = _resolve_randoms(randoms, n, S_c, K, perturb, noise_std, dev, match_reference_rng)
    keys = ["opacity_coarse"] if test_time else ["rgb_coarse", "depth_coarse", "opacity_coarse"]
    if K > 0:
        keys += ["rgb_fine", "depth_fine", "opacity_fine"]
    res = {}
    for k in keys:
        shape = (n, 3) if k.startswith("rgb") else (n,)
        t = out[k] if out is not None and k in out else torch.empty(shape, dtype=torch.float32, pin_memory=pinned)
        if t.is_cuda or t.shape != shape or t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError(f"out[{k!r}] must be a contiguous float32 CPU tensor of shape {shape}")
        res[k] = t
    packed = (packed_weights(models[0]), packed_weights(models[1]) if K > 0 else None)
    args = _render_args(rays, S_c, K, use_disp, perturb, noise_std, white_back, test_time, packed, (pr, nc, ur, nf),
                        res, seed)
    _lib.call("nerfb200_render_rays_host", dev, ctypes.byref(args))
    return res


def render_rays_loss(models: List[torch.nn.Module],
                     embeddings: List[torch.nn.Module],
                     rays: torch.Tensor,
                     rgbs: torch.Tensor,
                     N_samples: int = 64,
                     use_disp: bool = False,
                     perturb: float = 0,
                     noise_std: float = 1,
                     N_importance: int = 0,
                     chunk: int = 1024 * 32,
                     white_back: bool = False,
                     *,
                     randoms: Optional[Dict[str, torch.Tensor]] = None,
                     match_reference_rng: bool = True,
                     occupancy=None) -> Dict[str, torch.Tensor]:
    """One training-step forward with the loss fused into the render launch: the reference's
    ``results = render_rays(...)`` (train.py:55-64), ``loss = MSELoss(results, rgbs)``
    (losses.py:9-14) and ``psnr(results['rgb_fine'], rgbs)`` (metrics.py:12-13, train.py:107-112) as
    ONE kernel.  Returns the render_rays result dict plus ``loss`` (differentiable scalar),
    ``psnr``, ``mse_coarse``, ``mse_fine``; ``loss.backward()`` runs the fused sm_90a backward with
    the gradient seed 2 (rgb - rgbs) / (3 N) formed inside the compositing-backward kernel.

    ``occupancy`` (a ``nerf_pl_b200.OccupancyGrid``) skips the empty samples of every ray (``train_skip.py``,
    DESIGN.md "Training with empty samples skipped"): the result gains ``'live_samples'`` (evaluated coarse, fine
    samples), and every result is differentiable, as without it.  It needs the render kernel's shapes and at most 2^22 rays
    (ValueError), and a grid on the rays' device (RuntimeError); each step synchronises once, to read back
    ``live_samples`` (``CapturedTrainStep(..., occupancy=grid)`` replays the step without synchronising)."""
    del chunk
    _check_render_inputs("render_rays_loss", models, embeddings, N_importance, rays)
    n, S_c, K = rays.shape[0], int(N_samples), int(N_importance)
    if n == 0:
        raise ValueError("empty ray batch")
    if occupancy is not None:
        from .train_skip import check_grid, check_shape
        check_shape(n, S_c, K)
        check_grid(occupancy, rays)
    rays_c = rays.detach().to(torch.float32).contiguous()
    pr, nc, ur, nf, seed = _resolve_randoms(randoms, n, S_c, K, float(perturb), float(noise_std), rays.device,
                                            match_reference_rng)
    if occupancy is not None:
        from .train_skip import render_rays_train_skip
        return render_rays_train_skip(models, rays_c, S_c, use_disp, float(perturb), float(noise_std), K, white_back,
                                      pr, nc, ur, nf, rgbs, occupancy, rng_seed=seed)
    from .training import render_rays_train
    return render_rays_train(models, rays_c, S_c, use_disp, float(perturb), float(noise_std), K, white_back,
                             pr, nc, ur, nf, target=rgbs, rng_seed=seed)


# ---------------------------------------------------------------------------------------------
# Autograd path (training): the fused kernel has produced the detached fine depths
# (models/rendering.py:225-229: no gradient flows through sampling); the differentiable part
# - embedding, MLP, quadrature at those depths - is evaluated with torch ops so that
# .backward() fills the parameters' .grad exactly as in the reference.  This is the
# ``autograd_impl="torch"`` path: plain torch autograd, kept as an independent check of the fused
# backward (nerf_pl_b200/training.py) in the GPU tests; the product's training path never uses it.
def _coarse_depths(rays: torch.Tensor, S: int, use_disp: bool, perturb: float, pr) -> torch.Tensor:
    near, far = rays[:, 6:7], rays[:, 7:8]
    t = torch.linspace(0, 1, S, device=rays.device)
    z = 1 / (1 / near * (1 - t) + 1 / far * t) if use_disp else near * (1 - t) + far * t
    z = z.expand(rays.shape[0], S)
    if perturb > 0:
        mid = 0.5 * (z[:, :-1] + z[:, 1:])
        upper = torch.cat((mid, z[:, -1:]), -1)
        lower = torch.cat((z[:, :1], mid), -1)
        z = lower + (upper - lower) * (perturb * pr)
    return z


def _embed_torch(x: torch.Tensor, n_freqs: int) -> torch.Tensor:
    parts = [x]
    for k in range(n_freqs):
        parts += [torch.sin((2.0 ** k) * x), torch.cos((2.0 ** k) * x)]
    return torch.cat(parts, -1)


def _pass_torch(model, rays, z, noise, noise_std, white_back, sigma_only):
    n, S = z.shape
    o, d = rays[:, 0:3], rays[:, 3:6]
    xyz = (o[:, None, :] + d[:, None, :] * z[:, :, None]).reshape(-1, 3)
    x = _embed_torch(xyz, 10)
    if not sigma_only:
        de = _embed_torch(d, 4)
        x = torch.cat((x, de.repeat_interleave(S, dim=0)), -1)
    raw = nerf_forward_torch(model, x, sigma_only)
    sig = raw.view(n, S) if sigma_only else raw.view(n, S, 4)[..., 3]
    delta = torch.cat((z[:, 1:] - z[:, :-1], torch.full_like(z[:, :1], 1e10)), -1) * d.norm(dim=-1, keepdim=True)
    if noise is not None:
        sig = sig + noise * noise_std
    alpha = 1 - torch.exp(-delta * torch.relu(sig))
    trans = torch.cumprod(torch.cat((torch.ones_like(alpha[:, :1]), 1 - alpha + 1e-10), -1), -1)[:, :-1]
    w = alpha * trans
    opac = w.sum(1)
    if sigma_only:
        return None, None, opac
    rgb = (w[..., None] * raw.view(n, S, 4)[..., :3]).sum(-2)
    depth = (w * z).sum(-1)
    if white_back:
        rgb = rgb + 1 - opac[:, None]
    return rgb, depth, opac


def _render_with_graph(models, embeddings, rays, S_c, K, use_disp, perturb, noise_std, white_back,
                       test_time, pr, nc, nf, z_fine):
    z_c = _coarse_depths(rays, S_c, use_disp, perturb, pr)
    rgb, depth, opac = _pass_torch(models[0], rays, z_c, nc if noise_std > 0 else None, noise_std,
                                   white_back, test_time)
    result = {"opacity_coarse": opac}
    if not test_time:
        result = {"rgb_coarse": rgb, "depth_coarse": depth, "opacity_coarse": opac}
    if K > 0:
        rgb, depth, opac = _pass_torch(models[1], rays, z_fine, nf if noise_std > 0 else None, noise_std,
                                       white_back, False)
        result.update(rgb_fine=rgb, depth_fine=depth, opacity_fine=opac)
    return result
