"""The training step with empty samples skipped: ``render_rays_loss(..., occupancy=grid)`` and, without the fused loss,
``render_rays(..., occupancy=grid)`` under a gradient graph (DESIGN.md "Training with empty samples skipped", §10g).

Every ray of the batch is rendered and enters the loss; inside a ray, a sample whose point lies in no occupied cell of
``grid`` gets sigma = 0 (no noise is added to it) and is not evaluated, so its weight is exactly 0 and it receives no
gradient.  An evaluated sample gets the network's sigma and rgb bit for bit as the fused training kernel computes
them, then the noise.  Rebuild the grid from the fine network as training goes (INTEGRATION.md section 7): density
that appears in a cell the grid calls empty is trained from the next rebuild on.

forward : ``nerfb200_train_samples_forward`` (include/nerf_pl_b200.h): perturbed depths and
          classification, the compacted rows of each network through the save-mode MLP, compositing with noise, the
          random resampling and the merge, the loss.  Every launch is sized for the worst case and reads the
          step's sample counts on the device; the eager call reads the two counts back once at the end.
backward: ``nerfb200_train_samples_backward``: per network, a plan kernel turns the device count into the launch
          parameters, then the compositing backward over the sparse sample lists (seeded by the upstream gradients
          of the pass's rgb, depth and opacity, plus the fused MSE term with a target) and the backward of a direct
          ``NeRF.forward`` call (chain, wgrad, reduction, unfold).
capturable mode (``live_samples=`` a device tensor): the ``_dev`` entries, which neither synchronise nor read host
          memory, so ``CapturedTrainStep(occupancy=grid)`` replays the step as one CUDA graph.
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional

import torch

from . import _lib
from .nerf import _aligned_buffer, packed_weights, packed_weights_pair
from .rendering import _ptr
from .training import _Lease, _grad_buffers, _params_of

MAX_RAYS = 1 << 22


class SkipTrainWorkspace:
    """Device workspace of one (device, n_rays, N_samples, N_importance) shape, sized for every sample evaluated and
    zeroed once: the steps of one batch shape share it whatever their evaluated sample counts, without reallocating or
    re-zeroing.  Pool and lease policy as ``TrainWorkspace``: a call holds its workspace until its backward runs or
    its graph is freed."""

    _pool: Dict[tuple, List["SkipTrainWorkspace"]] = {}

    def __init__(self, dev: torch.device, n: int, S_c: int, K: int) -> None:
        nbytes = int(_lib.load().nerfb200_train_samples_workspace_bytes(n, S_c, K))
        if nbytes == 0:
            raise ValueError("invalid training shape")
        self.key = (dev.index, n, S_c, K)
        self.buf = _aligned_buffer(nbytes, dev)
        self.buf.zero_()
        self.bytes = nbytes
        self.busy = False

    @classmethod
    def acquire(cls, dev: torch.device, n: int, S_c: int, K: int) -> "SkipTrainWorkspace":
        free = cls._pool.setdefault((dev.index, n, S_c, K), [])
        for ws in free:
            if not ws.busy:
                ws.busy = True
                return ws
        ws = cls(dev, n, S_c, K)
        ws.busy = True
        free.append(ws)
        return ws

    @classmethod
    def clear(cls) -> None:
        cls._pool.clear()


def check_shape(n: int, S_c: int, K: int) -> None:
    """The render kernel's envelope, and at most ``MAX_RAYS`` rays (ValueError otherwise)."""
    if S_c not in (32, 64, 128) or K < 0 or K % 32 or S_c + K > 192 or not 1 <= n <= MAX_RAYS:
        raise ValueError("occupancy= needs N_samples in {32, 64, 128}, N_importance a multiple of 32 with "
                         f"N_samples + N_importance <= 192, and 1 <= N_rays <= {MAX_RAYS}")


def check_grid(occupancy, rays: torch.Tensor) -> None:
    from .culling import OccupancyGrid
    if not isinstance(occupancy, OccupancyGrid):
        raise ValueError("occupancy must be a nerf_pl_b200.OccupancyGrid")
    if occupancy.device != rays.device:
        raise RuntimeError(f"the occupancy grid is on {occupancy.device}, the rays on {rays.device}")


_OUTPUTS = ("rgb_coarse", "depth_coarse", "opacity_coarse", "rgb_fine", "depth_fine", "opacity_fine")


def _aligned16(t: torch.Tensor) -> torch.Tensor:
    return t if t.data_ptr() % 16 == 0 else t.clone()


class SkipRenderFunction(torch.autograd.Function):
    """rays + randoms [+ target] + 48 parameter tensors -> the six result tensors [+ loss4].  Every output carries a
    gradient: the backward's seed per pass is the upstream gradient of its rgb, depth and opacity plus, with a target,
    the fused MSE term scaled by d(loss4[2]) (composite_bwd_kernel's seed, include/nerf_pl_b200.h)."""

    @staticmethod
    def forward(ctx, cfg: Dict, rays, pr, nc, ur, nf, target, *params):
        models, grid = cfg["models"], cfg["occupancy"]
        S_c, K = cfg["N_samples"], cfg["N_importance"]
        n, dev = rays.shape[0], rays.device
        f32 = dict(dtype=torch.float32, device=dev)
        out = [torch.empty(n, 3, **f32), torch.empty(n, **f32), torch.empty(n, **f32)]
        if K > 0:
            out += [torch.empty(n, 3, **f32), torch.empty(n, **f32), torch.empty(n, **f32)]
        loss_out = torch.empty(4, **f32) if target is not None else None
        if K > 0:
            blob_c, blob_f = packed_weights_pair(models[0], models[1])
        else:
            blob_c, blob_f = packed_weights(models[0]), None
        own, live_dev = cfg.get("workspace"), cfg.get("live_out")
        if own is not None and own.key != (dev.index, n, S_c, K):
            raise ValueError("the given training workspace is of another shape")
        lease = _Lease(own if own is not None else SkipTrainWorkspace.acquire(dev, n, S_c, K))
        seed = cfg.get("rng_seed")
        if seed is None:
            rng = dict(rng_seed=0, rng_in_kernel=0)
        elif torch.is_tensor(seed):
            rng = dict(rng_seed=seed.data_ptr(), rng_in_kernel=2)
        else:
            rng = dict(rng_seed=seed, rng_in_kernel=1)
        extras = cfg.get("extras") or {}
        args = _lib.TrainSamplesArgs(
            rays=rays.data_ptr(), n_rays=n, packed_coarse=blob_c.data_ptr(), packed_fine=_ptr(blob_f),
            n_samples=S_c, n_importance=K, use_disp=int(cfg["use_disp"]), white_back=int(cfg["white_back"]),
            perturb=cfg["perturb"], noise_std=cfg["noise_std"], perturb_rand=_ptr(pr), noise_coarse=_ptr(nc),
            u_rand=_ptr(ur), noise_fine=_ptr(nf), bits=grid.bits.data_ptr(), N=grid.N,
            ranges=(ctypes.c_double * 6)(*grid.ranges), levels=grid.levels, target=_ptr(target),
            loss_out=_ptr(loss_out),
            **dict(zip(_OUTPUTS, [o.data_ptr() for o in out])), **{k: _ptr(t) for k, t in extras.items()}, **rng)
        if live_dev is None:
            live = (ctypes.c_int64 * 2)()
            _lib.call("nerfb200_train_samples_forward", dev, ctypes.byref(args), lease.ws.buf.data_ptr(),
                      lease.ws.bytes, live)
            cfg["live_samples"] = (int(live[0]), int(live[1]))
        else:
            live = None
            _lib.call("nerfb200_train_samples_forward_dev", dev, ctypes.byref(args), lease.ws.buf.data_ptr(),
                      lease.ws.bytes, ctypes.cast(live_dev.data_ptr(), ctypes.POINTER(ctypes.c_int64)))
            cfg["live_samples"] = live_dev
        ctx.args, ctx.live, ctx.lease, ctx.K, ctx.has_loss = args, live, lease, K, target is not None
        # what the args point to (detached aliases of the outputs: see FusedRenderFunction)
        ctx.keep = (rays, pr, nc, ur, nf, target, [o.detach() for o in out], blob_c, blob_f, grid.bits, seed)
        ctx.n_params = len(params)
        ctx.save_for_backward(*params)
        ctx.set_materialize_grads(False)
        return tuple(out) + ((loss_out,) if target is not None else ())

    @staticmethod
    def backward(ctx, *gouts):
        lease = ctx.lease
        if lease.ws is None:
            raise RuntimeError("the backward of this render has already run (retain_graph=True is not supported)")
        n_out = 6 if ctx.K > 0 else 3
        params = list(ctx.saved_tensors)
        g6 = [None if t is None else t.detach().to(torch.float32).contiguous() for t in gouts[:n_out]]
        g4 = gouts[n_out] if ctx.has_loss else None
        if g4 is None and all(t is None for t in g6):
            lease.release()
            return (None,) * (7 + ctx.n_params)
        args = ctx.args
        for name, t in zip(_OUTPUTS, g6):
            setattr(args, "g_" + name, _ptr(t))
        if g4 is None:              # no MSE term in the seed
            args.target = args.loss_out = None
            loss_grad = None
        else:
            g4 = g4.detach().to(torch.float32).contiguous()
            loss_grad = g4.data_ptr() + 8
        dev = params[0].device
        grads, tables = _grad_buffers(params, dev)
        nets = 2 if ctx.K > 0 else 1
        (pc, gc) = tables[0]
        pf, gf = tables[1] if nets > 1 else (None, None)
        if ctx.live is None:                     # capturable: the device path writes every network's gradients
            _lib.call("nerfb200_train_samples_backward_dev", dev, ctypes.byref(args), lease.ws.buf.data_ptr(),
                      lease.ws.bytes, loss_grad, pc, pf, gc, gf)
        else:
            for ps in range(nets):
                if ctx.live[ps] == 0:            # no evaluated sample: nothing launched for this network
                    for t in grads[24 * ps:24 * ps + 24]:
                        t.zero_()
            _lib.call("nerfb200_train_samples_backward", dev, ctypes.byref(args), lease.ws.buf.data_ptr(),
                      lease.ws.bytes, ctx.live, loss_grad, pc, pf, gc, gf)
        lease.release()
        ctx.keep = ctx.args = None
        if nets == 1:
            grads = grads[:24] + [None] * (ctx.n_params - 24)
        return (None,) * 7 + tuple(grads)


def render_rays_train_skip(models, rays, N_samples, use_disp, perturb, noise_std, N_importance, white_back, pr, nc, ur,
                           nf, target: Optional[torch.Tensor], occupancy, rng_seed=None, extras: bool = False,
                           workspace: Optional[SkipTrainWorkspace] = None,
                           live_samples: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """``render_rays_train`` with empty samples skipped: the result keys of ``render_rays_loss`` plus
    ``'live_samples'`` (evaluated coarse, fine samples); with ``target=None``, ``render_rays``' keys plus
    ``'live_samples'``, without the loss.  Every result tensor is differentiable.  ``extras`` adds, for tests: ``z_vals_coarse``,
    ``z_vals_fine``, ``weights_coarse``, ``weights_fine``, ``samples_coarse`` / ``samples_fine`` (n, S, 4: network
    rgb and sigma, 0 where skipped) and ``mask_coarse`` / ``mask_fine`` ((n, 6) int32, bit b of word w: sample
    32 w + b evaluated), and ``dsigma_coarse`` / ``dsigma_fine`` (n S) and ``dprergb_coarse`` / ``dprergb_fine``
    (n S, 3), which ``loss.backward()`` fills in their first ``live_samples`` rows with the per-row d loss / d sigma
    and d loss / d (rgb before the sigmoid) of the evaluated samples, ray-major in depth-index order.

    ``live_samples`` (a device int64 tensor of 2 elements) selects the capturable mode: no host synchronisation, the
    counts are written into that tensor, which is also the result's ``'live_samples'``, and the backward writes
    every network's gradients itself (exact zeros for a network with no evaluated sample).  ``workspace`` is a
    ``SkipTrainWorkspace`` of this shape that the caller owns (outside the pool), as ``render_rays_train`` takes."""
    S_c, K = int(N_samples), int(N_importance)
    n, dev = rays.shape[0], rays.device
    if live_samples is not None and (live_samples.dtype != torch.int64 or live_samples.numel() != 2
                                     or live_samples.device != dev or not live_samples.is_contiguous()):
        raise ValueError("live_samples must be a contiguous int64 tensor of 2 elements on the rays' device")
    f32 = dict(dtype=torch.float32, device=dev)
    ex = {}
    if extras:
        ex = dict(z_coarse=torch.empty(n, S_c, **f32), weights_coarse=torch.empty(n, S_c, **f32),
                  samples_coarse=torch.empty(n, S_c, 4, **f32),
                  mask_coarse=torch.empty(n, 6, dtype=torch.int32, device=dev),
                  dsigma_coarse=torch.zeros(n * S_c, **f32), dprergb_coarse=torch.zeros(n * S_c, 3, **f32))
        if K > 0:
            ex.update(z_fine=torch.empty(n, S_c + K, **f32), weights_fine=torch.empty(n, S_c + K, **f32),
                      samples_fine=torch.empty(n, S_c + K, 4, **f32),
                      mask_fine=torch.empty(n, 6, dtype=torch.int32, device=dev),
                      dsigma_fine=torch.zeros(n * (S_c + K), **f32), dprergb_fine=torch.zeros(n * (S_c + K), 3, **f32))
    cfg = dict(models=list(models), occupancy=occupancy, N_samples=S_c, N_importance=K, use_disp=bool(use_disp),
               perturb=float(perturb), noise_std=float(noise_std), white_back=bool(white_back), rng_seed=rng_seed,
               extras=ex, workspace=workspace, live_out=live_samples)
    params = _params_of(models, K)
    if target is not None:
        target = target.detach().to(torch.float32).contiguous()
        if target.shape != (n, 3):
            raise ValueError("target must be (N_rays, 3)")
    outs = SkipRenderFunction.apply(cfg, _aligned16(rays), pr, nc, ur, nf, target, *params)
    res = {"rgb_coarse": outs[0], "depth_coarse": outs[1], "opacity_coarse": outs[2]}
    k = 3
    if K > 0:
        res.update(rgb_fine=outs[3], depth_fine=outs[4], opacity_fine=outs[5])
        k = 6
    if target is not None:
        l4 = outs[k]
        res.update(loss=l4[2], psnr=l4[3].detach(), mse_coarse=l4[0].detach(), mse_fine=l4[1].detach())
    res["live_samples"] = cfg["live_samples"]
    names = dict(z_coarse="z_vals_coarse", z_fine="z_vals_fine")
    res.update({names.get(key, key): t for key, t in ex.items()})
    return res
