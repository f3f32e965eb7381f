"""Training path of ``render_rays`` (reference: train.py:103-117 — ``results = render_rays(...)``,
``loss = MSELoss(results, rgbs)``, ``loss.backward()`` through models/rendering.py + models/nerf.py):
a ``torch.autograd.Function`` around the fused sm_90a kernels.  No torch op, cuBLAS call or
autograd graph is involved in either direction.

forward : ONE fused ``render_rays_kernel`` launch in training mode.  It renders exactly like
          inference and additionally leaves in the training workspace, per sample, what the backward
          needs: encoded input + the 8 hidden activations (fp16, in the tensor core's MN-major
          operand layout), ReLU sign bits, the direction-layer output, raw sigma / rgb, the depths.
          Optionally the MSE loss / PSNR of the batch are reduced in the same launch
          (``render_rays_loss``).
backward: ``nerfb200_render_backward`` (include/nerf_pl_b200.h): compositing backward -> rgb head ->
          wgmma dgrad chain -> wgmma split-K wgrad -> fixed-order reduction -> unfolding of the
          packed final.dir layer; fills the 48 ``.grad`` tensors.
The sampling of the fine depths carries no gradient (models/rendering.py:225-227 ``.detach()``).

``nerf_forward_train`` (end of this file) trains a direct ``NeRF.forward`` call the same way, for callers that
render with their own code: one save-mode launch of the MLP kernel, then the same backward kernels seeded from
the upstream (B, 4) gradient.
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional

import torch

from . import _lib
from .nerf import (_EXPECTED_SHAPES, _aligned_buffer, nerf_forward_fused, nerf_parameters, packed_weights,
                   packed_weights_pair)
from .data import _EpochBatches, next_step_schedule
from .rendering import _draw_randoms, _ptr, _render_args


class _Workspace:
    """A 1024-byte aligned device buffer (``buf``, ``bytes`` long) prepared by the library entry ``init`` as
    ``init(buf, bytes, *args, stream)``.  ``busy``: held by a call whose backward is pending."""

    def __init__(self, dev: torch.device, nbytes: int, init: str, *args) -> None:
        self.buf = _aligned_buffer(nbytes, dev)
        self.bytes = nbytes
        self.busy = False
        _lib.call(init, dev, self.buf.data_ptr(), nbytes, *args)


class TrainWorkspace(_Workspace):
    """Device workspace of one (device, n_rays, N_samples, N_importance) shape, reused across steps.
    A render holds its workspace (``busy``) from its forward until its backward runs, or until its graph is
    freed without one (a skipped batch, a render under grad mode used only for a metric), so that a second
    forward (gradient accumulation over several batches) gets its own buffer.  The pool of a shape holds as many
    workspaces as there were pending backwards at once."""

    _pool: Dict[tuple, List["TrainWorkspace"]] = {}

    def __init__(self, dev: torch.device, n: int, S_c: int, K: int) -> None:
        nbytes = int(_lib.load().nerfb200_train_workspace_bytes(n, S_c, K))
        if nbytes == 0:
            raise ValueError("invalid training shape")
        self.key = (dev.index, n, S_c, K)
        super().__init__(dev, nbytes, "nerfb200_train_workspace_init", n, S_c, K)

    @classmethod
    def acquire(cls, dev: torch.device, n: int, S_c: int, K: int) -> "TrainWorkspace":
        key = (dev.index, n, S_c, K)
        free = cls._pool.setdefault(key, [])
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


class _Lease:
    """A call's hold on its workspace (``TrainWorkspace`` or ``NerfTrainWorkspace``): released by the backward,
    or when autograd frees the graph (the ctx that owns the lease is destroyed) without one."""
    __slots__ = ("ws",)

    def __init__(self, ws) -> None:
        self.ws = ws

    def release(self) -> None:
        if self.ws is not None:
            self.ws.busy = False
            self.ws = None

    def __del__(self) -> None:
        self.release()


_OUTPUTS = ("rgb_coarse", "depth_coarse", "opacity_coarse", "rgb_fine", "depth_fine", "opacity_fine")


class FusedRenderFunction(torch.autograd.Function):
    """rays + pre-drawn randoms [+ target] + 48 parameter tensors -> the six result tensors [+ loss4]."""

    @staticmethod
    def forward(ctx, cfg: Dict, rays, pr, nc, ur, nf, target, *params):
        models = cfg["models"]
        S_c, K = cfg["N_samples"], cfg["N_importance"]
        n = rays.shape[0]
        dev = rays.device
        f32 = dict(dtype=torch.float32, device=dev)
        out = [torch.empty(n, 3, **f32), torch.empty(n, **f32), torch.empty(n, **f32)]
        if K > 0:
            out += [torch.empty(n, 3, **f32), torch.empty(n, **f32), torch.empty(n, **f32)]
        loss_out = torch.empty(4, **f32) if target is not None else None
        if K > 0:
            blob_c, blob_f = packed_weights_pair(models[0], models[1])      # one launch for both images
        else:
            blob_c, blob_f = packed_weights(models[0]), None
        own = cfg.get("workspace")        # a workspace outside the pool (CapturedTrainStep's)
        if own is not None and own.key != (dev.index, n, S_c, K):
            raise ValueError("the given training workspace is of another shape")
        lease = _Lease(own if own is not None else TrainWorkspace.acquire(dev, n, S_c, K))
        args = _render_args(rays, S_c, K, cfg["use_disp"], cfg["perturb"], cfg["noise_std"], cfg["white_back"], False,
                            (blob_c, blob_f), (pr, nc, ur, nf), dict(zip(_OUTPUTS, out)), cfg.get("rng_seed"),
                            lease.ws, target, loss_out)
        _lib.call("nerfb200_render_rays", dev, ctypes.byref(args))
        ctx.cfg = cfg
        ctx.lease = lease
        # the backward takes the same render args without the loss epilogue (its seed comes in the backward args)
        args.target = args.loss_out = None
        ctx.args = args
        # what the args point to.  Detached aliases of the outputs: the returned tensors themselves on ctx would form
        # a cycle (output -> grad_fn -> ctx -> output) that keeps a dropped graph, and with it the workspace, alive
        ctx.keep = (rays, pr, nc, ur, nf, target, [o.detach() for o in out], blob_c, blob_f, lease.ws)
        ctx.n_params = len(params)
        ctx.save_for_backward(*params)
        ctx.set_materialize_grads(False)
        res = tuple(out)
        if loss_out is not None:
            res = res + (loss_out,)
        return res

    @staticmethod
    def backward(ctx, *gouts):
        lease = ctx.lease
        if lease.ws is None:
            raise RuntimeError("the fused backward of this render has already run (its training workspace is released "
                               "after one backward; retain_graph=True is not supported with autograd_impl='fused')")
        params = list(ctx.saved_tensors)
        rays, target = ctx.keep[0], ctx.keep[5]
        K = ctx.cfg["N_importance"]
        g = [None if t is None else t.detach().to(torch.float32).contiguous() for t in gouts]
        g6 = g[:6] + [None] * (6 - min(len(g), 6))
        if K == 0:
            g6 = g[:3] + [None] * 3
        n_out = 6 if K > 0 else 3
        loss_grad = None
        use_target = None
        if target is not None:
            g4 = g[n_out]
            if g4 is not None:
                # d(loss_out)/d(rgb): element 2 = MSELoss (elements 0 / 1 = its coarse / fine terms: the same
                # seed restricted to one pass is not provided); take the gradient of the total loss
                loss_grad = g4          # the kernel reads element 2 (address passed below)
                use_target = target
        grads, tables = _grad_buffers(params, rays.device)
        (pc, gc), (pf, gf) = tables[0], (tables[1] if K > 0 else (None, None))
        bargs = _lib.BackwardArgs(
            render=ctypes.pointer(ctx.args), params_coarse=pc, params_fine=pf,
            g_rgb_coarse=_ptr(g6[0]), g_depth_coarse=_ptr(g6[1]), g_opacity_coarse=_ptr(g6[2]),
            g_rgb_fine=_ptr(g6[3]), g_depth_fine=_ptr(g6[4]), g_opacity_fine=_ptr(g6[5]),
            target=_ptr(use_target), loss_grad=None if loss_grad is None else loss_grad.data_ptr() + 8,
            grads_coarse=gc, grads_fine=gf)
        _lib.call("nerfb200_render_backward", rays.device, ctypes.byref(bargs))
        lease.release()
        ctx.keep = ctx.args = None
        if K == 0:
            grads = grads[:24] + [None] * (ctx.n_params - 24)
        return (None, None, None, None, None, None, None, *grads)


_SIZE_CACHE: Dict[int, tuple] = {}


def _param_sizes(params):
    key = len(params)
    hit = _SIZE_CACHE.get(key)
    if hit is None:
        hit = ([p.numel() for p in params], [tuple(p.shape) for p in params])
        _SIZE_CACHE[key] = hit
    return hit


def _grad_buffers(params, dev):
    """The gradients of ``params`` as views of one allocation (the kernels write every element), and per network
    (24 parameters each) the ctypes pointer arrays (parameters, gradients) the backward entries take."""
    sizes, shapes = _param_sizes(params)
    flat = torch.empty(sum(sizes), dtype=torch.float32, device=dev)
    grads = [t.view(shp) for t, shp in zip(flat.split(sizes), shapes)]
    tables = [((ctypes.c_void_p * 24)(*[p.data_ptr() for p in params[i:i + 24]]),
               (ctypes.c_void_p * 24)(*[t.data_ptr() for t in grads[i:i + 24]])) for i in range(0, len(params), 24)]
    return grads, tables


def _params_of(models, N_importance) -> List[torch.Tensor]:
    params = nerf_parameters(models[0])
    if N_importance > 0:
        params = params + nerf_parameters(models[1])
    return params          # shapes / contiguity are validated by packed_weights()


def render_rays_train(models, rays, N_samples, use_disp, perturb, noise_std, N_importance, white_back,
                      pr, nc, ur, nf, target: Optional[torch.Tensor] = None,
                      rng_seed=None, workspace: Optional[TrainWorkspace] = None) -> Dict[str, torch.Tensor]:
    """Differentiable render_rays (test_time=False) through FusedRenderFunction.  With ``target``
    (n,3) the result also carries ``loss`` (losses.py:9-14 MSELoss of the batch), ``psnr``
    (metrics.py:4-13, of the finest pass), ``mse_coarse`` and ``mse_fine`` computed by the same
    launch; ``loss.backward()`` then seeds the backward inside the kernels."""
    cfg = dict(models=list(models), N_samples=int(N_samples), N_importance=int(N_importance),
               use_disp=bool(use_disp), perturb=float(perturb), noise_std=float(noise_std),
               white_back=bool(white_back), rng_seed=rng_seed, workspace=workspace)
    params = _params_of(models, N_importance)
    if target is not None:
        target = target.detach().to(torch.float32).contiguous()
        if target.shape != (rays.shape[0], 3):
            raise ValueError("target must be (N_rays, 3)")
    outs = FusedRenderFunction.apply(cfg, rays, pr, nc, ur, nf, target, *params)
    res = {"rgb_coarse": outs[0], "depth_coarse": outs[1], "opacity_coarse": outs[2]}
    k = 3
    if N_importance > 0:
        res.update(rgb_fine=outs[3], depth_fine=outs[4], opacity_fine=outs[5])
        k = 6
    if target is not None:
        l4 = outs[k]
        res.update(loss=l4[2], psnr=l4[3].detach(), mse_coarse=l4[0].detach(), mse_fine=l4[1].detach())
    return res


# ---------------------------------------------------------------------------------------------
# Training a direct NeRF.forward call (reference models/nerf.py:83-124) for callers that render with their own code:
# one save-mode launch of the MLP kernel forward (nerfb200_nerf_forward_train), the sm_90a backward kernels of the
# render path seeded from the upstream (B, 4) gradient (nerfb200_nerf_backward).
class NerfTrainWorkspace(_Workspace):
    """Device workspace of one ``nerf_forward_train`` call over ``n`` samples, from a per-device pool.

    A call holds its workspace from its forward until its backward runs, or until its graph is freed without a
    backward (outputs used only for metrics under grad mode).  Pool policy: a call takes an idle workspace of
    exactly its ``n``; if there is none it first releases every idle workspace of another size on that device, then
    makes one.  So calls whose ``n`` varies (the last chunk of a point loop) do not accumulate workspaces: the pool
    holds the workspaces of the calls whose backward is pending, plus at most the idle ones of a single size."""

    _pool: Dict[int, List["NerfTrainWorkspace"]] = {}

    def __init__(self, dev: torch.device, n: int) -> None:
        nbytes = int(_lib.load().nerfb200_nerf_train_workspace_bytes(n))
        if nbytes == 0:
            raise ValueError(f"invalid sample count {n}")
        self.n = n
        super().__init__(dev, nbytes, "nerfb200_nerf_train_workspace_init", n)

    @classmethod
    def acquire(cls, dev: torch.device, n: int) -> "NerfTrainWorkspace":
        pool = cls._pool.setdefault(dev.index, [])
        for ws in pool:
            if not ws.busy and ws.n == n:
                ws.busy = True
                return ws
        pool[:] = [ws for ws in pool if ws.busy]
        ws = cls(dev, n)
        ws.busy = True
        pool.append(ws)
        return ws

    @classmethod
    def pool_size(cls, dev: torch.device) -> int:
        return len(cls._pool.get(dev.index, []))

    @classmethod
    def clear(cls) -> None:
        cls._pool.clear()


class FusedNerfFunction(torch.autograd.Function):
    """(model, x (B, 90) fp32 contiguous, 24 parameter tensors) -> (B, 4) [rgb, sigma]."""

    @staticmethod
    def forward(ctx, model, x, *params):
        n = x.shape[0]
        dev = x.device
        out = torch.empty(n, 4, dtype=torch.float32, device=dev)
        ctx.n = n
        ctx.lease = None
        if n > 0:
            blob = packed_weights(model)
            lease = _Lease(NerfTrainWorkspace.acquire(dev, n))
            _lib.call("nerfb200_nerf_forward_train", dev, x.data_ptr(), n, x.stride(0), blob.data_ptr(),
                      lease.ws.buf.data_ptr(), out.data_ptr())
            ctx.lease = lease
            ctx.blob = blob
        ctx.save_for_backward(*params)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        params = list(ctx.saved_tensors)
        if ctx.n == 0:
            return (None, None, *[torch.zeros_like(p) for p in params])
        lease = ctx.lease
        if lease is None or lease.ws is None:
            raise RuntimeError("the fused NeRF backward of this call has already run (its workspace is released "
                               "after one backward; retain_graph=True is not supported with autograd_impl='fused')")
        dev = params[0].device
        g = g.detach().to(torch.float32).contiguous()
        if g.data_ptr() % 16:
            g = g.clone()
        grads, [(pc, gc)] = _grad_buffers(params, dev)
        _lib.call("nerfb200_nerf_backward", dev, g.data_ptr(), ctx.n, ctx.blob.data_ptr(), pc, lease.ws.buf.data_ptr(), gc)
        lease.release()
        ctx.blob = None
        return (None, None, *grads)


def nerf_forward_train(model: torch.nn.Module, x: torch.Tensor) -> torch.Tensor:
    """``model(x)`` (reference models/nerf.py:83-124, ``sigma_only=False``) for training on the sm_90a kernels:
    ``x`` (B, 90) embedded xyz + direction -> (B, 4) [rgb, sigma].  Works for this package's ``NeRF`` (its
    ``forward`` calls this when ``autograd_impl == "fused"``) and, duck-typed through ``nerf_parameters``, for
    the reference's own ``models.nerf.NeRF`` instances.

    When a graph is needed (grad mode on, a parameter requires grad) the forward is one save-mode launch whose
    output equals ``nerf_forward_fused`` bit for bit, and ``backward`` fills the gradients of the 24 parameters
    with the sm_90a kernels.  Several calls before one ``backward()`` (coarse and fine nets, a chunked point loop,
    one model called twice) each hold their own workspace (``NerfTrainWorkspace``); their gradients are summed
    by autograd.  Otherwise this is ``nerf_forward_fused``.

    Raises ``ValueError`` for what the kernels do not do: ``x.requires_grad`` (no gradient with respect to the
    input), a non-default architecture, ``x`` not of shape (B, 90); ``RuntimeError`` for CPU tensors.  A backward
    whose per-sample gradients exceed their layer's fp16 range (device status 102), or are not finite (status 103: a
    non-finite input or upstream gradient), is reported by the next library call or ``nerfb200_check_status``."""
    if not x.is_cuda:
        raise RuntimeError("nerf_pl_b200.nerf_forward_train runs on CUDA tensors only (no CPU fallback)")
    if x.requires_grad:
        raise ValueError("autograd_impl='fused' computes no gradient with respect to x; detach the input or use "
                         "autograd_impl='torch'")
    if x.dim() != 2 or x.shape[1] != 90:
        raise ValueError(f"autograd_impl='fused' expects x of shape (B, 90), got {tuple(x.shape)}")
    is_default = getattr(model, "is_default_arch", None)
    if is_default is not None and not is_default():
        raise ValueError("autograd_impl='fused' supports the reference's default NeRF(D=8, W=256, 63, 27, skips=[4]) only")
    try:
        params = nerf_parameters(model)
    except (KeyError, AttributeError) as e:
        raise ValueError(f"autograd_impl='fused' supports the reference's default NeRF only (missing {e})") from None
    for p, shp in zip(params, _EXPECTED_SHAPES):
        if tuple(p.shape) != shp:
            raise ValueError(f"autograd_impl='fused' supports the reference's default NeRF only: parameter of shape "
                             f"{tuple(p.shape)}, expected {shp}")
        if p.device != x.device:
            raise ValueError("x and the NeRF parameters must be on the same device")
    if not (torch.is_grad_enabled() and any(p.requires_grad for p in params)):
        return nerf_forward_fused(model, x)
    return FusedNerfFunction.apply(model, x.detach().to(torch.float32).contiguous(), *params)


# ---------------------------------------------------------------------------------------------
# One training step (batch gather, fused render + loss, fused backward, capturable FusedAdam) as ONE CUDA graph.
_CAPTURED_SEEDS = 0


class CapturedTrainStep:
    """The reference's training step (train.py:103-117 with the optimiser step) captured once as a CUDA graph and
    replayed by ``step()``: no Python, no host-side kernel launches and no host synchronisation per step.

    ``models`` (coarse[, fine]) are trained on ``batches`` (a ``DeviceRayBatches`` or ``DeviceViewBatches``) by ``optimizer``, a
    ``FusedAdam(capturable=True)`` over their parameters; the other arguments are ``render_rays_loss``'s.  Each
    replay gathers the next batch from a device-resident epoch permutation at a device-side offset, renders it with
    the loss fused in, runs the backward and the Adam update.  Only full batches are used (``drop_last`` semantics:
    ``len(batches)`` with ``drop_last=True`` steps per epoch); when the host-side step count completes an epoch,
    ``step()`` draws the next permutation into the same buffer before the replay.  ``step()`` returns the device
    scalars ``(loss, psnr)`` of the step; they are overwritten by the next replay, so clone them to keep them.

    Random inputs: ``randoms=None`` draws the uniforms (and the noise when ``noise_std > 0``) with torch's CUDA
    generator, which advances across replays by itself.  ``randoms="kernel"`` (or ``{"seed": s}``) draws the
    uniforms inside the render kernel keyed by a device word (``seed_word``) that each replay increments, so replay
    k uses seed s + k.

    Construction runs ``warmup`` eager steps on a side stream (first-call set-up: library attributes, packed weight
    images, Adam state, the step's workspace), then restores the parameters, the Adam state and the seed they
    changed, sets the gradients to None and captures one step; it raises ``RuntimeError`` with torch's reason if
    the capture fails.  The step's training workspace belongs to this object for its whole life (it is not in
    ``TrainWorkspace``'s pool), so eager training calls of the same shape between replays never touch it.
    The gradients of every parameter the optimizer holds are set to None before the warm-up and before the capture,
    so parameters outside ``models`` (the fine model when ``N_importance == 0``, other groups) are neither warmed up
    nor updated by the replays.  Between replays the models' ``.grad`` are the graph's own buffers.  ``launches_per_step`` is the number of
    library kernels one replay runs (counted while capturing).

    ``occupancy`` (a ``nerf_pl_b200.OccupancyGrid``) captures the step with empty samples skipped, as
    ``render_rays_loss(..., occupancy=grid)`` computes it.  The step copies the grid's bits into a buffer it owns
    and uses a ``SkipTrainWorkspace`` of its own; ``set_occupancy(grid)`` copies a rebuilt grid of the same ``N``,
    ranges and ``dilate`` into that buffer between replays, and ``live_samples`` is the device int64 pair of the last
    replay's evaluated coarse and fine sample counts.

    ``occupancy`` may also be a ``nerf_pl_b200.DensityGrid``, which the step then keeps current itself: the grid's
    ``update`` from the last trained model (the fine one, or the coarse one when ``N_importance == 0``) is captured
    as a second graph, and ``step()`` replays it before the training step whenever ``steps % update_every == 0``
    (so replay 0 starts from a refreshed grid).  The training graph reads the density grid's own bits, and
    ``set_occupancy`` raises.  The warm-up also runs the update and restores the grid's density, bits and key.
    ``launches_per_update`` is the number of library kernels one update replay runs."""

    def __init__(self, models, batches, optimizer, N_samples: int = 64, use_disp: bool = False, perturb: float = 1.0,
                 noise_std: float = 1.0, N_importance: int = 64, white_back: bool = False, randoms=None,
                 warmup: int = 3, occupancy=None, update_every: Optional[int] = None):
        from .optim import FusedAdam
        global _CAPTURED_SEEDS
        if not (isinstance(optimizer, FusedAdam) and optimizer.capturable):
            raise ValueError("CapturedTrainStep needs FusedAdam(..., capturable=True): a non-capturable step reads "
                             "its step count on the host and would replay step 1 forever")
        if not isinstance(batches, _EpochBatches):
            raise TypeError("batches must be a nerf_pl_b200.DeviceRayBatches or DeviceViewBatches")
        S_c, K = int(N_samples), int(N_importance)
        if K > 0 and len(models) < 2:
            raise ValueError("N_importance > 0 needs a fine model (models[1])")
        B = batches.batch_size
        self.per_epoch = batches.samples_per_rank // B
        if self.per_epoch == 0:
            raise ValueError("the dataset has no full batch for this rank")
        self.models = list(models)[:2 if K > 0 else 1]
        self.params = _params_of(self.models, K)
        owned = {id(p) for g in optimizer.param_groups for p in g["params"]}
        if any(id(p) not in owned for p in self.params):
            raise ValueError("the optimizer does not hold every parameter of the models")
        self.batches, self.optimizer = batches, optimizer
        self.cfg = dict(N_samples=S_c, use_disp=bool(use_disp), perturb=float(perturb), noise_std=float(noise_std),
                        N_importance=K, white_back=bool(white_back))
        dev = batches.device
        self.seed_word = None
        if isinstance(randoms, str) or (isinstance(randoms, dict) and "seed" in randoms):
            if isinstance(randoms, str):
                if randoms != "kernel":
                    raise ValueError("randoms must be None, 'kernel' or {'seed': int}")
                _CAPTURED_SEEDS += 1
                s = (torch.initial_seed() * 0x9E3779B97F4A7C15 + _CAPTURED_SEEDS * 0xBF58476D1CE4E5B9) \
                    & 0xFFFFFFFFFFFFFFFF
            else:
                s = int(randoms["seed"]) & 0xFFFFFFFFFFFFFFFF
            s = s - (1 << 64) if s >= 1 << 63 else s          # the same 64 bits as an int64
            self.seed_word = torch.tensor(s, dtype=torch.int64, device=dev)
        elif randoms is not None:
            raise ValueError("randoms must be None, 'kernel' or {'seed': int}")
        from .density_grid import DensityGrid
        self._grid = self.density_grid = None
        self.update_every = None
        if isinstance(occupancy, DensityGrid):
            if update_every is None or int(update_every) != update_every or int(update_every) < 1:
                raise ValueError(f"occupancy=DensityGrid needs update_every, an int >= 1 (got {update_every!r})")
            self.update_every = int(update_every)
            self.density_grid = occupancy
            occupancy = occupancy.grid              # the training graph reads the density grid's own bits
        elif update_every is not None:
            raise ValueError("update_every needs occupancy=DensityGrid (a grid the step maintains itself)")
        if occupancy is None:
            self.workspace = TrainWorkspace(dev, B, S_c, K)
        else:
            from .culling import OccupancyGrid
            from .train_skip import SkipTrainWorkspace, check_shape
            check_shape(B, S_c, K)
            self._check_grid(occupancy, dev)
            r = occupancy.ranges
            self._grid = occupancy if self.density_grid is not None else \
                OccupancyGrid(occupancy.bits.clone(), occupancy.N, r[0:2], r[2:4], r[4:6], occupancy.dilate,
                              occupancy.levels)
            self.workspace = SkipTrainWorkspace(dev, B, S_c, K)
            self._live = torch.zeros(2, dtype=torch.int64, device=dev)
        self._perm = batches.next_permutation().clone()
        self._offset = torch.zeros((), dtype=torch.int64, device=dev)
        self._arange = torch.arange(B, device=dev)
        self.steps = 0                  # replays so far
        self.epoch = 0                  # epoch of the next replay (0-based)
        self._warm_and_capture(int(warmup), dev)

    def _body(self):
        """One step on the static buffers (run eagerly while warming up, then once under capture)."""
        c = self.cfg
        B, S_c, K = self._arange.shape[0], c["N_samples"], c["N_importance"]
        idx = self._perm.index_select(0, self._offset + self._arange)
        batch = self.batches.gather(idx)
        if self.seed_word is not None:
            pr = ur = None
            nc = torch.randn(B, S_c, device=idx.device) if c["noise_std"] > 0 else None
            nf = torch.randn(B, S_c + K, device=idx.device) if c["noise_std"] > 0 and K > 0 else None
        else:
            pr, nc, ur, nf = _draw_randoms(B, S_c, K, c["perturb"], c["noise_std"], idx.device, False)
        if self._grid is None:
            res = render_rays_train(self.models, batch["rays"], S_c, c["use_disp"], c["perturb"], c["noise_std"], K,
                                    c["white_back"], pr, nc, ur, nf, target=batch["rgbs"], rng_seed=self.seed_word,
                                    workspace=self.workspace)
        else:
            from .train_skip import render_rays_train_skip
            res = render_rays_train_skip(self.models, batch["rays"], S_c, c["use_disp"], c["perturb"], c["noise_std"],
                                         K, c["white_back"], pr, nc, ur, nf, batch["rgbs"], self._grid,
                                         rng_seed=self.seed_word, workspace=self.workspace, live_samples=self._live)
        res["loss"].backward()
        self.optimizer.step()
        self._offset.add_(B)
        if self.seed_word is not None:
            self.seed_word.add_(1)
        self.batch_indices = idx
        self.randoms = {k: v for k, v in (("perturb_rand", pr), ("noise_coarse", nc), ("u_rand", ur),
                                          ("noise_fine", nf)) if v is not None}
        return res["loss"].detach(), res["psnr"]

    def _warm_and_capture(self, warmup: int, dev) -> None:
        opt = self.optimizer
        with torch.no_grad():
            saved_p = [p.detach().clone() for p in self.params]
            saved_st = [{k: v.clone() for k, v in opt.state[p].items()} if len(opt.state.get(p, {})) else None
                        for p in self.params]
            saved_seed = None if self.seed_word is None else self.seed_word.clone()
            dg = self.density_grid
            saved_dg = None if dg is None else (dg._density.clone(), dg.bits.clone(), dg.key.clone())
        opt.sync_lr()
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(max(warmup, 1)):
                if dg is not None:
                    dg.update(self.models[-1])
                opt.zero_grad(set_to_none=True)     # every parameter the optimizer holds: no stale gradient steps
                self._offset.zero_()        # every warm-up step takes the first batch: never past the permutation
                self._body()
        torch.cuda.current_stream(dev).wait_stream(side)
        with torch.no_grad():               # the warm-up steps leave no trace
            for p, q in zip(self.params, saved_p):
                p.copy_(q)
            for p, snap in zip(self.params, saved_st):
                st = opt.state[p]
                for k in ("step", "exp_avg", "exp_avg_sq"):
                    if snap is None:
                        st[k].zero_()
                    else:
                        st[k].copy_(snap[k])
            self._offset.zero_()
            if saved_seed is not None:
                self.seed_word.copy_(saved_seed)
            if saved_dg is not None:
                for t, v in zip((dg._density, dg.bits, dg.key), saved_dg):
                    t.copy_(v)
        opt.zero_grad(set_to_none=True)     # captured: only the models' parameters get gradients, hence updates
        lib = _lib.load()
        self.update_graph = None
        self.launches_per_update = 0
        if dg is not None:
            self.update_graph = torch.cuda.CUDAGraph()
            n0 = lib.nerfb200_launch_count()
            try:
                with torch.cuda.graph(self.update_graph):
                    dg.update(self.models[-1])
            except Exception as e:
                raise RuntimeError(f"CapturedTrainStep: capturing the density grid update failed: {e}") from e
            self.launches_per_update = int(lib.nerfb200_launch_count() - n0)
        self.graph = torch.cuda.CUDAGraph()
        n0 = lib.nerfb200_launch_count()
        try:
            with torch.cuda.graph(self.graph):
                self._loss, self._psnr = self._body()
        except Exception as e:
            raise RuntimeError(f"CapturedTrainStep: capturing the training step failed: {e}") from e
        self.launches_per_step = int(lib.nerfb200_launch_count() - n0)

    @staticmethod
    def _check_grid(grid, dev) -> None:
        from .culling import OccupancyGrid
        if not isinstance(grid, OccupancyGrid):
            raise ValueError("occupancy must be a nerf_pl_b200.OccupancyGrid")
        if grid.device != dev:
            raise RuntimeError(f"the occupancy grid is on {grid.device}, the step trains on {dev}")

    @property
    def live_samples(self) -> Optional[torch.Tensor]:
        """The last replay's evaluated (coarse, fine) sample counts, a device int64 tensor (None without a grid)."""
        return None if self._grid is None else self._live

    def set_occupancy(self, grid) -> None:
        """Copy a rebuilt grid's bits into the step's own grid buffer (stream-ordered before the next replay).  The
        graph holds N, the ranges and dilate by value: a grid that differs in any of them is a ValueError."""
        if self._grid is None:
            raise ValueError("this step was captured without occupancy=")
        if self.density_grid is not None:
            raise ValueError("this step maintains its DensityGrid itself (update_every); set_occupancy does not apply")
        self._check_grid(grid, self._grid.device)
        g = self._grid
        if (grid.N, tuple(grid.ranges), grid.dilate) != (g.N, tuple(g.ranges), g.dilate):
            raise ValueError("set_occupancy needs a grid of the captured N, ranges and dilate "
                             f"({g.N}, {tuple(g.ranges)}, {g.dilate}); got ({grid.N}, {tuple(grid.ranges)}, "
                             f"{grid.dilate})")
        if grid.levels != g.levels:
            raise ValueError(f"set_occupancy needs a grid of the captured levels ({g.levels}); got {grid.levels}")
        g.bits.copy_(grid.bits)

    def step(self):
        """Replay one training step; returns the device scalars (loss, psnr) of this step."""
        reshuffle, epoch, _ = next_step_schedule(self.steps, self.per_epoch)
        if reshuffle:                       # the previous epoch is done: reshuffle outside the graph
            self._perm.copy_(self.batches.next_permutation())
            self._offset.zero_()
            self.epoch = epoch
        self.optimizer.sync_lr()
        if self.update_graph is not None and self.steps % self.update_every == 0:
            self.update_graph.replay()
        self.graph.replay()
        self.steps += 1
        return self._loss, self._psnr
