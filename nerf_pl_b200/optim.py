"""``FusedAdam``: torch.optim.Adam's update for all parameters in one sm_90a launch
(C ABI ``nerfb200_adam_step``).  Drop-in for the optimiser the reference builds in
``utils/__init__.py:16-18`` (``Adam(parameters, lr=hparams.lr, eps=eps, weight_decay=hparams.weight_decay)``):
same constructor arguments, same state (``step`` a 0-dim float32 CPU tensor per parameter, ``exp_avg``,
``exp_avg_sq``), so checkpoints move between the two in both directions.  Adam's arithmetic in fp32, bias-corrected,
L2 weight decay added to the gradient; no amsgrad / maximize.  The bias corrections come from the host in double
(csrc/bwd_kernels.cuh adam_kernel states where the result differs from torch's).

As in torch.optim.Adam, a parameter whose ``grad`` is None is skipped and keeps its own step count; parameters at
different step counts get their own bias corrections (one launch per distinct step).

``capturable=True`` (as in ``torch.optim.Adam(capturable=True)``): the step reads nothing on the host, so a CUDA graph
can capture and replay it (``nerf_pl_b200.training.CapturedTrainStep``).  ``step`` is then a 0-dim float32 tensor on
the parameter's device, the learning rate is read from a device scalar per group, and the bias corrections are formed
on the device (C ABI ``nerfb200_adam_step_dev``; one launch for all tensors whatever their step counts).
``group["lr"]`` stays a float that schedulers change as usual: each eager ``step()`` and each
``CapturedTrainStep.step()`` copies it into the device scalar when it has changed (``sync_lr``).  m and v are
bit-identical to the non-capturable update; p can differ by an ulp where the device ``pow`` rounds a bias correction
differently from the host's.  ``load_state_dict`` puts the step counts on the device (capturable) or the host (not
capturable), whichever form the checkpoint has, so checkpoints move between both forms and ``torch.optim.Adam``.
A captured graph holds the addresses of the state tensors: after ``load_state_dict`` capture a new graph."""
from __future__ import annotations

import ctypes

import torch

from . import _lib


def _check_tensor(t: torch.Tensor, p: torch.Tensor, contiguous: bool = True) -> None:
    """``t`` (``p`` itself, its gradient or a state tensor) is what the kernel can read for parameter ``p``;
    non-contiguous gradients are copied before the launch."""
    if t.is_sparse or not t.is_cuda or t.dtype != torch.float32 or (contiguous and not t.is_contiguous()) \
            or t.shape != p.shape or t.device != p.device:
        raise RuntimeError("FusedAdam needs contiguous float32 CUDA parameters and state with dense gradients")


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.0,
                 capturable: bool = False):
        if lr < 0 or eps < 0 or not 0 <= betas[0] < 1 or not 0 <= betas[1] < 1 or weight_decay < 0:
            raise ValueError("invalid Adam hyper-parameter")
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        if capturable:
            defaults["capturable"] = True
        super().__init__(params, defaults)
        self._cache = {}
        self._lr_dev = {}           # group index -> device fp32 scalar (capturable)
        self._lr_host = {}          # group index -> the float last copied into it

    @property
    def capturable(self) -> bool:
        return bool(self.defaults.get("capturable", False))

    def __setstate__(self, state):
        """Runs in ``load_state_dict`` (and unpickling): a number ``step`` (checkpoints of earlier versions) becomes
        a tensor as torch.optim.Adam stores it, on the parameter's device when capturable and on the host otherwise;
        the launch tables of the replaced state are dropped.  The mode is this optimiser's, not the checkpoint's."""
        super().__setstate__(state)
        cap = self.capturable
        for group in self.param_groups:
            if cap:
                group["capturable"] = True
            elif "capturable" in group:
                group["capturable"] = False
            for p in group["params"]:
                st = self.state.get(p, {})
                if len(st):
                    step = st["step"]
                    if not torch.is_tensor(step):
                        step = torch.tensor(float(step), dtype=torch.float32)
                    st["step"] = step.to(dtype=torch.float32, device=p.device if cap else "cpu")
        self._cache = {}
        self.__dict__.setdefault("_lr_dev", {})
        self._lr_host = {}

    def sync_lr(self) -> None:
        """Copy each group's ``lr`` into its device scalar where it has changed (capturable; a no-op otherwise).
        Not to be called while a graph is being captured: the copy is a host value."""
        if not self.capturable:
            return
        for gi, group in enumerate(self.param_groups):
            lr = float(group["lr"])
            t = self._lr_dev.get(gi)
            if t is None:
                dev = next((p.device for p in group["params"]), None)
                if dev is None:
                    continue
                t = torch.empty((), dtype=torch.float32, device=dev)
                self._lr_dev[gi] = t
                self._lr_host.pop(gi, None)
            if self._lr_host.get(gi) != lr:
                t.fill_(lr)
                self._lr_host[gi] = lr

    @staticmethod
    def _tables(ps, sts):
        """The pointer tables of one or more launches (at most 64 tensors each) over parameters ``ps``."""
        chunks = []
        for i0 in range(0, len(ps), 64):
            ch, cs = ps[i0:i0 + 64], sts[i0:i0 + 64]
            n = len(ch)
            arr = lambda vals: (ctypes.c_void_p * n)(*vals)
            chunks.append(dict(ps=ch, p=arr([p.data_ptr() for p in ch]), m=arr([s["exp_avg"].data_ptr() for s in cs]),
                               v=arr([s["exp_avg_sq"].data_ptr() for s in cs]),
                               numel=(ctypes.c_int64 * n)(*[p.numel() for p in ch])))
        return chunks

    def _cached_tables(self, gi, ps, sts, steps=None):
        """The launch tables of group ``gi`` (``_tables``; with the capturable step counts ``steps``, each chunk also
        gets their ``step`` table).  They hold raw pointers: rebuilt, after checking the tensors, whenever a parameter
        or a state tensor is another allocation."""
        key = (tuple([p.data_ptr() for p in ps]) + tuple([st["exp_avg"].data_ptr() for st in sts]) +
               tuple([st["exp_avg_sq"].data_ptr() for st in sts]))
        if steps is not None:
            key += tuple([s.data_ptr() for s in steps])
        cache = self._cache.get(gi)
        if cache is None or cache["key"] != key:
            for p, st in zip(ps, sts):
                for t in (p, p.grad, st["exp_avg"], st["exp_avg_sq"]):
                    _check_tensor(t, p, contiguous=t is not p.grad)
            chunks = self._tables(ps, sts)
            if steps is not None:
                for ch, i0 in zip(chunks, range(0, len(ps), 64)):
                    ch["step"] = (ctypes.c_void_p * len(ch["ps"]))(*[s.data_ptr() for s in steps[i0:i0 + 64]])
            cache = dict(key=key, chunks=chunks)
            self._cache[gi] = cache
        return cache["chunks"]

    @staticmethod
    def _grads(ch):
        """The chunk's gradients, made contiguous where they are not (the caller keeps them alive through the launch),
        and their pointer array."""
        gs = [p.grad if p.grad.is_contiguous() else p.grad.contiguous() for p in ch["ps"]]
        return gs, (ctypes.c_void_p * len(gs))(*[g.data_ptr() for g in gs])

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        cap = self.capturable
        if cap:
            if torch.cuda.is_current_stream_capturing():
                if len(self._lr_dev) < len(self.param_groups):
                    raise RuntimeError("FusedAdam(capturable=True): run one eager step before capturing a graph")
            else:
                self.sync_lr()
        for gi, group in enumerate(self.param_groups):
            if group.get("amsgrad") or group.get("maximize") or group.get("decoupled_weight_decay"):
                raise RuntimeError("FusedAdam has no amsgrad / maximize / decoupled weight decay")
            ps = [p for p in group["params"] if p.grad is not None]
            if not ps:
                continue
            sts = [self.state[p] for p in ps]
            for p, st in zip(ps, sts):
                if len(st) == 0:
                    st["step"] = torch.zeros((), dtype=torch.float32, device=p.device if cap else "cpu")
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                elif not torch.is_tensor(st["step"]):
                    st["step"] = torch.tensor(float(st["step"]), dtype=torch.float32)
            steps = [st["step"] for st in sts]
            if cap:
                self._step_dev(gi, group, ps, sts, steps)
                continue
            ts = [int(s) for s in steps]
            chunks = self._cached_tables(gi, ps, sts)
            if all(t == ts[0] for t in ts):
                launches = [(ts[0], chunks)]
            else:                                 # parameters at different step counts (some skipped a step)
                by_t = {}
                for i, t in enumerate(ts):
                    by_t.setdefault(t, []).append(i)
                launches = [(t, self._tables([ps[i] for i in ix], [sts[i] for i in ix])) for t, ix in by_t.items()]
            b1, b2 = group["betas"]
            for t, chunks in launches:
                for ch in chunks:
                    gs, garr = self._grads(ch)
                    _lib.call("nerfb200_adam_step", ps[0].device, len(gs), ch["p"], garr, ch["m"], ch["v"], ch["numel"],
                              float(group["lr"]), float(b1), float(b2), float(group["eps"]),
                              float(group["weight_decay"]), t + 1)
            torch._foreach_add_(steps, 1.0)
        return loss

    def _step_dev(self, gi, group, ps, sts, steps) -> None:
        """The capturable update of one group: no host value that changes from step to step enters the launch."""
        for st, p in zip(sts, ps):
            if not (torch.is_tensor(st["step"]) and st["step"].device == p.device and st["step"].dim() == 0
                    and st["step"].dtype == torch.float32):
                raise RuntimeError("FusedAdam(capturable=True) keeps each step count as a 0-dim float32 tensor on the "
                                   "parameter's device")
        lr = self._lr_dev[gi]
        b1, b2 = group["betas"]
        for ch in self._cached_tables(gi, ps, sts, steps):
            gs, garr = self._grads(ch)
            _lib.call("nerfb200_adam_step_dev", ps[0].device, len(gs), ch["p"], garr, ch["m"], ch["v"], ch["numel"],
                      lr.data_ptr(), ch["step"], float(b1), float(b2), float(group["eps"]),
                      float(group["weight_decay"]))
        torch._foreach_add_(steps, 1.0)
