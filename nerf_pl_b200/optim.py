"""``FusedAdam``: torch.optim.Adam's update for all parameters in one sm_90a launch
(C ABI ``nerfb200_adam_step``).  Drop-in for the optimiser the reference builds in
``utils/__init__.py:16-18`` (``Adam(parameters, lr=hparams.lr, eps=eps, weight_decay=hparams.weight_decay)``):
same constructor arguments, same state (``step`` a 0-dim float32 CPU tensor per parameter, ``exp_avg``,
``exp_avg_sq``), so checkpoints move between the two in both directions.  Adam's arithmetic in fp32, bias-corrected,
L2 weight decay added to the gradient; no amsgrad / maximize.  The bias corrections come from the host in double
(csrc/bwd_kernels.cuh adam_kernel states where the result differs from torch's).

As in torch.optim.Adam, a parameter whose ``grad`` is None is skipped and keeps its own step count; parameters at
different step counts get their own bias corrections (one launch per distinct step)."""
from __future__ import annotations

import ctypes

import torch

from . import _lib
from .nerf import _stream_ptr


def _check_tensor(t: torch.Tensor, p: torch.Tensor, contiguous: bool = True) -> None:
    """``t`` (``p`` itself, its gradient or a state tensor) is what the kernel can read for parameter ``p``;
    non-contiguous gradients are copied before the launch."""
    if t.is_sparse or not t.is_cuda or t.dtype != torch.float32 or (contiguous and not t.is_contiguous()) \
            or t.shape != p.shape or t.device != p.device:
        raise RuntimeError("FusedAdam needs contiguous float32 CUDA parameters and state with dense gradients")


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.0):
        if lr < 0 or eps < 0 or not 0 <= betas[0] < 1 or not 0 <= betas[1] < 1 or weight_decay < 0:
            raise ValueError("invalid Adam hyper-parameter")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self._cache = {}

    def __setstate__(self, state):
        """Runs in ``load_state_dict`` (and unpickling): a number ``step`` (checkpoints of earlier versions) becomes
        a tensor as torch.optim.Adam stores it, and the launch tables of the replaced state are dropped."""
        super().__setstate__(state)
        for group in self.param_groups:
            for p in group["params"]:
                st = self.state.get(p, {})
                if len(st) and not torch.is_tensor(st["step"]):
                    st["step"] = torch.tensor(float(st["step"]), dtype=torch.float32)
        self._cache = {}

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

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        lib = _lib.load()
        for gi, group in enumerate(self.param_groups):
            if group.get("amsgrad") or group.get("maximize") or group.get("decoupled_weight_decay"):
                raise RuntimeError("FusedAdam has no amsgrad / maximize / decoupled weight decay")
            ps = [p for p in group["params"] if p.grad is not None]
            if not ps:
                continue
            sts = [self.state[p] for p in ps]
            for p, st in zip(ps, sts):
                if len(st) == 0:
                    st["step"] = torch.tensor(0.0, dtype=torch.float32)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                elif not torch.is_tensor(st["step"]):
                    st["step"] = torch.tensor(float(st["step"]), dtype=torch.float32)
            steps = [st["step"] for st in sts]
            ts = [int(s) for s in steps]
            # the tables hold raw pointers: rebuilt whenever a parameter or a state tensor is another allocation
            key = (tuple([p.data_ptr() for p in ps]) + tuple([st["exp_avg"].data_ptr() for st in sts]) +
                   tuple([st["exp_avg_sq"].data_ptr() for st in sts]))
            cache = self._cache.get(gi)
            if cache is None or cache["key"] != key:
                for p, st in zip(ps, sts):
                    for t in (p, p.grad, st["exp_avg"], st["exp_avg_sq"]):
                        _check_tensor(t, p, contiguous=t is not p.grad)
                cache = dict(key=key, chunks=self._tables(ps, sts), dev=ps[0].device)
                self._cache[gi] = cache
            if all(t == ts[0] for t in ts):
                launches = [(ts[0], cache["chunks"])]
            else:                                 # parameters at different step counts (some skipped a step)
                by_t = {}
                for i, t in enumerate(ts):
                    by_t.setdefault(t, []).append(i)
                launches = [(t, self._tables([ps[i] for i in ix], [sts[i] for i in ix])) for t, ix in by_t.items()]
            b1, b2 = group["betas"]
            with torch.cuda.device(cache["dev"]):
                for t, chunks in launches:
                    for ch in chunks:
                        gs = [p.grad if p.grad.is_contiguous() else p.grad.contiguous() for p in ch["ps"]]
                        garr = (ctypes.c_void_p * len(gs))(*[g.data_ptr() for g in gs])
                        _lib.check(lib.nerfb200_adam_step(len(gs), ch["p"], garr, ch["m"], ch["v"], ch["numel"],
                                                          float(group["lr"]), float(b1), float(b2), float(group["eps"]),
                                                          float(group["weight_decay"]), t + 1, _stream_ptr()),
                                   "nerfb200_adam_step")
            torch._foreach_add_(steps, 1.0)
        return loss
