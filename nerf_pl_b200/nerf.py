"""``Embedding`` and ``NeRF`` with the reference's constructor signature, attribute names,
parameter names/shapes and checkpoint keys (reference: models/nerf.py:4-38, 41-124), backed by
the sm_90a kernels of ``libnerf_pl_b200.so``.

The modules are ordinary ``nn.Module``s so ``utils.get_optimizer`` / ``load_ckpt``
(reference utils/__init__.py:10-30, 55-76) and pytorch-lightning keep working.  Inference
(``torch.no_grad`` / no parameter requires grad) runs the wgmma kernel through the C ABI;
when autograd needs a graph the layers are evaluated with torch ops so gradients exist, or, with
``model.autograd_impl = "fused"``, by the sm_90a training kernels (``training.nerf_forward_train``).
"""
from __future__ import annotations

import ctypes
from typing import List, Sequence

import torch
from torch import nn

from . import _lib
from ._lib import _stream_ptr  # noqa: F401  (defined in _lib; code that imported it from this module keeps working)

_PARAM_ORDER = (
    [(f"xyz_encoding_{i}", 0) for i in range(1, 9)]
    + [("xyz_encoding_final", None), ("dir_encoding", 0), ("sigma", None), ("rgb", 0)]
)


def nerf_parameters(model: nn.Module) -> List[torch.Tensor]:
    """The 24 parameter tensors of a NeRF in state_dict order (works for this package's NeRF and,
    by duck typing, for the reference's own ``models.nerf.NeRF``)."""
    # plain dict look-ups: nn.Module.__getattr__ and Sequential.__getitem__ are Python-level and
    # this runs on every render_rays call (the packed-image cache key)
    out = []
    mods = model._modules
    for name, idx in _PARAM_ORDER:
        mod = mods[name]
        lin = mod._modules[str(idx)] if idx is not None else mod
        ps = lin._parameters
        out.append(ps["weight"])
        out.append(ps["bias"])
    return out


_EXPECTED_SHAPES = (
    [(256, 63), (256,)] + [(256, 256), (256,)] * 3 + [(256, 319), (256,)] + [(256, 256), (256,)] * 3
    + [(256, 256), (256,), (128, 283), (128,), (1, 256), (1,), (3, 128), (3,)]
)


def _aligned_buffer(nbytes: int, dev) -> torch.Tensor:
    """``nbytes`` of device memory at a 1024-byte boundary: the library wants that alignment, torch's caching
    allocator guarantees 512.  The view keeps the larger allocation it is cut from alive."""
    raw = torch.empty(nbytes + 1024, dtype=torch.uint8, device=dev)
    off = (-raw.data_ptr()) % 1024
    return raw[off:off + nbytes]


class PackedWeights:
    """Device-resident packed image of one NeRF (csrc/layout.h).

    Refresh policy: while any parameter requires grad the image is re-packed on EVERY use — weights
    under training change between calls in ways no cheap key sees (the reference's own RAdam / Ranger
    update through ``p.data.copy_`` (utils/optimizers.py:88,163,242), which does not bump
    ``Tensor._version``); one 2.4 MB pack kernel per call is negligible next to a training step.
    Frozen networks (``requires_grad_(False)``, the inference configuration) are re-packed when a
    parameter's storage or ``_version`` changes (``load_state_dict``, ``.to(device)``, in-place
    ops); call ``invalidate_packed(model)`` after editing frozen weights through ``.data``."""

    def __init__(self) -> None:
        self.blob = None
        self.key = None
        self.ptrs = None

    def prepare(self, model: nn.Module) -> bool:
        """Everything except the pack launch; True if the image has to be (re)packed."""
        params = nerf_parameters(model)
        trainable = False
        for p in params:
            if p.requires_grad:
                trainable = True
                break
        ptrs = tuple([p.data_ptr() for p in params])          # also changes with the device
        key = None
        if not trainable:
            key = (ptrs, tuple([p._version for p in params]))
            if self.blob is not None and key == self.key:
                return False
        if ptrs != self.ptrs:            # first use / storage changed: validate, (re)allocate, rebuild the pointer table
            for p, shp in zip(params, _EXPECTED_SHAPES):
                if tuple(p.shape) != shp:
                    raise ValueError(
                        f"nerf_pl_b200 supports the reference's default NeRF(D=8, W=256, 63, 27, skips=[4]); "
                        f"got a parameter of shape {tuple(p.shape)}, expected {shp}")
                if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous():
                    raise ValueError("NeRF parameters must be contiguous float32 CUDA tensors")
            dev = params[0].device
            if self.blob is None or self.blob.device != dev:
                self.blob = _aligned_buffer(_lib.load().nerfb200_packed_bytes(), dev)
            self.arr = (ctypes.c_void_p * 24)(*[ctypes.c_void_p(a) for a in ptrs])
            self.blob_ptr = ctypes.c_void_p(self.blob.data_ptr())
            self.ptrs = ptrs
            self.dev = dev
        self.key = key
        return True

    def get(self, model: nn.Module) -> torch.Tensor:
        if self.prepare(model):
            _lib.call("nerfb200_pack_weights", self.dev, self.arr, self.blob_ptr)
        return self.blob


def invalidate_packed(model: nn.Module) -> None:
    """Force the next use of ``model`` to re-pack its weights (after editing frozen weights via ``.data``)."""
    cache = model.__dict__.get("_nerfb200_packed")
    if cache is not None:
        cache.key = None
        if cache.blob is not None:
            cache.key = ()


def _cache_of(model: nn.Module) -> PackedWeights:
    cache = model.__dict__.get("_nerfb200_packed")
    if cache is None:
        cache = PackedWeights()
        model.__dict__["_nerfb200_packed"] = cache
    return cache


def packed_weights(model: nn.Module) -> torch.Tensor:
    return _cache_of(model).get(model)


def packed_weights_pair(coarse: nn.Module, fine: nn.Module):
    """Packed images of both networks of a render; when both need (re)packing - every training step - ONE launch
    (``nerfb200_pack_weights_pair``) does it."""
    ca, cb = _cache_of(coarse), _cache_of(fine)
    if ca is cb:
        blob = ca.get(coarse)
        return blob, blob
    na, nb_ = ca.prepare(coarse), cb.prepare(fine)
    if na and nb_ and ca.dev == cb.dev:
        _lib.call("nerfb200_pack_weights_pair", ca.dev, ca.arr, ca.blob_ptr, cb.arr, cb.blob_ptr)
    else:
        for need, c in ((na, ca), (nb_, cb)):
            if need:
                _lib.call("nerfb200_pack_weights", c.dev, c.arr, c.blob_ptr)
    return ca.blob, cb.blob


class Embedding(nn.Module):
    """x -> (x, sin(2^k x), cos(2^k x), ...) with the input kept (reference models/nerf.py:4-38)."""

    def __init__(self, in_channels: int, N_freqs: int, logscale: bool = True):
        super().__init__()
        self.N_freqs = N_freqs
        self.in_channels = in_channels
        self.funcs = [torch.sin, torch.cos]
        self.out_channels = in_channels * (2 * N_freqs + 1)
        if logscale:
            self.freq_bands = 2 ** torch.linspace(0, N_freqs - 1, N_freqs)
        else:
            self.freq_bands = torch.linspace(1, 2 ** (N_freqs - 1), N_freqs)
        self.logscale = logscale

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        # embed_kernel reads (n, 3) rows and takes at most 16 frequencies; every other input goes through torch ops
        fused = (x.is_cuda and self.logscale and self.in_channels == 3 and x.dtype == torch.float32
                 and x.dim() == 2 and x.shape[-1] == 3 and self.N_freqs <= 16
                 and not (torch.is_grad_enabled() and x.requires_grad))
        if fused:
            xc = x.contiguous()
            out = torch.empty(xc.shape[0], self.out_channels, dtype=torch.float32, device=x.device)
            _lib.call("nerfb200_embed", x.device, xc.data_ptr(), xc.shape[0], self.N_freqs, out.data_ptr())
            return out
        if not x.is_cuda:
            raise RuntimeError("nerf_pl_b200.Embedding runs on CUDA tensors only (no CPU fallback)")
        parts = [x]
        for f in self.freq_bands.tolist():
            parts.append(torch.sin(f * x))
            parts.append(torch.cos(f * x))
        return torch.cat(parts, dim=-1)


class NeRF(nn.Module):
    """8x256 ReLU MLP with a skip at layer 5, sigma head, 256 linear, 283->128 direction layer and
    a sigmoid rgb head (reference models/nerf.py:41-124); same submodule names and state_dict keys.

    ``autograd_impl`` (instance attribute, not part of the state_dict) selects how a call that needs a
    gradient graph is evaluated: ``"torch"`` (default) with torch ops, ``"fused"`` with the sm_90a
    forward-with-save and backward kernels (``nerf_pl_b200.training.nerf_forward_train``; full
    ``(B, 90) -> (B, 4)`` output of the default architecture, no gradient with respect to ``x``)."""

    def __init__(self, D: int = 8, W: int = 256, in_channels_xyz: int = 63, in_channels_dir: int = 27,
                 skips: Sequence[int] = (4,)):
        super().__init__()
        self.autograd_impl = "torch"
        self.D, self.W = D, W
        self.in_channels_xyz, self.in_channels_dir = in_channels_xyz, in_channels_dir
        self.skips = list(skips)
        for i in range(D):
            fan_in = in_channels_xyz if i == 0 else (W + in_channels_xyz if i in self.skips else W)
            setattr(self, f"xyz_encoding_{i + 1}", nn.Sequential(nn.Linear(fan_in, W), nn.ReLU(True)))
        self.xyz_encoding_final = nn.Linear(W, W)
        self.dir_encoding = nn.Sequential(nn.Linear(W + in_channels_dir, W // 2), nn.ReLU(True))
        self.sigma = nn.Linear(W, 1)
        self.rgb = nn.Sequential(nn.Linear(W // 2, 3), nn.Sigmoid())

    def is_default_arch(self) -> bool:
        return (self.D == 8 and self.W == 256 and self.in_channels_xyz == 63
                and self.in_channels_dir == 27 and self.skips == [4])

    def forward(self, x: torch.Tensor, sigma_only: bool = False) -> torch.Tensor:
        if not x.is_cuda:
            raise RuntimeError("nerf_pl_b200.NeRF runs on CUDA tensors only (no CPU fallback)")
        impl = getattr(self, "autograd_impl", "torch")
        if impl not in ("torch", "fused"):
            raise ValueError(f"NeRF.autograd_impl must be 'torch' or 'fused', got {impl!r}")
        needs_graph = torch.is_grad_enabled() and (
            x.requires_grad or any(p.requires_grad for p in self.parameters()))
        if needs_graph and impl == "fused":
            if sigma_only:
                raise ValueError("autograd_impl='fused' trains the full (B, 90) -> (B, 4) output; sigma_only=True "
                                 "is not supported")
            from .training import nerf_forward_train
            return nerf_forward_train(self, x)
        if needs_graph or not self.is_default_arch():
            return nerf_forward_torch(self, x, sigma_only)
        return nerf_forward_fused(self, x, sigma_only)


def nerf_forward_fused(model: nn.Module, x: torch.Tensor, sigma_only: bool = False) -> torch.Tensor:
    """NeRF.forward through the wgmma tile engine (C ABI ``nerfb200_nerf_forward``)."""
    width = 63 if sigma_only else 90
    if x.dim() != 2 or x.shape[1] != width:
        raise ValueError(f"expected x of shape (B, {width}), got {tuple(x.shape)}")
    xc = x.detach().to(torch.float32).contiguous()
    blob = packed_weights(model)
    out = torch.empty(xc.shape[0], 1 if sigma_only else 4, dtype=torch.float32, device=x.device)
    _lib.call("nerfb200_nerf_forward", x.device, xc.data_ptr(), xc.shape[0], xc.stride(0), blob.data_ptr(),
              int(sigma_only), out.data_ptr())
    return out


def nerf_forward_torch(model: nn.Module, x: torch.Tensor, sigma_only: bool = False) -> torch.Tensor:
    """Differentiable evaluation with torch ops (autograd path; also the torch-fp32 check used by
    the GPU tests).  Same maths as reference models/nerf.py:100-124."""
    cx = model.in_channels_xyz
    enc = x[:, :cx]
    h = enc
    for i in range(model.D):
        if i in model.skips:
            h = torch.cat((enc, h), dim=-1)
        h = getattr(model, f"xyz_encoding_{i + 1}")(h)
    sigma = model.sigma(h)
    if sigma_only:
        return sigma
    feat = model.xyz_encoding_final(h)
    d = model.dir_encoding(torch.cat((feat, x[:, cx:]), dim=-1))
    return torch.cat((model.rgb(d), sigma), dim=-1)
