"""The reference's image metrics on the device: ``ssim`` (metrics.py:15-20) and ``visualize_depth``
(utils/visualization.py:6-18), each one call into ``include/nerf_pl_b200.h``.  Definitions, provenance and
measured numbers: DESIGN.md "Image metrics"."""
from __future__ import annotations

import ctypes

import torch

from . import _lib

COLORMAP_JET = 2                       # cv2.COLORMAP_JET, visualize_depth's default cmap
_REDUCTIONS = {"mean": 0, "sum": 1, "none": 2}


def _cuda_float32(t, name: str, fn: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f"nerf_pl_b200.{fn} runs on CUDA tensors only (no CPU fallback): {name}")
    if t.dtype != torch.float32:
        raise ValueError(f"{fn}: {name} must be float32, got {t.dtype}")
    return t.detach()


def ssim(image_pred: torch.Tensor, image_gt: torch.Tensor, reduction: str = "mean") -> torch.Tensor:
    """Drop-in for metrics.ssim: ``1 - 2 * kornia.losses.ssim(image_pred, image_gt, 3, reduction)`` with kornia
    0.2.0's definition, in [-1, 1].  (B, C, H, W) float32 CUDA tensors of any strides (``rgb.view(H, W, 3)
    .permute(2, 0, 1)[None]`` is read in place).  'mean' / 'sum': a 0-dim tensor, computed without a host
    synchronisation; 'none': the (B, C, H, W) map."""
    if reduction not in _REDUCTIONS:
        raise ValueError(f"ssim: reduction must be 'mean', 'sum' or 'none', got {reduction!r}")
    x = _cuda_float32(image_pred, "image_pred", "ssim")
    y = _cuda_float32(image_gt, "image_gt", "ssim")
    if x.dim() != 4 or x.shape != y.shape:
        raise ValueError(f"ssim: image_pred and image_gt must have the same (B, C, H, W) shape, got "
                         f"{tuple(x.shape)} and {tuple(y.shape)}")
    if x.device != y.device:
        raise ValueError("ssim: image_pred and image_gt are on different devices")
    b, c, h, w = x.shape
    out = torch.empty(x.shape if reduction == "none" else (), dtype=torch.float32, device=x.device)
    ws = None
    if reduction != "none":
        ws = _lib.workspace(_lib.load().nerfb200_ssim_workspace_bytes(b, c, h, w), x.device)
    strides = [(ctypes.c_int64 * 4)(*t.stride()) for t in (x, y)]
    _lib.call("nerfb200_ssim", x.device, x.data_ptr(), strides[0], y.data_ptr(), strides[1], b, c, h, w,
              _REDUCTIONS[reduction], None if ws is None else ws.data_ptr(), 0 if ws is None else ws.numel(),
              out.data_ptr())
    return out


def visualize_depth(depth: torch.Tensor, cmap: int = COLORMAP_JET) -> torch.Tensor:
    """Drop-in for utils.visualization.visualize_depth with the default ``cmap=cv2.COLORMAP_JET``: (H, W) float32
    CUDA depth -> (3, H, W) float32 CUDA image, bit for bit the reference's, kept on the device.  The channels are in
    cv2's order (channel 0 is blue), as the reference returns them.  Any other ``cmap`` raises ValueError."""
    if cmap != COLORMAP_JET:
        raise ValueError(f"visualize_depth: only cmap=cv2.COLORMAP_JET ({COLORMAP_JET}) is supported, got {cmap!r}")
    d = _cuda_float32(depth, "depth", "visualize_depth")
    if d.dim() != 2:
        raise ValueError(f"visualize_depth: depth must be (H, W), got {tuple(d.shape)}")
    h, w = d.shape
    out = torch.empty(3, h, w, dtype=torch.float32, device=d.device)
    ws = _lib.workspace(_lib.load().nerfb200_visualize_depth_workspace_bytes(h, w), d.device)
    _lib.call("nerfb200_visualize_depth", d.device, d.data_ptr(), h, w, d.stride(0), d.stride(1), ws.data_ptr(),
              ws.numel(), out.data_ptr())
    return out
