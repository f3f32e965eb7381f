"""SSIM as the reference's metrics.ssim defines it, restated for the tests.

metrics.ssim(pred, gt, reduction) = 1 - 2 * kornia.losses.ssim(pred, gt, 3, reduction).  kornia 0.2.0's published
SSIM (kornia/losses/ssim.py): a 3 x 3 window, the outer product of the size-3 Gaussian with sigma 1.5 normalised to
sum 1; each channel filtered with it (F.conv2d, zero padding 1, groups = C); sigma_x^2, sigma_y^2 and sigma_xy as
filter(x*y) - mu_x*mu_y; C1 = 0.01^2, C2 = 0.03^2; ssim_map = ((2 mu1 mu2 + C1)(2 sigma12 + C2)) /
((mu1^2 + mu2^2 + C1)(sigma1^2 + sigma2^2 + C2)); loss = clamp(1 - ssim_map, 0, 1) / 2, then 'mean' | 'sum' | 'none'.
Later kornia versions clamp (1 - ssim_map) / 2 instead; the two differ where ssim_map < 0.  No kornia build was
available to compare with: this follows the published source.

``ssim`` is the float64 numpy / scipy restatement the device kernel is checked against; ``ssim_torch_f32`` composes
the same steps in float32 torch the way kornia 0.2.0 composes them, to measure what float32 changes."""
import math

import numpy as np
from scipy import ndimage

C1, C2 = 0.01 ** 2, 0.03 ** 2
SIGMA = 1.5


def window():
    """(3, 3) float64: the normalised Gaussian's outer product."""
    g = np.exp(-(np.arange(3) - 1.0) ** 2 / (2 * SIGMA ** 2))
    g /= g.sum()
    return np.outer(g, g)


def _filter(img):
    """Each (b, c) plane of a (B, C, H, W) float64 array filtered with the window, zero padded."""
    return ndimage.correlate(img, window()[None, None], mode="constant", cval=0.0)


def ssim_map(pred, gt):
    """(B, C, H, W) float64 ssim_map."""
    x, y = np.asarray(pred, np.float64), np.asarray(gt, np.float64)
    assert x.ndim == 4 and x.shape == y.shape
    mu1, mu2 = _filter(x), _filter(y)
    mu1_sq, mu2_sq, mu1_mu2 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    sigma1_sq = _filter(x * x) - mu1_sq
    sigma2_sq = _filter(y * y) - mu2_sq
    sigma12 = _filter(x * y) - mu1_mu2
    return ((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))


def _reduce(loss, reduction):
    if reduction == "mean":
        return loss.mean()
    if reduction == "sum":
        return loss.sum()
    assert reduction == "none"
    return loss


def dssim(pred, gt, reduction="mean"):
    """kornia 0.2.0's loss: clamp(1 - ssim_map, 0, 1) / 2, reduced."""
    return _reduce(np.clip(1.0 - ssim_map(pred, gt), 0.0, 1.0) / 2.0, reduction)


def dssim_later_kornia(pred, gt, reduction="mean"):
    """Later kornia's loss, clamp((1 - ssim_map) / 2, 0, 1): not what this package computes."""
    return _reduce(np.clip((1.0 - ssim_map(pred, gt)) / 2.0, 0.0, 1.0), reduction)


def ssim(pred, gt, reduction="mean"):
    """metrics.ssim in float64: 1 - 2 * dssim."""
    return 1.0 - 2.0 * dssim(pred, gt, reduction)


def ssim_torch_f32(pred, gt, reduction="mean"):
    """metrics.ssim composed in float32 torch the way kornia 0.2.0 composes it (window from math.exp, matmul outer
    product, F.conv2d with groups = C, the same order of operations)."""
    import torch
    import torch.nn.functional as F
    img1, img2 = torch.as_tensor(pred, dtype=torch.float32), torch.as_tensor(gt, dtype=torch.float32)
    gauss = torch.tensor([math.exp(-(x - 3 // 2) ** 2 / float(2 * SIGMA ** 2)) for x in range(3)])
    gauss = gauss / gauss.sum()
    kernel2d = torch.matmul(gauss.unsqueeze(-1), gauss.unsqueeze(-1).t())
    c = img1.shape[1]
    kernel = kernel2d.repeat(c, 1, 1, 1)

    def filt(t):
        return F.conv2d(t, kernel, padding=1, groups=c)
    mu1, mu2 = filt(img1), filt(img2)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    sigma1_sq = filt(img1 * img1) - mu1_sq
    sigma2_sq = filt(img2 * img2) - mu2_sq
    sigma12 = filt(img1 * img2) - mu1_mu2
    smap = ((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))
    loss = torch.clamp(torch.tensor(1.) - smap, min=0, max=1) / 2.
    if reduction == "mean":
        loss = torch.mean(loss)
    elif reduction == "sum":
        loss = torch.sum(loss)
    return 1 - 2 * loss
