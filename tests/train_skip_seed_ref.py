"""Float64 restatement of the sparse compositing backward with the general seed (csrc/train_skip_kernels.cuh
train_skip_bwd_kernel, the seed of composite_bwd_kernel): upstream gradients of one pass's rgb, depth and opacity,
plus the fused MSE term when a target is given.  tests/train_skip_ref.py states the forward and the MSE-only backward.

Per ray:
  g  = g_rgb + [target] loss_grad * 2 (rgb_out - target) / (3 n_rays)
  gd = g_depth,  go = g_opacity - [white_back] sum_ch g
  dL/dw_i = <g, c_i> + gd z_i + go
and from there train_skip_ref.backward's formulas (skipped samples: sigma = 0, no noise, no gradient).
"""
import numpy as np


def backward(z, sigma, rgb, ev, dirs, noise, noise_std, white_back, g_rgb=None, g_depth=None, g_opacity=None,
             mse=None):
    """d L / d sigma (R, S) and d L / d rgb_pre (R, S, 3) of one pass in float64, 0 at skipped samples.  g_rgb (R, 3),
    g_depth (R), g_opacity (R): upstream gradients or None (0); mse: None or (rgb_out (R, 3), target (R, 3), n_rays,
    loss_grad)."""
    z = np.asarray(z, np.float64)
    R = z.shape[0]
    s = np.where(ev, np.asarray(sigma, np.float64) + (0.0 if noise is None else np.asarray(noise, np.float64) * noise_std),
                 0.0)
    c = np.where(ev[..., None], np.asarray(rgb, np.float64), 0.0)
    g = np.zeros((R, 3)) if g_rgb is None else np.asarray(g_rgb, np.float64).copy()
    if mse is not None:
        rgb_out, target, n_rays, loss_grad = mse
        g = g + loss_grad * 2.0 * (np.asarray(rgb_out, np.float64) - np.asarray(target, np.float64)) / (3.0 * n_rays)
    gd = np.zeros(R) if g_depth is None else np.asarray(g_depth, np.float64)
    go = np.zeros(R) if g_opacity is None else np.asarray(g_opacity, np.float64).copy()
    if white_back:
        go = go - g.sum(1)
    dn = np.linalg.norm(np.asarray(dirs, np.float64), axis=1)
    delta = np.concatenate([z[:, 1:] - z[:, :-1], np.full((R, 1), 1e10)], 1) * dn[:, None]
    e = np.exp(-delta * np.maximum(s, 0.0))
    alpha = 1.0 - e
    om = 1.0 - alpha + 1e-10
    T = np.cumprod(np.concatenate([np.ones((R, 1)), om], 1), 1)[:, :-1]
    w = alpha * T
    dw = (g[:, None, :] * c).sum(2) + gd[:, None] * z + go[:, None]
    a = w * dw
    after = np.cumsum(a[:, ::-1], 1)[:, ::-1] - a                   # sum over j > i
    dalpha = T * dw - after / om
    ds = np.where(ev & (s > 0), dalpha * delta * e, 0.0)
    dpre = np.where(ev[..., None], w[..., None] * g[:, None, :] * c * (1.0 - c), 0.0)
    return ds, dpre
