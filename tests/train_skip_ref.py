"""Float64 restatement of the training step with empty samples skipped (nerf_pl_b200/train_skip.py, DESIGN.md
"Training with empty samples skipped"): compositing with skipped samples at sigma = 0 and no noise, and the compositing
backward over the evaluated samples only (csrc/train_skip_kernels.cuh train_skip_bwd_kernel).

Per ray, with depths z (S), |d|, network sigma s_i and colour c_i of the evaluated samples (ev_i):
  sigma_i = s_i + noise_i * noise_std if ev_i else 0
  delta_i = (z_{i+1} - z_i) |d|  (delta_{S-1} = 1e10 |d|),  alpha_i = 1 - exp(-delta_i relu(sigma_i))
  w_i = alpha_i prod_{j<i} (1 - alpha_j + 1e-10);  rgb = sum w_i c_i (+ 1 - sum w_i with white_back)
The loss is losses.py's mean over rays and channels; its gradient seed is 2 (rgb - target) / (3 n_rays).
"""
import numpy as np
import torch


def forward(z, samples, ev, rays, noise, noise_std, white_back):
    """float64 rgb (R, 3), depth, opacity, weights (R, S) of one pass from the device's depths z (R, S), samples
    (R, S, 4) [rgb, sigma] (0 where skipped) and evaluated set ev (R, S)."""
    z = np.asarray(z, np.float64)
    s = np.asarray(samples, np.float64)[..., 3].copy()
    if noise is not None and noise_std > 0:
        s = s + np.asarray(noise, np.float64) * noise_std
    s = np.where(ev, s, 0.0)
    c = np.asarray(samples, np.float64)[..., :3]
    d = np.asarray(rays, np.float64)[:, 3:6]
    delta = np.concatenate([z[:, 1:] - z[:, :-1], np.full((z.shape[0], 1), 1e10)], 1) * np.linalg.norm(d, axis=1)[:, None]
    with np.errstate(over="ignore", invalid="ignore"):
        alpha = 1.0 - np.exp(-delta * np.maximum(s, 0.0))
    trans = np.cumprod(np.concatenate([np.ones((z.shape[0], 1)), 1.0 - alpha + 1e-10], 1), 1)[:, :-1]
    w = alpha * trans
    opac = w.sum(1)
    rgb = (w[..., None] * c).sum(1)
    if white_back:
        rgb = rgb + (1.0 - opac)[:, None]
    return {"rgb": rgb, "depth": (w * z).sum(1), "opacity": opac, "weights": w}


def assert_close(ref, got, weights=None, ref_weights=False, tol=2e-5):
    """The float32 device values against the float64 restatement: rgb / opacity / weights within `tol` absolute,
    depth within `tol` relative to the largest depth."""
    for k in ("rgb", "opacity"):
        err = np.abs(np.asarray(got[k], np.float64) - ref[k]).max()
        assert err <= tol, (k, err)
    scale = max(1.0, np.abs(ref["depth"]).max())
    err = np.abs(np.asarray(got["depth"], np.float64) - ref["depth"]).max()
    assert err <= tol * scale, ("depth", err)
    if ref_weights:
        err = np.abs(np.asarray(weights, np.float64) - ref["weights"]).max()
        assert err <= tol, ("weights", err)


def backward(z, sigma, rgb, ev, dirs, noise, noise_std, white_back, rgb_out, target, n_rays):
    """Closed-form float64 d loss / d sigma (R, S) and d loss / d rgb_pre (R, S, 3) of the network outputs of one
    pass (composite_bwd_kernel's formulas), 0 at skipped samples.  sigma, rgb: the network's raw sigma and sigmoid
    colour (values at skipped samples are ignored)."""
    z = np.asarray(z, np.float64)
    s = np.where(ev, np.asarray(sigma, np.float64) + (0.0 if noise is None else np.asarray(noise, np.float64) * noise_std),
                 0.0)
    c = np.where(ev[..., None], np.asarray(rgb, np.float64), 0.0)
    g = 2.0 * (np.asarray(rgb_out, np.float64) - np.asarray(target, np.float64)) / (3.0 * n_rays)
    go = -g.sum(1) if white_back else np.zeros(z.shape[0])
    dn = np.linalg.norm(np.asarray(dirs, np.float64), axis=1)
    delta = np.concatenate([z[:, 1:] - z[:, :-1], np.full((z.shape[0], 1), 1e10)], 1) * dn[:, None]
    e = np.exp(-delta * np.maximum(s, 0.0))
    alpha = 1.0 - e
    om = 1.0 - alpha + 1e-10
    T = np.cumprod(np.concatenate([np.ones((z.shape[0], 1)), om], 1), 1)[:, :-1]
    w = alpha * T
    dw = (g[:, None, :] * c).sum(2) + go[:, None]
    a = w * dw
    after = np.cumsum(a[:, ::-1], 1)[:, ::-1] - a                   # sum over j > i
    dalpha = T * dw - after / om
    ds = np.where(ev & (s > 0), dalpha * delta * e, 0.0)
    dpre = np.where(ev[..., None], w[..., None] * g[:, None, :] * c * (1.0 - c), 0.0)
    return ds, dpre


def composite_torch(z, sigma, rgb, dirs, white_back):
    """Differentiable float64 compositing (torch) of sigma (R, S) (noise and skipping already applied), rgb (R, S, 3)."""
    delta = torch.cat([z[:, 1:] - z[:, :-1], torch.full_like(z[:, :1], 1e10)], 1) * dirs.norm(dim=1, keepdim=True)
    alpha = 1 - torch.exp(-delta * torch.relu(sigma))
    trans = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1 - alpha + 1e-10], 1), 1)[:, :-1]
    w = alpha * trans
    opac = w.sum(1)
    c = (w[..., None] * rgb).sum(1)
    if white_back:
        c = c + (1 - opac)[:, None]
    return c, (w * z).sum(1), opac


BWD_BAR = 1e-3      # max error / max |reference| of d sigma and of d rgb_pre (tests/train_tape.py BARS["composite"])


def backward_errors(ds_rows, dp_rows, ev, ds_ref, dp_ref):
    """Max error over the pass's largest reference value of the device's per-row d sigma (rows) and d rgb_pre
    (rows, 3) against the float64 reference (R, S) / (R, S, 3), rows being the evaluated samples (R, S) in ray-major,
    depth-index order.  The reference must be 0 at every skipped sample (no row carries its gradient)."""
    ds_rows = np.asarray(ds_rows, np.float64)
    dp_rows = np.asarray(dp_rows, np.float64)
    assert not ds_ref[~ev].any() and not dp_ref[~ev].any()
    es = np.abs(ds_rows - ds_ref[ev]).max(initial=0.0) / max(np.abs(ds_ref).max(initial=0.0), 1e-30)
    ep = np.abs(dp_rows - dp_ref[ev]).max(initial=0.0) / max(np.abs(dp_ref).max(initial=0.0), 1e-30)
    return float(es), float(ep)
