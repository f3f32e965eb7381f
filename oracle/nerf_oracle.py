"""CPU oracle: a numpy fp32 restatement of the reference's render_rays hot path.

TEST INFRASTRUCTURE ONLY.  Nothing in the product package (``nerf_pl_b200/``) imports this
module; only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` legs may use it, and only as the checker / the CPU arm.

Every function restates one reference function and cites it (paths relative to the
kwea123/nerf_pl checkout).  Parity is PINNED: ``tests/golden/*.npz`` hold outputs of the
reference's own Python path (models/rendering.py + models/nerf.py, imported read-only in the
build container by ``tests/golden/make_golden.py``); ``tests/test_oracle_golden.py`` checks this
restatement against them.

Weights are a dict of float32 arrays keyed like the reference state_dict
(``xyz_encoding_1.0.weight`` ... ``rgb.0.bias``; models/nerf.py:69-81).
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np

F32 = np.float32

LAYER_SHAPES = (
    [("xyz_encoding_1.0", 256, 63)]
    + [(f"xyz_encoding_{i}.0", 256, 256) for i in (2, 3, 4)]
    + [("xyz_encoding_5.0", 256, 319)]
    + [(f"xyz_encoding_{i}.0", 256, 256) for i in (6, 7, 8)]
    + [("xyz_encoding_final", 256, 256), ("dir_encoding.0", 128, 283), ("sigma", 1, 256), ("rgb.0", 3, 128)]
)
PARAM_KEYS = [f"{n}.{s}" for n, _, _ in LAYER_SHAPES for s in ("weight", "bias")]


# ------------------------------------------------------------------ synthetic weights / rays
def make_weights(seed: int, pseudo_trained: bool = True) -> Dict[str, np.ndarray]:
    """Deterministic weights with nn.Linear's default init distribution (U(-1/sqrt(fan_in), ..),
    models/nerf.py:63-81 use the torch default).  ``pseudo_trained`` scales the sigma / rgb heads
    so opacities and colours are non-degenerate (SURVEY.md section 8d) and pushes sigma away from 0."""
    rs = np.random.RandomState(seed)
    w = {}
    for name, out_f, in_f in LAYER_SHAPES:
        bound = 1.0 / np.sqrt(in_f)
        w[name + ".weight"] = rs.uniform(-bound, bound, size=(out_f, in_f)).astype(F32)
        w[name + ".bias"] = rs.uniform(-bound, bound, size=(out_f,)).astype(F32)
    if pseudo_trained:
        w["sigma.weight"] = (w["sigma.weight"] * F32(30.0)).astype(F32)
        w["sigma.bias"] = (w["sigma.bias"] + F32(0.5)).astype(F32)
        w["rgb.0.weight"] = (w["rgb.0.weight"] * F32(8.0)).astype(F32)
    return w


def make_rays(n: int, seed: int, kind: str = "blender") -> np.ndarray:
    """(n, 8) rays [o, d, near, far].  'blender': unit directions, near=2, far=6
    (datasets/blender.py:34-35, ray_utils.py:43); 'ndc': forward-facing NDC-style rays with
    non-unit directions, near=0, far=1 (datasets/llff.py:236-241)."""
    rs = np.random.RandomState(seed)
    if kind == "blender":
        o = np.array([0.0, 0.0, 4.0]) + 0.1 * rs.randn(n, 3)
        d = rs.randn(n, 3)
        d[:, 2] = -np.abs(d[:, 2]) - 1.0
        d /= np.linalg.norm(d, axis=-1, keepdims=True)
        near, far = np.full((n, 1), 2.0), np.full((n, 1), 6.0)
    elif kind == "ndc":
        o = np.concatenate([rs.uniform(-1, 1, (n, 2)), -np.ones((n, 1))], -1)
        d = np.concatenate([rs.uniform(-0.4, 0.4, (n, 2)), np.full((n, 1), 2.0)], -1)
        near, far = np.zeros((n, 1)), np.ones((n, 1))
    else:
        raise ValueError(kind)
    return np.concatenate([o, d, near, far], -1).astype(F32)


# ------------------------------------------------------------------ models/nerf.py
def embed(x: np.ndarray, n_freqs: int) -> np.ndarray:
    """Embedding.forward, logscale freq bands 2^k (models/nerf.py:16-17, 33-38)."""
    x = x.astype(F32)
    out = [x]
    for k in range(n_freqs):
        f = F32(2.0 ** k)
        out.append(np.sin(f * x, dtype=F32))
        out.append(np.cos(f * x, dtype=F32))
    return np.concatenate(out, -1)


def _linear(w: Dict[str, np.ndarray], name: str, x: np.ndarray) -> np.ndarray:
    y = x @ w[name + ".weight"].T          # fp32 GEMM (BLAS), nn.Linear = x W^T + b
    y += w[name + ".bias"]
    return y


def nerf_forward(w: Dict[str, np.ndarray], x: np.ndarray, sigma_only: bool = False) -> np.ndarray:
    """NeRF.forward (models/nerf.py:100-124): 8 ReLU layers with the encoded input re-injected
    in front of the hidden state before layer 5, raw sigma from layer 8, linear 'final',
    [final, dir] -> 128 ReLU -> 3 sigmoid; output [rgb, sigma]."""
    x = np.ascontiguousarray(x, dtype=F32)
    enc = np.ascontiguousarray(x[:, :63])
    h = enc
    for i in range(8):
        if i == 4:
            h = np.concatenate([enc, h], -1)
        h = _linear(w, f"xyz_encoding_{i + 1}.0", h)
        np.maximum(h, F32(0), out=h)
    sigma = _linear(w, "sigma", h)
    if sigma_only:
        return sigma
    feat = _linear(w, "xyz_encoding_final", h)
    d = _linear(w, "dir_encoding.0", np.concatenate([feat, x[:, 63:90]], -1))
    np.maximum(d, F32(0), out=d)
    pre = _linear(w, "rgb.0", d)
    rgb = (F32(1) / (F32(1) + np.exp(-pre, dtype=F32))).astype(F32)
    return np.concatenate([rgb, sigma], -1)


# ------------------------------------------------------------------ torchsearchsorted
def searchsorted(a: np.ndarray, v: np.ndarray, side: str = "left") -> np.ndarray:
    """Row-wise np.searchsorted with single-row broadcasting
    (torchsearchsorted/src/torchsearchsorted/utils.py:4-15, searchsorted.py:23-35).  A NaN in ``v`` gives 0, as the
    reference's CUDA kernel gives it (every comparison with NaN is false, so its search ends left of a[0]); numpy
    itself sorts NaN above +inf."""
    nrow = max(a.shape[0], v.shape[0])
    out = np.empty((nrow, v.shape[1]), dtype=np.int64)
    if a.shape[0] == 1:                 # one sorted row for every query: one call
        res = np.searchsorted(a[0], v.reshape(-1), side=side).reshape(v.shape)
        out[:] = res
    else:
        for r in range(nrow):
            out[r] = np.searchsorted(a[r], v[0 if v.shape[0] == 1 else r], side=side)
    out[np.broadcast_to(np.isnan(v), out.shape)] = 0
    return out


# ------------------------------------------------------------------ models/rendering.py
def linspace01(n: int) -> np.ndarray:
    """torch.linspace(0, 1, n) in fp32: step=(end-start)/(n-1); lower half start+step*i,
    upper half end-step*(n-1-i)."""
    if n == 1:
        return np.zeros(1, F32)
    step = F32(1.0) / F32(n - 1)
    i = np.arange(n)
    lo = (step * i.astype(F32)).astype(F32)
    hi = (F32(1.0) - (step * (n - 1 - i).astype(F32)).astype(F32)).astype(F32)
    return np.where(i < n // 2, lo, hi).astype(F32)


def sample_pdf(bins: np.ndarray, weights: np.ndarray, n_importance: int, det: bool = False,
               eps: float = 1e-5, u: Optional[np.ndarray] = None) -> np.ndarray:
    """sample_pdf (models/rendering.py:14-55).  ``u`` replaces the torch.rand draw (:39)."""
    n_rays, n_w = weights.shape
    weights = (weights.astype(F32) + F32(eps)).astype(F32)
    pdf = (weights / weights.sum(-1, keepdims=True, dtype=F32)).astype(F32)
    cdf = np.cumsum(pdf, -1, dtype=F32)
    cdf = np.concatenate([np.zeros_like(cdf[:, :1]), cdf], -1)
    if det:
        u = np.broadcast_to(linspace01(n_importance), (n_rays, n_importance))
    elif u is None:
        raise ValueError("non-deterministic sample_pdf needs the pre-drawn u")
    u = np.ascontiguousarray(u, dtype=F32)
    inds = searchsorted(cdf, u, side="right")
    below = np.maximum(inds - 1, 0)
    above = np.minimum(inds, n_w)
    cdf_b, cdf_a = np.take_along_axis(cdf, below, 1), np.take_along_axis(cdf, above, 1)
    bins_b, bins_a = np.take_along_axis(bins, below, 1), np.take_along_axis(bins, above, 1)
    denom = (cdf_a - cdf_b).astype(F32)
    denom[denom < F32(eps)] = F32(1)
    return (bins_b + ((u - cdf_b) / denom).astype(F32) * (bins_a - bins_b)).astype(F32)


def volume_render(sigmas, rgbs, z_vals, dirs, noise=None, noise_std=0.0, white_back=False):
    """The quadrature inside inference() (models/rendering.py:143-170).
    Returns (weights, rgb|None, depth|None, opacity)."""
    deltas = (z_vals[:, 1:] - z_vals[:, :-1]).astype(F32)
    deltas = np.concatenate([deltas, np.full_like(deltas[:, :1], 1e10)], -1)
    deltas = (deltas * np.linalg.norm(dirs.astype(F32), axis=-1, keepdims=True).astype(F32)).astype(F32)
    s = sigmas.astype(F32)
    if noise is not None:
        s = (s + noise.astype(F32) * F32(noise_std)).astype(F32)
    alphas = (F32(1) - np.exp(-deltas * np.maximum(s, F32(0)), dtype=F32)).astype(F32)
    shifted = np.concatenate([np.ones_like(alphas[:, :1]), (F32(1) - alphas + F32(1e-10)).astype(F32)], -1)
    weights = (alphas * np.cumprod(shifted, -1, dtype=F32)[:, :-1]).astype(F32)
    opacity = weights.sum(1, dtype=F32)
    if rgbs is None:
        return weights, None, None, opacity
    rgb = (weights[..., None] * rgbs).sum(-2, dtype=F32)
    depth = (weights * z_vals).sum(-1, dtype=F32)
    if white_back:
        rgb = (rgb + F32(1) - opacity[:, None]).astype(F32)
    return weights, rgb, depth, opacity


def _inference(w, xyz, dirs, dir_emb, z_vals, weights_only, noise, noise_std, white_back):
    """inference() closure (models/rendering.py:115-141) without the memory-only chunk loop."""
    n, S = z_vals.shape
    x = embed(xyz.reshape(-1, 3), 10)
    if not weights_only:
        x = np.concatenate([x, np.repeat(dir_emb, S, axis=0)], -1)
    out = nerf_forward(w, x, sigma_only=weights_only)
    if weights_only:
        return volume_render(out.reshape(n, S), None, z_vals, dirs, noise, noise_std, white_back)
    out = out.reshape(n, S, 4)
    return volume_render(out[..., 3], out[..., :3], z_vals, dirs, noise, noise_std, white_back)


def coarse_depths(rays, n_samples, use_disp=False, perturb=0.0, perturb_rand=None):
    """models/rendering.py:189-204."""
    near, far = rays[:, 6:7].astype(F32), rays[:, 7:8].astype(F32)
    t = linspace01(n_samples)[None, :]
    if not use_disp:
        z = (near * (F32(1) - t) + far * t).astype(F32)
    else:
        z = (F32(1) / (F32(1) / near * (F32(1) - t) + F32(1) / far * t)).astype(F32)
    z = np.broadcast_to(z, (rays.shape[0], n_samples)).astype(F32)
    if perturb > 0:
        mid = (F32(0.5) * (z[:, :-1] + z[:, 1:])).astype(F32)
        upper = np.concatenate([mid, z[:, -1:]], -1)
        lower = np.concatenate([z[:, :1], mid], -1)
        z = (lower + (upper - lower) * (F32(perturb) * perturb_rand.astype(F32))).astype(F32)
    return z


def render_rays(weights: List[Dict[str, np.ndarray]], rays: np.ndarray, N_samples=64, use_disp=False,
                perturb=0.0, noise_std=1.0, N_importance=0, white_back=False, test_time=False,
                randoms: Optional[Dict[str, np.ndarray]] = None, extras: bool = False):
    """render_rays (models/rendering.py:175-244).  ``randoms`` holds the pre-drawn tensors the
    reference takes from the global torch RNG: perturb_rand (:203), noise_coarse / noise_fine
    (:152), u_rand (:39)."""
    randoms = randoms or {}
    rays = rays.astype(F32)
    o, d = rays[:, 0:3], rays[:, 3:6]
    dir_emb = embed(d, 4)
    z = coarse_depths(rays, N_samples, use_disp, perturb, randoms.get("perturb_rand"))
    xyz = (o[:, None, :] + d[:, None, :] * z[:, :, None]).astype(F32)
    nz = randoms.get("noise_coarse") if noise_std > 0 else None
    res = {}
    if test_time:
        w_c, _, _, opac = _inference(weights[0], xyz, d, dir_emb, z, True, nz, noise_std, white_back)
        res["opacity_coarse"] = opac
    else:
        w_c, rgb, depth, opac = _inference(weights[0], xyz, d, dir_emb, z, False, nz, noise_std, white_back)
        res.update(rgb_coarse=rgb, depth_coarse=depth, opacity_coarse=opac)
    if extras:
        res["weights_coarse"] = w_c
    if N_importance > 0:
        mid = (F32(0.5) * (z[:, :-1] + z[:, 1:])).astype(F32)
        z_new = sample_pdf(mid, w_c[:, 1:-1], N_importance, det=(perturb == 0), u=randoms.get("u_rand"))
        z = np.sort(np.concatenate([z, z_new], -1), -1)
        xyz = (o[:, None, :] + d[:, None, :] * z[:, :, None]).astype(F32)
        nz = randoms.get("noise_fine") if noise_std > 0 else None
        w_f, rgb, depth, opac = _inference(weights[1], xyz, d, dir_emb, z, False, nz, noise_std, white_back)
        res.update(rgb_fine=rgb, depth_fine=depth, opacity_fine=opac)
        if extras:
            res.update(z_vals_fine=z, weights_fine=w_f)
    return res


# ------------------------------------------------------------------ datasets/ray_utils.py ("next" rows)
def generate_rays(H: int, W: int, focal: float, c2w: np.ndarray, near: float, far: float, ndc: bool = False):
    """get_ray_directions (datasets/ray_utils.py:16-22) + get_rays (:41-51) [+ get_ndc_rays (:75-92)
    with near plane 1.0 and near/far = 0/1 as datasets/llff.py:236-241] -> (H*W, 8) rays."""
    j, i = np.meshgrid(np.arange(H, dtype=F32), np.arange(W, dtype=F32), indexing="ij")
    dirs = np.stack([(i - F32(W / 2)) / F32(focal), -(j - F32(H / 2)) / F32(focal), -np.ones_like(i)], -1)
    c2w = np.asarray(c2w, dtype=F32).reshape(3, 4)
    d = (dirs.reshape(-1, 3) @ c2w[:, :3].T).astype(F32)
    d = (d / np.linalg.norm(d, axis=-1, keepdims=True)).astype(F32)
    o = np.broadcast_to(c2w[:, 3], d.shape).astype(F32)
    if ndc:
        n1 = F32(1.0)
        t = -(n1 + o[:, 2]) / d[:, 2]
        o = (o + t[:, None] * d).astype(F32)
        ox_oz, oy_oz = o[:, 0] / o[:, 2], o[:, 1] / o[:, 2]
        sx, sy = F32(-1.0 / (W / (2.0 * focal))), F32(-1.0 / (H / (2.0 * focal)))
        o2 = F32(1) + F32(2) * n1 / o[:, 2]
        o_n = np.stack([sx * ox_oz, sy * oy_oz, o2], -1)
        d_n = np.stack([sx * (d[:, 0] / d[:, 2] - ox_oz), sy * (d[:, 1] / d[:, 2] - oy_oz), F32(1) - o2], -1)
        o, d, near, far = o_n.astype(F32), d_n.astype(F32), 0.0, 1.0
    nf = np.broadcast_to(np.array([near, far], F32), (d.shape[0], 2))
    return np.concatenate([o, d, nf], -1).astype(F32)


def to_uint8(img: np.ndarray) -> np.ndarray:
    """eval.py:126-128."""
    return (np.clip(img, 0, 1) * 255).astype(np.uint8)


def psnr(a: np.ndarray, b: np.ndarray) -> float:
    """metrics.py:4-13: -10 log10(mse)."""
    mse = float(np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2))
    return float("inf") if mse == 0 else -10.0 * np.log10(mse)
