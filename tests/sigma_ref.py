"""References for the sigma field of mesh extraction (tests/test_gpu_mesh_field.py).

* The float64 positional encoding γ(x) and its fp16 rounding ``e16``, and the fp16 roundings the in-kernel
  encoding (``encode_row``: Cody-Waite reduction + MUFU sin/cos, then ``__float2half_rn``) may legitimately pick:
  a feature whose exact value lies within ``BAND`` of an fp16 rounding boundary may land on either side.
* ``sigma_grid_expected``: what ``sigma_grid`` must equal given the point-wise sigma of ``grid_positions``.
* ``sigma64`` / ``sigma_fp16_replay``: sigma in float64 (``nerf_forward_torch`` on a float64 copy of the
  module) and the fp16 replay of the kernel's roundings (fp16 weights and encoded input, each hidden layer's
  activations rounded to fp16, float64 accumulation, fp32 sigma head on the unrounded last layer), which sets
  the bar of the level-set check ``field_report``.
"""
from __future__ import annotations

import numpy as np
import torch

F64 = np.float64
N_FREQS = 10
# encoding error of the kernel: MUFU sin/cos 2^-21.4 plus the two-constant reduction (< 2^-22.5 up to
# |x| = 61, tests/test_sigma_ref.py), well inside 2^-20
BAND = 2.0 ** -20
MAX_ROUNDINGS = 16          # points with more candidate encodings (more than four two-way features) are excluded
# the level-set bars are these multiples of the fp16 replay's own distance from float64
BAR_MEAN, BAR_P99, BAR_MAX = 2.0, 2.0, 4.0


def embed64(xyz) -> np.ndarray:
    """γ(x) in float64 for fp32 positions (n, 3) -> (n, 63), models/nerf.py:33-38 order.  2^k x is exact in fp32,
    so these are the exact features of the positions the kernel sees."""
    x = np.asarray(xyz, np.float32).astype(F64)
    parts = [x]
    for k in range(N_FREQS):
        parts += [np.sin(2.0 ** k * x), np.cos(2.0 ** k * x)]
    return np.concatenate(parts, 1)


def e16(xyz) -> np.ndarray:
    """The float64 embedding rounded to fp16 (correctly rounded), as float32: exact under ``__float2half_rn``."""
    return embed64(xyz).astype(np.float16).astype(np.float32)


def _f16_range(v: np.ndarray, band: float):
    """fp16 values (as uint16 ordinal keys) that a value within ``band`` of v may round to: [lo, hi]."""
    lo = (v - band).astype(np.float16)
    hi = (v + band).astype(np.float16)
    return lo, hi


def _ordinal(h: np.ndarray) -> np.ndarray:
    """Monotone integer key of fp16 values (-0 and +0 share key 0)."""
    b = h.view(np.uint16).astype(np.int64)
    return np.where(b & 0x8000, -(b & 0x7FFF), b)


def _from_ordinal(o: np.ndarray) -> np.ndarray:
    b = np.where(o < 0, (-o) | 0x8000, o).astype(np.uint16)
    return b.view(np.float16)


def candidate_encodings(xyz, band: float = BAND, max_roundings: int = MAX_ROUNDINGS):
    """Every fp16 encoding the kernel may form for each point.

    Returns (rows (m, 63) float32, owner (m,) int64, n_choices (n,) int64): for each point with at most
    ``max_roundings`` combinations, all combinations of the fp16 values its features may round to (the first row of a
    point is ``e16``); points with more combinations own no row.  The three raw coordinates are rounded from fp32 by
    both paths and are never ambiguous."""
    v = embed64(xyz)
    n = len(v)
    lo, hi = _f16_range(v, band)
    olo, ohi = _ordinal(lo), _ordinal(hi)
    olo[:, :3] = ohi[:, :3] = _ordinal(v[:, :3].astype(np.float32).astype(np.float16))
    width = ohi - olo + 1
    choices = np.prod(np.minimum(width, max_roundings + 1), axis=1)
    base = v.astype(np.float16)
    base[:, :3] = v[:, :3].astype(np.float32).astype(np.float16)
    rows, owner = [base.astype(np.float32)[choices <= max_roundings]], [np.nonzero(choices <= max_roundings)[0]]
    amb = np.nonzero((choices > 1) & (choices <= max_roundings))[0]
    for p in amb:
        cols = np.nonzero(width[p] > 1)[0]
        grids = np.meshgrid(*[np.arange(olo[p, c], ohi[p, c] + 1) for c in cols], indexing="ij")
        combos = np.stack([g.ravel() for g in grids], 1)
        r = np.repeat(base[p][None].astype(np.float32), len(combos), 0)
        r[:, cols] = _from_ordinal(combos).astype(np.float32)
        keep = ~(r == base[p].astype(np.float32)).all(1)     # e16 itself is already the point's first row
        rows.append(r[keep])
        owner.append(np.full(int(keep.sum()), p))
    return np.concatenate(rows), np.concatenate(owner).astype(np.int64), choices


def matches_a_rounding(dev_sigma, cand_sigma, owner, n: int) -> np.ndarray:
    """(n,) bool: the device's sigma of a point equals (bit for bit) the sigma of one of its candidate encodings."""
    d = np.asarray(dev_sigma, np.float32).view(np.uint32)
    c = np.asarray(cand_sigma, np.float32).view(np.uint32)
    hit = np.zeros(n, bool)
    np.logical_or.at(hit, owner, c == d[owner])
    return hit


def sigma_grid_expected(point_sigma, N: int) -> np.ndarray:
    """(N, N, N) ``max(sigma, 0)`` of the grid_positions points in their flat order."""
    return np.maximum(np.asarray(point_sigma, np.float32), np.float32(0)).reshape(N, N, N)


def grid_mismatches(grid, point_sigma, N: int) -> int:
    """Number of grid entries that differ (bitwise) from ``sigma_grid_expected``."""
    a = np.ascontiguousarray(np.asarray(grid, np.float32)).view(np.uint32)
    b = np.ascontiguousarray(sigma_grid_expected(point_sigma, N)).view(np.uint32)
    return int((a != b).sum())


# ----------------------------------------------------------------------------------- float64 and fp16 replay
def _linear_weights(w, dtype, device):
    return {k: torch.as_tensor(np.asarray(v), dtype=dtype, device=device) for k, v in w.items()}


def sigma64(w, xyz, device="cpu", chunk: int = 1 << 18) -> np.ndarray:
    """Raw sigma in float64: ``nerf_forward_torch`` on a float64 copy of the module, float64 embedding."""
    from nerf_pl_b200.nerf import NeRF, nerf_forward_torch
    m = NeRF()
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in w.items()})
    m = m.double().to(device)
    out = []
    with torch.no_grad():
        for s in range(0, len(xyz), chunk):
            e = torch.from_numpy(embed64(xyz[s:s + chunk])).to(device)
            out.append(nerf_forward_torch(m, e, sigma_only=True)[:, 0].cpu().numpy())
    return np.concatenate(out) if out else np.zeros(0)


def _r16(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.float16).to(torch.float64)


def sigma_fp16_replay(w, xyz, device="cpu", chunk: int = 1 << 18, drop_relu: int = 0,
                      acc=torch.float64) -> np.ndarray:
    """Raw sigma with the kernel's roundings replayed in float64: fp16 encoded input and big-layer weights, each
    hidden layer's ReLU output rounded to fp16 (layer 8 feeds the fp32 sigma head unrounded), float64 sums.
    ``drop_relu = l`` leaves out layer l's ReLU (a defect the level-set bar must reject); ``acc = torch.float32``
    sums in fp32 instead, as the tensor cores do."""
    t = _linear_weights(w, torch.float64, device)
    W = [None] + [_r16(t[f"xyz_encoding_{l}.0.weight"]) for l in range(1, 9)]
    b = [None] + [t[f"xyz_encoding_{l}.0.bias"] for l in range(1, 9)]
    out = []
    with torch.no_grad():
        for s in range(0, len(xyz), chunk):
            x = torch.from_numpy(e16(xyz[s:s + chunk]).astype(F64)).to(device)
            h = x
            for l in range(1, 9):
                inp = torch.cat([x, h], 1) if l == 5 else h
                pre = ((inp.to(acc) @ W[l].T.to(acc)).to(torch.float64) + b[l].to(acc).to(torch.float64))
                a = pre if l == drop_relu else torch.relu(pre)
                h = a if l == 8 else _r16(a)
            out.append((h @ t["sigma.weight"][0] + t["sigma.bias"][0]).cpu().numpy())
    return np.concatenate(out) if out else np.zeros(0)


def error_stats(a, ref) -> dict:
    d = np.abs(np.asarray(a, F64) - np.asarray(ref, F64))
    return {"max": float(d.max()), "p99": float(np.quantile(d, 0.99)), "mean": float(d.mean())}


def field_report(dev, s64, rep, thr: float) -> dict:
    """Device sigma against float64 with bars from the fp16 replay of the same points.

    dev, s64, rep: sigma of the same points (the same ReLU applied to all three).  Returns the device's and the
    replay's error statistics, the bars, the points whose inside/outside call (sigma > thr) differs from
    float64's and whether each check holds: mean / p99 / max within BAR_MEAN / BAR_P99 / BAR_MAX times the replay's,
    and every point classified differently within the max bar of the threshold."""
    e_dev, e_rep = error_stats(dev, s64), error_stats(rep, s64)
    bars = {"mean": BAR_MEAN * e_rep["mean"], "p99": BAR_P99 * e_rep["p99"], "max": BAR_MAX * e_rep["max"]}
    flip = (np.asarray(dev, F64) > thr) != (np.asarray(s64, F64) > thr)
    flip_gap = float(np.abs(np.asarray(s64, F64)[flip] - thr).max()) if flip.any() else 0.0
    ok = {k: e_dev[k] <= bars[k] for k in bars}
    ok["flips"] = flip_gap <= bars["max"]
    return {"dev": e_dev, "replay": e_rep, "bars": bars, "flips": int(flip.sum()), "flip_gap": flip_gap, "ok": ok}


# ----------------------------------------------------------------------------------------- level set
def crossings(grid, thr: float):
    """Index-space crossing points (linear interpolation) of every sign-changing grid edge (inside: > thr), and the
    (n, 2) flat indices of each edge's endpoints, in marching cubes' vertex order."""
    s = np.asarray(grid, F64)
    inside = s > thr
    n0, n1, n2 = s.shape
    mask = np.zeros(s.shape + (3,), bool)
    mask[:-1, :, :, 0] = inside[:-1] != inside[1:]
    mask[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    mask[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    pi, pj, pk, ax = np.nonzero(mask)
    a = np.stack([pi, pj, pk], 1)
    b = a + np.eye(3, dtype=np.int64)[ax]
    f0, f1 = s[pi, pj, pk], s[b[:, 0], b[:, 1], b[:, 2]]
    pos = a.astype(F64)
    pos[np.arange(len(ax)), ax] += (thr - f0) / (f1 - f0)
    flat = lambda q: (q[:, 0] * n1 + q[:, 1]) * n2 + q[:, 2]
    return pos, np.stack([flat(a), flat(b)], 1)


def index_to_world(pos, N: int, x_range, y_range, z_range) -> np.ndarray:
    """Exact world position of index-space points of the sigma grid: axis 0 is y, axis 1 is x ('xy' meshgrid)."""
    def lin(r, t):
        return r[0] + t * (r[1] - r[0]) / (N - 1)
    return np.stack([lin(x_range, pos[:, 1]), lin(y_range, pos[:, 0]), lin(z_range, pos[:, 2])], 1)
