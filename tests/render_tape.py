"""Numpy emulation of the render kernel's resampling stages and float64 references of its fp32 stages.

The hierarchical resampling of the fused render kernel (csrc/render_kernel.cuh pdf_to_cdf_ray, inverse_cdf and the
rank merge) and of the stand-alone sample_pdf_kernel (csrc/aux_kernels.cuh) uses only correctly rounded fp32
operations (explicit __f*_rn, plain adds, the exact x 0.5), so it is reproduced here BIT FOR BIT from the kernel's
own inputs: its coarse compositing weights and coarse depths.  Every operation below is one float32 operation in the
kernel's order:

  * `cdf_fused`: the warp's strided partial sums + xor butterfly for the total, `per` = ceil(nw / 32) contiguous
    samples per lane summed in order, a Hillis-Steele inclusive scan (shfl_up by 1, 2, 4, ..), then excl + loc[p];
  * `cdf_standalone`: the same total, then lane 0 adds the pdf sequentially;
  * `inverse_cdf`: the kernel's own lo / hi / mid search (exact also on a cdf that is not monotone), the clamps, the
    denom < 1e-5 -> 1 rule and the lerp between bin mid-points;
  * `z_fine`: u (tensor, Philox replica or linspace), inverse_cdf, sort(cat(z_coarse, z_new)); it also reports the
    rays on which the merge takes its exhaustive-count branch (a list with an inversion).

Compositing uses expf (not correctly rounded), so it is held to fp32-rounding bars against float64 (`composite64`)
on the device's own sigma / rgb / depths instead.  `sample_pdf64` is the float64 resampling with a per-sample
conditioning flag.  Imports nothing from the product: used by tests/test_render_tape.py (CPU) and
tests/test_gpu_render_stages.py.
"""
from __future__ import annotations

from typing import Optional

import numpy as np

F32, F64 = np.float32, np.float64
EPS_W = F32(1e-5)        # the weight padding of sample_pdf (models/rendering.py:28) and its denom threshold (:50)
U32 = 2.0 ** -24         # unit roundoff of float32
LANES = 32
# Defects the CPU tests inject into the emulation (each must be rejected by the comparators).
DEFECTS = ("w_shift", "side_left", "no_eps", "no_denom_rule", "drop_coarse", "segment")


def _butterfly_total(part):
    """warp_sum: xor butterfly over the 32 lanes of (R, 32) partials; every lane ends with the same value."""
    v = part.astype(F32)
    lanes = np.arange(LANES)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[:, lanes ^ o]).astype(F32)
    return v[:, 0]


def _strided_total(wp):
    """The total of the padded weights wp (R, nw): lane l adds wp[l], wp[l + 32], .. in order, then the butterfly."""
    R, nw = wp.shape
    part = np.zeros((R, LANES), F32)
    for i in range(nw):
        part[:, i % LANES] = (part[:, i % LANES] + wp[:, i]).astype(F32)
    return _butterfly_total(part)


def cdf_fused(w, defect: Optional[str] = None):
    """pdf_to_cdf_ray on the compositing weights w (R, S) of the coarse pass -> cdf (R, S - 1), cdf[:, 0] = 0."""
    w = np.asarray(w, F32)
    R, S = w.shape
    nw = S - 2
    off = 0 if defect == "w_shift" else 1
    eps = F32(0) if defect == "no_eps" else EPS_W
    wp = (w[:, off:off + nw] + eps).astype(F32)
    total = _strided_total(wp)
    per = (nw + 31) >> 5
    shift = 1 if defect == "segment" else 0        # lane segments start one sample late
    loc = np.zeros((R, LANES, per), F32)
    run = np.zeros((R, LANES), F32)
    idx = np.zeros((LANES, per), np.int64)
    for p in range(per):
        i = np.arange(LANES) * per + p + shift
        idx[:, p] = i
        ok = i < nw
        pdf = np.zeros((R, LANES), F32)
        pdf[:, ok] = (wp[:, i[ok]] / total[:, None]).astype(F32)
        run = (run + pdf).astype(F32)
        loc[:, :, p] = run
    incl = run.copy()
    lanes = np.arange(LANES)
    for o in (1, 2, 4, 8, 16):
        up = incl[:, np.maximum(lanes - o, 0)]
        incl = np.where(lanes[None, :] >= o, (incl + up).astype(F32), incl)
    excl = np.concatenate([np.zeros((R, 1), F32), incl[:, :-1]], 1)
    cdf = np.zeros((R, S - 1), F32)
    for p in range(per):
        i = idx[:, p]
        ok = i < nw
        cdf[:, i[ok] + 1] = (excl[:, ok] + loc[:, ok, p]).astype(F32)
    return cdf


def cdf_standalone(w):
    """sample_pdf_kernel's cdf from the weights w (R, nw): total as in the fused kernel, then lane 0 adds the pdf
    in order -> cdf (R, nw + 1)."""
    w = np.asarray(w, F32)
    R, nw = w.shape
    wp = (w + EPS_W).astype(F32)
    total = _strided_total(wp)
    cdf = np.zeros((R, nw + 1), F32)
    run = np.zeros(R, F32)
    for i in range(nw):
        run = (run + (wp[:, i] / total).astype(F32)).astype(F32)
        cdf[:, i + 1] = run
    return cdf


def bins_from_depths(z):
    """Bin mid-points 0.5 (z[k] + z[k+1]) as the fused kernel forms them (models/rendering.py:225)."""
    z = np.asarray(z, F32)
    return (F32(0.5) * (z[:, :-1] + z[:, 1:]).astype(F32)).astype(F32)


def search_right(cdf, u, defect: Optional[str] = None):
    """The kernel's binary search: lo = 0, hi = nw + 1; cdf[mid] <= u -> lo = mid + 1 (searchsorted 'right')."""
    R, n = cdf.shape
    lo = np.zeros(u.shape, np.int64)
    hi = np.full(u.shape, n, np.int64)
    rows = np.arange(R)[:, None]
    while True:
        act = lo < hi
        if not act.any():
            return lo
        mid = (lo + hi) >> 1
        c = cdf[rows, np.minimum(mid, n - 1)]
        go = (c < u) if defect == "side_left" else (c <= u)
        lo = np.where(act & go, mid + 1, lo)
        hi = np.where(act & ~go, mid, hi)


def inverse_cdf(cdf, bins, u, defect: Optional[str] = None):
    """inverse_cdf / the second half of sample_pdf_kernel: cdf (R, nw + 1), bins (R, nw + 1), u (R, K) -> (R, K)."""
    cdf, bins, u = np.asarray(cdf, F32), np.asarray(bins, F32), np.asarray(u, F32)
    nw = cdf.shape[1] - 1
    lo = search_right(cdf, u, defect)
    below = np.maximum(lo - 1, 0)
    above = np.minimum(lo, nw)
    rows = np.arange(cdf.shape[0])[:, None]
    c0, c1 = cdf[rows, below], cdf[rows, above]
    b0, b1 = bins[rows, below], bins[rows, above]
    denom = (c1 - c0).astype(F32)
    if defect != "no_denom_rule":
        denom = np.where(denom < EPS_W, F32(1), denom).astype(F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = ((u - c0).astype(F32) / denom).astype(F32)
    return (b0 + (t * (b1 - b0).astype(F32)).astype(F32)).astype(F32)


def linspace01(n: int):
    """csrc/render_kernel.cuh linspace01 (= torch.linspace(0, 1, n) in fp32)."""
    if n <= 1:
        return np.zeros(max(n, 0), F32)
    step = F32(1) / F32(n - 1)
    i = np.arange(n)
    lo = (step * i.astype(F32)).astype(F32)
    hi = (F32(1) - (step * (n - 1 - i).astype(F32)).astype(F32)).astype(F32)
    return np.where(i < n // 2, lo, hi).astype(F32)


def fine_uniforms(n_rays: int, K: int, perturb: float, u_rand=None, seed: Optional[int] = None, ray0: int = 0):
    """The u the kernel inverts: the u_rand tensor, the Philox stream 1 (rng_in_kernel), or linspace when perturb = 0."""
    if perturb <= 0:
        return np.broadcast_to(linspace01(K), (n_rays, K)).copy()
    if seed is not None:
        from tests import philox
        return philox.uniform(seed, n_rays, K, 1, ray0)
    return np.asarray(u_rand, F32)


def z_fine(w_coarse, z_coarse, u, defect: Optional[str] = None):
    """The fused kernel's fine depths from its own coarse weights (R, S), coarse depths (R, S) and u (R, K).
    Returns (z_fine (R, S + K), z_new in the kernel's slot order (R, K), exhaustive (R,) bool: the ray has an
    inversion in one of the two lists, so the merge of its group counts ranks exhaustively)."""
    zc = np.asarray(z_coarse, F32)
    cdf = cdf_fused(w_coarse, defect)
    us = np.sort(np.asarray(u, F32), axis=1, kind="stable")      # the slot of u_j is its rank (ties by index)
    znew = inverse_cdf(cdf, bins_from_depths(zc), us, defect)
    if defect == "drop_coarse":                                     # one coarse depth lost, a new one doubled
        zc = np.concatenate([zc[:, :1], zc[:, 2:], znew[:, -1:]], 1)
    exhaustive = (zc[:, 1:] < zc[:, :-1]).any(1) | (znew[:, 1:] < znew[:, :-1]).any(1)
    return np.sort(np.concatenate([zc, znew], 1), 1), znew, exhaustive


# ------------------------------------------------------------------------------------------- float64 references
def sample_pdf64(bins, w, u, sequential: bool = False):
    """sample_pdf (models/rendering.py:14-55) in float64 on the fp32 inputs bins (R, nw + 1), w (R, nw), u (R, K);
    `sequential`: the cdf is one running sum (sample_pdf_kernel), not the fused kernel's lane segments and scan.
    Returns (z (R, K), flagged (R, K) bool, bar (R, K)).

    A sample is flagged when fp32 may legitimately pick another bin or branch than float64: u within the fp32
    error of a cdf knot, or c1 - c0 within the error of the two knots of the 1e-5 threshold.  The error of a knot c
    is `tol` = 2 (a + 2) 2^-24 c: a sum of positive terms along a = per + 6 additions (nw + 5 for a running sum), the
    pdf division and the total's relative error.  With trained weights the threshold case is common above the surface: an empty bin
    has pdf ~ 1e-5 / total, and two knots near 1 carry ~1e-7 each.  There float64 and fp32 may differ by up to a
    bin width.  Elsewhere fp32 must agree with float64 to `bar`: the bin width times the relative error the knot
    errors make in (u - c0) / denom, plus 4 ulps of the result."""
    bins, w, u = np.asarray(bins, F64), np.asarray(w, F64), np.asarray(u, F64)
    R, nw = w.shape
    wp = w + 1e-5
    cdf = np.concatenate([np.zeros((R, 1)), np.cumsum(wp / wp.sum(1, keepdims=True), 1)], 1)
    rows = np.arange(R)[:, None]
    inds = np.stack([np.searchsorted(cdf[r], u[r], side="right") for r in range(R)]) if R else np.zeros(u.shape, int)
    below, above = np.maximum(inds - 1, 0), np.minimum(inds, nw)
    c0, c1 = cdf[rows, below], cdf[rows, above]
    b0, b1 = bins[rows, below], bins[rows, above]
    d = c1 - c0
    branch = d < 1e-5
    den = np.where(branch, 1.0, d)
    z = b0 + (u - c0) / den * (b1 - b0)
    a = nw + 5 if sequential else (nw + 31) // 32 + 6
    tol = (a + 2) * 2.0 * U32 * cdf
    near_knot = (np.abs(u[:, :, None] - cdf[:, None, :]) <= tol[:, None, :]).any(2)
    t0, t1 = tol[rows, below], tol[rows, above]
    near_thr = np.abs(d - 1e-5) <= t0 + t1
    flagged = near_knot | near_thr
    bar = np.abs(b1 - b0) * 3 * t1 / den + 4 * np.spacing(np.abs(z).astype(F32)).astype(F64)
    return z, flagged, bar


def composite64(sigma, z, dirs, rgb=None, noise=None, noise_std=0.0, white_back=False):
    """The compositing quadrature (models/rendering.py:143-170) in float64 on fp32 inputs sigma (R, S), z (R, S),
    dirs (R, 3), rgb (R, S, 3) or None, noise (R, S) or None.  Returns (weights, rgb | None, depth | None,
    opacity).  Overflow to inf (huge sigma) gives alpha = 1 exactly, as in fp32."""
    s = np.asarray(sigma, F64)
    zz = np.asarray(z, F64)
    dn = np.linalg.norm(np.asarray(dirs, F64), axis=1, keepdims=True)
    delta = np.concatenate([zz[:, 1:] - zz[:, :-1], np.full((len(zz), 1), 1e10)], 1) * dn
    if noise is not None:
        s = s + np.asarray(noise, F64) * noise_std
    with np.errstate(over="ignore", invalid="ignore"):
        x = delta * np.maximum(s, 0)
        alpha = 1 - np.exp(-np.where(np.isnan(x), 0.0, x))
    f = 1 - alpha + 1e-10
    T = np.concatenate([np.ones((len(s), 1)), np.cumprod(f, 1)[:, :-1]], 1)
    w = alpha * T
    opac = w.sum(1)
    if rgb is None:
        return w, None, None, opac
    c = (w[..., None] * np.asarray(rgb, F64)).sum(1)
    if white_back:
        c = c + (1 - opac)[:, None]
    return w, c, (w * zz).sum(1), opac


def composite_errors(sig, rgb, z, d, noise, noise_std, white_back, w, c, dp, op) -> dict:
    """The device's volume_render outputs w (R, S), c (R, 3) | None, dp (R) | None, op (R) against float64 on its
    inputs: weights in units of weight_units(S) against composite64 (the last sample apart), opacity / rgb / depth in
    units of sum_bar_units against float64 sums of the device's own weights.  Returns {metric: worst value}; compare
    with BARS["weights"], BARS["weights_last"] and BARS["sums"]."""
    S = np.asarray(sig).shape[1]
    w64, _, _, _ = composite64(sig, z, d, None, noise, noise_std)
    dw = np.abs(np.asarray(w, F64) - w64) / weight_units(S)
    wd = np.asarray(w, F64)
    opac = wd.sum(1)
    e = {"weights": float(dw[:, :-1].max()) if S > 1 else 0.0, "weights_last": float(dw[:, -1].max()),
         "opacity": float((np.abs(op - opac) / sum_bar_units(S, np.abs(wd).sum(1))).max())}
    if c is not None:
        col = (wd[..., None] * rgb).sum(1)
        absc = np.abs(wd[..., None] * rgb).sum(1)
        extra = 0.0
        if white_back:
            col, absc = col + (1 - opac)[:, None], absc + np.abs(wd).sum(1)[:, None]
            extra = 2 * U32 * (np.abs(col) + 1)
        e["rgb"] = float((np.abs(c - col) / sum_bar_units(S, absc, extra)).max())
        e["depth"] = float((np.abs(dp - (wd * np.asarray(z, F64)).sum(1))
                            / sum_bar_units(S, np.abs(wd * np.asarray(z, F64)).sum(1))).max())
    return e


def composite_violations(e: dict) -> list:
    """The metrics of `composite_errors` above their BARS."""
    bad = []
    for k, v in e.items():
        bar = BARS["weights_last" if k == "weights_last" else "weights" if k == "weights" else "sums"]
        if not v <= bar:
            bad.append(f"{k}: {v:.3g} > {bar}")
    return bad


def check_resampling(z_dev, w_coarse, z_coarse, u, defect: Optional[str] = None) -> dict:
    """The fine depths z_dev (R, S + K) the kernel returned, against `z_fine` on its own coarse weights and depths
    (bitwise), and the emulated new depths against `sample_pdf64`.  Returns {'differ': elements of z_dev that are not
    bit-equal to the emulation, 'f64_bad': unflagged new depths outside sample_pdf64's bar, 'flagged': flagged new
    depths, 'exhaustive': rays whose merge counts ranks exhaustively, 'nonfinite_mismatch': new depths finite in one
    of fp32 / float64 only}."""
    zf, znew, exh = z_fine(w_coarse, z_coarse, u, defect)
    z_dev = np.asarray(z_dev, F32)
    same = (z_dev == zf) | (np.isnan(z_dev) & np.isnan(zf))
    w = np.asarray(w_coarse, F32)
    us = np.sort(np.asarray(u, F32), axis=1, kind="stable")
    z64, flagged, bar = sample_pdf64(bins_from_depths(z_coarse), w[:, 1:-1], us)
    with np.errstate(invalid="ignore"):
        bad = ~(np.abs(znew.astype(F64) - z64) <= bar) & ~flagged & np.isfinite(z64)
    return {"differ": int((~same).sum()), "f64_bad": int(bad.sum()), "flagged": int(flagged.sum()),
            "exhaustive": int(exh.sum()), "nonfinite_mismatch": int((np.isfinite(znew) != np.isfinite(z64)).sum())}


def weight_units(S: int) -> float:
    """The unit the compositing weights are measured in: (S + 8) 2^-24.  The kernel's weights carry an absolute
    error of a few 2^-24 from alpha (the 2-ulp expf, 1 - e, the fp32 product delta |d| sigma), plus up to one such
    term per preceding factor 1 - alpha + 1e-10 of the transmittance and the scan's S + 5 product roundings."""
    return (S + 8) * U32


def sum_bar_units(S: int, terms_abs_sum, extra=0.0):
    """Bound of an fp32 sum of S products as composite_ray forms it: P = S / 32 fmaf per lane, then the 5-level
    butterfly: gamma_(P + 5) sum |terms| (+ `extra` for an addition after the sum)."""
    P = S // LANES
    return (P + 5 + 1) * U32 * np.asarray(terms_abs_sum, F64) + extra + 1e-38     # 0 / 0: no error


# Worst values measured on one H100 80GB HBM3 (400 W power limit) over the case matrix of
# tests/test_gpu_render_stages.py stand next to the bars.  z_fine and the mode-invariance checks are bitwise.  The
# bars are rounding bounds, not fits to the measurements: weights ~6 units in the worst case, the sums gamma_(P+6).
BARS = {
    "weights": 1.0,          # max |w - w64| in units of weight_units(S); worst 0.037 (S = 32, noise)
    "weights_last": 1.0,     # the last sample of a ray (DESIGN.md 5 (ii)); same units; worst 0.30 (far < near)
    "sums": 1.0,             # |rgb / depth / opacity - float64 sum of the device's weights| / sum_bar_units; worst 0.36
    "loss": 1.0,             # |mse / loss - float64| / ((rays per helper warp + 8) 2^-24 mse); worst 0.10
    "psnr": 1.0,             # |psnr - float64| / (4.34 rel. mse bound + 4 ulp(psnr)); worst 0.14
    "sample_pdf64": 0,       # unflagged fp32 samples outside sample_pdf64's bar (edge rays excepted); worst 0
}
