"""Float64 numpy reference of empty-space skipping (nerf_pl_b200.culling, csrc/occupancy_kernels.cuh).

The conventions it restates (DESIGN.md "Empty-space skipping"):

* the sigma grid is ``sigma[i, j, k] = sigma(x_j, y_i, z_k)`` (``nb.sigma_grid``: the first index is y);
* cell ``(cx, cy, cz)`` spans ``[x_cx, x_cx+1] x [y_cy, y_cy+1] x [z_cz, z_cz+1]`` and is occupied iff one of its 8
  corner points has ``sigma > threshold``; arrays of cells here are indexed ``occ[cx, cy, cz]``;
* the occupied set is dilated by ``dilate`` cells in Chebyshev distance;
* the bit field holds cell ``c = (cz * M + cy) * M + cx`` (``M = N - 1``, x fastest) as bit ``c % 32`` of word ``c // 32``;
* a ray ``[o, d, near, far]`` is live iff the segment ``o + t d``, ``t in [near, far]``, meets the closed box of an
  occupied cell grown by the float32 rounding bound ``delta`` of ray_live; outside the box is empty; a ray with a
  non-finite value or ``far <= near`` is live;
* a culled ray gets what a ray through vacuum renders: opacity 0, depth 0, rgb 1 with ``white_back`` else 0.
"""
import numpy as np

RESULT_KEYS = ("rgb_coarse", "depth_coarse", "opacity_coarse", "rgb_fine", "depth_fine", "opacity_fine")


def cells_from_sigma(sigma, threshold):
    """occ[cx, cy, cz] of a (N, N, N) sigma grid in ``nb.sigma_grid``'s order."""
    s = np.asarray(sigma).astype(np.float64).transpose(1, 0, 2) > float(threshold)     # s[x, y, z]
    M = s.shape[0] - 1
    occ = np.zeros((M, M, M), bool)
    for dx in (0, 1):
        for dy in (0, 1):
            for dz in (0, 1):
                occ |= s[dx:dx + M, dy:dy + M, dz:dz + M]
    return occ


def dilate(occ, r):
    """Every cell within Chebyshev distance r of an occupied cell."""
    out = np.asarray(occ, bool).copy()
    M = out.shape[0]
    for axis in range(3):
        src = out.copy()
        for s in range(1, min(int(r), M - 1) + 1):
            a = [slice(None)] * 3
            b = [slice(None)] * 3
            a[axis], b[axis] = slice(s, None), slice(None, M - s)
            out[tuple(a)] |= src[tuple(b)]
            out[tuple(b)] |= src[tuple(a)]
    return out


def pack_bits(occ):
    """uint32 words of occ[cx, cy, cz]."""
    flat = np.asarray(occ, bool).transpose(2, 1, 0).reshape(-1)
    pad = (-len(flat)) % 32
    by = np.packbits(np.concatenate([flat, np.zeros(pad, bool)]), bitorder="little")
    return by.view("<u4").astype(np.uint32)


def unpack_bits(words, N):
    M = N - 1
    flat = np.unpackbits(np.asarray(words, "<u4").view(np.uint8), bitorder="little")[:M ** 3].astype(bool)
    return flat.reshape(M, M, M).transpose(2, 1, 0)


def occupancy(sigma, threshold, r):
    return dilate(cells_from_sigma(sigma, threshold), r)


GROWTH = 2.0 ** -22     # delta_a = GROWTH |scale_a| (|o_a| + |d_a| max(|near|, |far|)): 4 float32 unit roundoffs


def _geometry(r, ranges, M):
    """Grid coordinates of float64 rays r (n, 8): o, d, zero (d == 0), inv (1 / d, 0 where zero) and the growth
    delta (n, 3) of each axis, each computed as the device computes it."""
    lo = np.array([a for a, _ in ranges], np.float64)
    hi = np.array([b for _, b in ranges], np.float64)
    scale = M / (hi - lo)
    o = (r[:, :3] - lo) * scale
    d = r[:, 3:6] * scale
    zero = d == 0.0
    inv = np.where(zero, 0.0, 1.0 / np.where(zero, 1.0, d))
    tmax = np.maximum(np.abs(r[:, 6]), np.abs(r[:, 7]))
    delta = np.where(zero, 0.0, GROWTH * np.abs(scale) * (np.abs(r[:, :3]) + np.abs(r[:, 3:6]) * tmax[:, None]))
    return o, d, zero, inv, delta


def _slab(o, d, zero, inv, lo, hi, t0, t1):
    """(meets, margin): whether o + t d, t in [t0, t1], meets the box [lo, hi] (all (n, 3); t0, t1 (n,)), the
    device's slab test; an axis with d == 0 tests o against [lo, hi] exactly.  ``margin`` is, in cells, how far a face
    of the box would have to move to flip the answer: the gap between the latest entry and the earliest exit time over
    the sum of 1 / |d| of the two axes that set them (t0 and t1 count 0)."""
    ta, tb = (lo - o) * inv, (hi - o) * inv
    tl = np.where(zero, -np.inf, np.minimum(ta, tb))
    th = np.where(zero, np.inf, np.maximum(ta, tb))
    w = np.where(zero, 0.0, np.abs(inv))
    tl = np.concatenate([t0[:, None], tl], 1)
    th = np.concatenate([t1[:, None], th], 1)
    w = np.concatenate([np.zeros((len(o), 1)), w], 1)
    i, j = np.argmax(tl, 1), np.argmin(th, 1)
    rows = np.arange(len(o))
    a, b = tl[rows, i], th[rows, j]
    inside = ~(zero & ((o < lo) | (o > hi))).any(1)
    ww = w[rows, i] + w[rows, j]
    margin = np.where(ww > 0.0, np.abs(b - a) / np.where(ww > 0.0, ww, 1.0), np.inf)
    return inside & (a <= b), np.where(inside, margin, np.inf)


_OFFSETS = np.array([(x, y, z) for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1)], np.int64)


def ray_live(rays, occ, ranges):
    """(flag (n) bool, margin (n) float64).  ``ranges`` = ((xmin, xmax), (ymin, ymax), (zmin, zmax)); the rays are
    taken in float32, as the device takes them.

    A ray is live iff the segment meets the closed box of an occupied cell grown by delta_a grid units on each axis
    (GROWTH; 0 on an axis with d_a = 0), or some delta_a >= 1/2 and the segment meets the box grown alike.  This is
    the device's walk step by step: the segment clipped to the grown box, Amanatides-Woo over the lattice extended by a
    ring of empty cells -1 and M, and at each visited cell the neighbours across the faces the segment comes within
    delta of (within delta / |d| of crossing them), each occupied one confirmed by a slab test against its grown box.
    The device also skips the neighbours that are the previous and next visited cells, which changes no flag.

    ``margin`` is, in cells, how far the ray stayed from every grown-box decision a rounding could flip: the clip
    against the grown box, and the slab test of every occupied cell next to (or at) a visited cell, admitted or
    not.  It covers the walk up to the cell that decided the flag."""
    occ = np.asarray(occ, bool)
    M = occ.shape[0]
    r = np.asarray(rays, np.float32).astype(np.float64).reshape(-1, 8)
    n = len(r)
    flag = np.zeros(n, bool)
    margin = np.full(n, np.inf)
    guard = ~np.isfinite(r).all(1) | ~(r[:, 7] > r[:, 6])
    flag[guard] = True
    with np.errstate(all="ignore"):
        o, d, zero, inv, delta = _geometry(r, ranges, M)
        ok, m = _slab(o, d, zero, inv, -delta, M + delta, r[:, 6], r[:, 7])
        margin = np.minimum(margin, m)
        ta, tb = (-delta - o) * inv, (M + delta - o) * inv
        t0 = np.maximum(r[:, 6], np.where(zero, -np.inf, np.minimum(ta, tb)).max(1))
        t1 = np.minimum(r[:, 7], np.where(zero, np.inf, np.maximum(ta, tb)).min(1))
        ok &= ~guard
        coarse = ok & (delta >= 0.5).any(1)
        flag[coarse] = True
        margin = np.minimum(margin, np.where(zero, np.inf, np.abs(delta - 0.5)).min(1))
        idx = np.nonzero(ok & ~coarse)[0]
        cell = np.clip(np.floor(o[idx] + t0[idx, None] * d[idx]), -1, M).astype(np.int64)
        te = t0[idx]
        for _ in range(3 * (M + 2) + 3):
            if len(idx) == 0:
                break
            oo, dd, zz, ii, de = o[idx], d[idx], zero[idx], inv[idx], delta[idx]
            tn = np.where(zz, np.inf, ((cell + (dd > 0.0)) - oo) * ii)
            ax = np.argmin(tn, 1)
            rows = np.arange(len(idx))
            tnext = tn[rows, ax]
            tx = np.minimum(tnext, t1[idx])
            # the faces behind and ahead that the segment comes within delta of inside the cell, by crossing time
            tlow = np.where(zz, -np.inf, ((cell + (dd < 0.0)) - oo) * ii)
            eps = de * np.abs(ii)
            back = np.where(zz, oo - cell <= 0.0, te[:, None] - tlow <= eps)
            ahead = np.where(zz, (cell + 1) - oo <= 0.0, tn - tx[:, None] <= eps)
            c0 = cell - np.where(dd < 0.0, ahead, back)
            c1 = cell + np.where(dd < 0.0, back, ahead)
            hit = np.zeros(len(idx), bool)
            for off in _OFFSETS:
                c = cell + off
                sel = np.nonzero(((c >= 0) & (c < M)).all(1))[0]
                sel = sel[occ[c[sel, 0], c[sel, 1], c[sel, 2]]]
                if len(sel) == 0:
                    continue
                cs = c[sel].astype(np.float64)
                meets, m = _slab(oo[sel], dd[sel], zz[sel], ii[sel], cs - de[sel], (cs + 1.0) + de[sel],
                                 t0[idx[sel]], t1[idx[sel]])
                margin[idx[sel]] = np.minimum(margin[idx[sel]], m)
                admitted = ((c[sel] >= c0[sel]) & (c[sel] <= c1[sel])).all(1)
                hit[sel] |= meets & admitted
            flag[idx[hit]] = True
            step = cell[rows, ax] + np.where(dd[rows, ax] > 0.0, 1, -1)
            go = ~hit & (tnext <= t1[idx]) & (step >= -1) & (step <= M)
            cell[rows, ax] = step
            idx, cell, te = idx[go], cell[go], tnext[go]
    margin[guard] = np.inf
    return flag, margin


def brute_live(rays, occ, ranges):
    """(n,) bool: the grown-box rule of ray_live by a slab test of every segment, t in [near, far], against every
    occupied cell's grown box, in float64.  For small grids."""
    occ = np.asarray(occ, bool)
    M = occ.shape[0]
    r = np.asarray(rays, np.float32).astype(np.float64).reshape(-1, 8)
    n = len(r)
    guard = ~np.isfinite(r).all(1) | ~(r[:, 7] > r[:, 6])
    cells = np.argwhere(occ).astype(np.float64)                 # (C, 3) [cx, cy, cz]
    live = guard.copy()
    with np.errstate(all="ignore"):
        o, d, zero, inv, delta = _geometry(r, ranges, M)
        box, _ = _slab(o, d, zero, inv, -delta, M + delta, r[:, 6], r[:, 7])
        live |= ~guard & box & (delta >= 0.5).any(1)
        rest = np.nonzero(~live)[0]
        t0, t1 = r[rest, 6], r[rest, 7]
        for c in cells:                                         # every ray against one cell's grown box at a time
            c = np.broadcast_to(c, (len(rest), 3))
            meets, _ = _slab(o[rest], d[rest], zero[rest], inv[rest], c - delta[rest], (c + 1.0) + delta[rest], t0, t1)
            live[rest] |= meets
    return live


def vacuum_results(n, keys, white_back):
    """What ``render_rays`` gives for n rays through vacuum: the weights are all 0, so opacity and depth are 0 and
    rgb is the background term ``1 - opacity`` (white_back) or 0."""
    out = {}
    for k in keys:
        if k.startswith("rgb"):
            out[k] = np.full((n, 3), 1.0 if white_back else 0.0, np.float32)
        else:
            out[k] = np.zeros(n, np.float32)
    return out


def scatter(compact, live_idx, n, white_back):
    """Full-size results of compacted ones (dict of arrays with len(live_idx) rows)."""
    out = vacuum_results(n, list(compact), white_back)
    for k, v in compact.items():
        out[k][live_idx] = v
    return out


def result_keys(N_importance, test_time):
    keys = ["opacity_coarse"] if test_time else ["rgb_coarse", "depth_coarse", "opacity_coarse"]
    return keys + (["rgb_fine", "depth_fine", "opacity_fine"] if N_importance > 0 else [])


def guard_cases():
    """(occ, ranges, rays, expected flags): one occupied cell, x [0, 1] x y [-1, 0] x z [1, 2], in a 4^3-cell grid over
    [-2, 2]^3, and one ray per guard of the walk."""
    occ = np.zeros((4, 4, 4), bool)
    occ[2, 1, 3] = True
    c = np.array([0.5, -0.5, 1.5])
    cases = [
        ([*(c - [5, 0, 0]), 1, 0, 0, 0, 10], True),      # two zero direction components, through the cell
        ([*(c - [5, 0, 1]), 1, 0, 0, 0, 10], False),     # the same, one cell lower
        ([0.5, -0.5, -1.5, 0, 0, 1, 0, 10], True),       # starts inside the box and walks up into the cell
        ([0.5, -0.5, -1.5, 0, 0, -1, 0, 10], False),     # starts inside and walks away
        ([*c, 0, 0, 0, 0, 10], True),                    # zero direction inside the occupied cell
        ([0.5, 0.5, 1.5, 0, 0, 0, 0, 10], False),        # zero direction inside an empty cell
        ([*(c - [5, 0, 0]), 1, 0, 0, 6, 2], True),       # far < near: live
        ([*(c - [5, 0, 1]), 1, 0, 0, 3, 3], True),       # far == near: live
        ([np.nan, 0, 0, 1, 0, 0, 0, 10], True),          # non-finite values: live
        ([0, 0, 0, np.inf, 0, 0, 0, 10], True),
        ([9, 9, 9, 1, 0, 0, 0, np.inf], True),
        ([9, 9, 9, 1, 0, 0, 0, 10], False),              # never enters the box
        ([9, -0.5, 1.5, 0, 1, 0, 0, 10], False),         # zero x component outside the box's x slab
        ([*(c - [5, 0, 0]), 1, 0, 0, 0, 4.4], False),    # ends in the cell before the occupied one
        ([*(c - [5, 0, 0]), 1, 0, 0, 5.6, 10], False),   # starts past it
        ([*(c + [5, 0, 0]), -1, 0, 0, 0, 10], True),     # the same line walked backwards
        ([*(c - [3, 3, 3]), 1, 1, 1, 0, 10], True),      # a diagonal through cell corners into the cell
    ]
    rays = np.array([r for r, _ in cases], np.float32)
    return occ, ((-2.0, 2.0),) * 3, rays, np.array([f for _, f in cases])
