"""Float64 numpy reference of empty-space skipping (nerf_pl_b200.culling, csrc/occupancy_kernels.cuh).

The conventions it restates (DESIGN.md "Empty-space skipping"):

* the sigma grid is ``sigma[i, j, k] = sigma(x_j, y_i, z_k)`` (``nb.sigma_grid``: the first index is y);
* cell ``(cx, cy, cz)`` spans ``[x_cx, x_cx+1] x [y_cy, y_cy+1] x [z_cz, z_cz+1]`` and is occupied iff one of its 8
  corner points has ``sigma > threshold``; arrays of cells here are indexed ``occ[cx, cy, cz]``;
* the occupied set is dilated by ``dilate`` cells in Chebyshev distance;
* the bit field holds cell ``c = (cz * M + cy) * M + cx`` (``M = N - 1``, x fastest) as bit ``c % 32`` of word ``c // 32``;
* a ray ``[o, d, near, far]`` is live iff the segment ``o + t d``, ``t in [near, far]``, clipped to the grid's box,
  crosses an occupied cell (Amanatides-Woo); outside the box is empty; a ray with a non-finite value or
  ``far <= near`` is live;
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


def ray_live(rays, occ, ranges):
    """(flag (n) bool, margin (n) float64).  ``ranges`` = ((xmin, xmax), (ymin, ymax), (zmin, zmax)); the rays are
    taken in float32, as the device takes them.  ``margin`` is, in cells, how far the ray's walk stayed from every
    decision that a rounding could flip: a cell edge or corner passed, the end of the segment against a cell face,
    the start point against a cell face, the box against the segment.  It only covers the walk up to the cell that
    decided the flag."""
    occ = np.asarray(occ, bool)
    M = occ.shape[0]
    r = np.asarray(rays, np.float32).astype(np.float64).reshape(-1, 8)
    n = len(r)
    lo = np.array([a for a, _ in ranges], np.float64)
    hi = np.array([b for _, b in ranges], np.float64)
    scale = M / (hi - lo)
    flag = np.zeros(n, bool)
    margin = np.full(n, np.inf)
    guard = ~np.isfinite(r).all(1) | ~(r[:, 7] > r[:, 6])
    flag[guard] = True
    with np.errstate(all="ignore"):
        o = (r[:, :3] - lo) * scale
        d = r[:, 3:6] * scale
        zero = d == 0.0
        inv = np.where(zero, 0.0, 1.0 / d)
        ta, tb = (0.0 - o) * inv, (M - o) * inv
        tlo = np.where(zero, -np.inf, np.minimum(ta, tb))
        thi = np.where(zero, np.inf, np.maximum(ta, tb))
        t0 = np.maximum(r[:, 6], tlo.max(1))
        t1 = np.minimum(r[:, 7], thi.min(1))
        outside = (zero & ((o < 0.0) | (o > M))).any(1)
        speed = np.abs(d)
        margin = np.minimum(margin, np.where(zero, np.minimum(np.abs(o), np.abs(o - M)), np.inf).min(1))
        margin = np.minimum(margin, np.abs(t1 - t0) * speed.max(1))
        idx = np.nonzero(~guard & ~outside & (t0 <= t1))[0]
        p0 = o[idx] + t0[idx, None] * d[idx]
        cell = np.clip(np.floor(p0), 0, M - 1).astype(np.int64)
        k = np.round(p0)
        margin[idx] = np.minimum(margin[idx], np.where((k <= 0) | (k >= M), np.inf, np.abs(p0 - k)).min(1))
        for _ in range(3 * M + 3):
            if len(idx) == 0:
                break
            hit = occ[cell[:, 0], cell[:, 1], cell[:, 2]]
            flag[idx[hit]] = True
            idx, cell = idx[~hit], cell[~hit]
            oo, dd, zz = o[idx], d[idx], zero[idx]
            tn = np.where(zz, np.inf, ((cell + (dd > 0.0)) - oo) * inv[idx])
            ax = np.argmin(tn, 1)
            rows = np.arange(len(idx))
            tmin = tn[rows, ax]
            gap = np.where(zz, np.inf, (tn - tmin[:, None]) * speed[idx])
            gap[rows, ax] = np.inf
            cell[rows, ax] += np.where(dd[rows, ax] > 0.0, 1, -1)
            inside = (cell[rows, ax] >= 0) & (cell[rows, ax] < M)
            # leaving the box ends the walk whichever side of t1 the crossing falls on
            end = np.where(inside & np.isfinite(tmin), np.abs(tmin - t1[idx]) * speed[idx][rows, ax], np.inf)
            margin[idx] = np.minimum(margin[idx], np.minimum(gap.min(1), end))
            go = (tmin <= t1[idx]) & inside
            idx, cell = idx[go], cell[go]
    margin[guard] = np.inf
    return flag, margin


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
