"""Float64 numpy restatement of cascaded occupancy grids (nerf_pl_b200.OccupancyGrid(levels=), DensityGrid(levels=),
csrc/occupancy_kernels.cuh, csrc/density_kernels.cuh, include/nerf_pl_b200.h; DESIGN.md §10h).

A grid of L levels over ranges (xmin, xmax, ymin, ymax, zmin, zmax) with N points and M = N - 1 cells per axis:

* level 0's box is the ranges as given; for k >= 1, with c = 0.5 (lo + hi) and h = 0.5 (hi - lo) in float64, level
  k's range on each axis is (c - 2^k h, c + 2^k h);
* level k's ceil(M^3 / 32) words follow level k - 1's; inside a level the one-level conventions hold
  (tests/occupancy_ref.py);
* a point belongs to the smallest level whose closed box holds it, tested in that level's grid coordinates
  g = (x - lo) * (M / (hi - lo)) as 0 <= g <= M on every axis; inside it the one-level closed-cell rule applies
  (tests/sample_skip_ref.py); outside the last level, or NaN, it is empty;
* a cell of level k >= 1 whose indices all lie in [ceil(M / 4), floor(3 M / 4)) lies inside level k - 1's box: it is
  *inner*, and always empty;
* building: each level is marked (the 8-corner rule, or the density threshold) with its inner cells empty, dilated
  within the level and packed with its inner cells cleared;
* the cell walk is the one-level walk on each level's box in turn; a ray is live if any level's walk is;
* a density grid update evaluates each level's non-inner cells, in cell order, with the jitter of cell c of level
  k drawn as philox(key, ray = c, element = 3 k + a, stream = 2) on level k's box; the key advances once.
"""
import numpy as np

from . import density_ref as dr
from . import occupancy_ref as oc
from . import philox
from . import sample_skip_ref as ss


def level_ranges(ranges, k):
    """(xmin, xmax, ymin, ymax, zmin, zmax) of level k."""
    r = [float(v) for v in ranges]
    if k == 0:
        return tuple(r)
    out = []
    for a in range(3):
        lo, hi = r[2 * a], r[2 * a + 1]
        c, h = 0.5 * (lo + hi), 0.5 * (hi - lo)
        e = h * 2.0 ** k
        out += [c - e, c + e]
    return tuple(out)


def pairs(r6):
    return ((r6[0], r6[1]), (r6[2], r6[3]), (r6[4], r6[5]))


def inner_range(N, k):
    """[a, b) of the inner cell indices of one axis of level k ((0, 0) at level 0)."""
    M = N - 1
    if k == 0:
        return 0, 0
    a = -(-M // 4)
    return a, max(3 * M // 4, a)


def inner_mask(N, k):
    """occ-shaped [cx, cy, cz] bool of the inner cells of level k."""
    M = N - 1
    a, b = inner_range(N, k)
    m = np.zeros((M, M, M), bool)
    m[a:b, a:b, a:b] = True
    return m


def words_per_level(N):
    return ((N - 1) ** 3 + 31) // 32


def split(words, N, L):
    return np.asarray(words).view(np.uint32).reshape(L, words_per_level(N))


def grid_coords(x, N, r6):
    lo = np.array(r6[0::2], np.float64)
    hi = np.array(r6[1::2], np.float64)
    return (np.asarray(x, np.float64) - lo) * (float(N - 1) / (hi - lo))


def level_of(x, N, L, ranges):
    """(P,) int: the level of each point of x (P, 3) (float32 or float64 values, taken as float64); -1 outside."""
    x = np.asarray(x).reshape(-1, 3)
    out = np.full(len(x), -1, np.int64)
    with np.errstate(invalid="ignore"):
        for k in reversed(range(L)):
            g = grid_coords(x, N, level_ranges(ranges, k))
            out[((g >= 0.0) & (g <= N - 1)).all(1)] = k
    return out


def point_evaluated(x, words, N, L, ranges):
    """bool (...) for points x (..., 3): in the closed box of an occupied cell of the point's level.  The values are
    taken as float64 (a float32 point is exact in it)."""
    x = np.asarray(x)
    flat = x.reshape(-1, 3)
    lev = level_of(flat, N, L, ranges)
    w = split(words, N, L)
    out = np.zeros(len(flat), bool)
    for k in range(L):
        sel = lev == k
        if sel.any():
            out[sel] = _evaluated_in_level(flat[sel], w[k], N, level_ranges(ranges, k))
    return out.reshape(x.shape[:-1])


def _evaluated_in_level(x, words, N, r6):
    """ss.point_evaluated_vec without its float32 cast."""
    M = N - 1
    g = grid_coords(x, N, r6)
    inside = ((g >= 0.0) & (g <= M)).all(1)
    g = np.where(inside[:, None], g, 0.0)
    f = np.floor(g)
    fl = f.astype(np.int64)
    c1 = np.minimum(fl, M - 1)
    c0 = np.where((f == g) & (fl > 0), fl - 1, c1)
    cells = np.stack([(cz[:, 2] * M + cy[:, 1]) * M + cx[:, 0]
                      for cz in (c0, c1) for cy in (c0, c1) for cx in (c0, c1)], 1)
    on = ((words[cells >> 5] >> (cells & 31).astype(np.uint32)) & 1) == 1
    return on.any(1) & inside


def evaluated(rays, z, words, N, L, ranges):
    """(R, S) bool: the evaluated samples of one pass (tests/sample_skip_ref.evaluated through a cascade)."""
    ev = point_evaluated(ss.sample_points(rays, z), words, N, L, ranges)
    ev[ss.plain_pass(rays, z)] = True
    return ev


def occupancy_levels(cells, dilate):
    """(L, M, M, M) bool [level, cx, cy, cz] from each level's marked cells: inner cells emptied, dilated within the
    level, inner cells cleared."""
    L, N = len(cells), cells[0].shape[0] + 1
    out = []
    for k in range(L):
        c = np.asarray(cells[k], bool) & ~inner_mask(N, k)
        out.append(oc.dilate(c, dilate) & ~inner_mask(N, k))
    return np.stack(out)


def pack(occ_levels):
    return np.concatenate([oc.pack_bits(o) for o in occ_levels])


def unpack(words, N, L):
    return np.stack([oc.unpack_bits(w, N) for w in split(words, N, L)])


def pack_sigma(sigma, threshold, dilate):
    """The bits of nerfb200_occupancy_pack_levels for sigma (L, N, N, N)."""
    return pack(occupancy_levels([oc.cells_from_sigma(s, threshold) for s in sigma], dilate))


def ray_live(rays, words, N, L, ranges):
    """(n,) bool: the per-level walk of tests/occupancy_ref.ray_live, OR-ed over the levels."""
    occ = unpack(words, N, L)
    live = np.zeros(len(np.asarray(rays).reshape(-1, 8)), bool)
    for k in range(L):
        live |= oc.ray_live(rays, occ[k], pairs(level_ranges(ranges, k)))[0]
    return live


# ---- the density grid ---------------------------------------------------------------------------------
def noninner_cells(N, k):
    """(count,) int64: the non-inner cells of level k in cell order (every cell at level 0)."""
    M = N - 1
    inner = inner_mask(N, k).transpose(2, 1, 0).reshape(-1)      # cell order
    return np.nonzero(~inner)[0].astype(np.int64)


def points(seed, N, L, ranges, k, start=0, count=None):
    """(count, 3) float32: the points of the non-inner cells of rank [start, start + count) of level k."""
    M = N - 1
    cells = noninner_cells(N, k)
    count = len(cells) - start if count is None else count
    c = cells[start:start + count]
    el = np.arange(3 * k, 3 * k + 3, dtype=np.uint64)
    rays = np.broadcast_to(c.astype(np.uint64)[:, None], (len(c), 3))
    words = philox.philox4x32_10(rays, np.broadcast_to(el >> np.uint64(2), rays.shape), np.full(rays.shape, 2, np.uint64),
                                 np.zeros(rays.shape, np.uint64), int(seed) & dr.MASK64)
    sel = np.broadcast_to((el & np.uint64(3)).astype(np.int64), rays.shape)
    u = ((np.choose(sel, words) >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)).astype(np.float64)
    r6 = level_ranges(ranges, k)
    lo = np.array(r6[0::2])
    hi = np.array(r6[1::2])
    cell = np.stack([c % M, (c // M) % M, c // (M * M)], 1).astype(np.float64)
    return (lo + (cell + u) * ((hi - lo) / float(M))).astype(np.float32)


def initial(N, L, seed):
    M = N - 1
    occ = np.stack([~inner_mask(N, k) for k in range(L)])
    return {"density": np.zeros(L * M ** 3, np.float32), "bits": pack(occ), "key": int(seed)}


def update(state, sigma_fn, N, L, ranges, threshold, decay, dilate):
    """The next state of a cascade density grid; ``sigma_fn(points (P, 3) float32) -> (P,) float32``."""
    M = N - 1
    C = M ** 3
    dens = np.asarray(state["density"], np.float32).copy()
    occ = []
    for k in range(L):
        cells = noninner_cells(N, k)
        d = dens[k * C:(k + 1) * C]
        d[cells] = dr.decay_max(d[cells], sigma_fn(points(state["key"], N, L, ranges, k)), decay)
        marked = np.zeros(C, bool)
        marked[cells] = d[cells].astype(np.float64) > float(threshold)
        occ.append(marked.reshape(M, M, M).transpose(2, 1, 0))
    return {"density": dens, "bits": pack(occupancy_levels(occ, dilate)), "key": state["key"] + 1}
