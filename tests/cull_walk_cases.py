"""Designed rays at the decisions of the cell walk (csrc/occupancy_kernels.cuh cull_level_live, restated by
tests/occupancy_ref.ray_live): one occupied cell at a time in a cascade, and rays on its lattice planes, lines,
corners and faces, through its corners and edges in every direction, starting or ending on them, rays whose float32
samples round onto its face while the exact segment stops short, and rays that miss it by 1e-3 of a cell.  Every
value is a float32; with a cell size that is a power of two every lattice value is exact."""
import numpy as np

from . import cascade_ref as cr

F32 = np.float32
DIRS = np.array([s for s in np.ndindex(3, 3, 3) if s != (1, 1, 1)], np.float64) - 1.0     # the 26 directions


def level_box(ranges, k):
    r = cr.level_ranges(ranges, k)
    return np.array(r[0::2], np.float64), np.array(r[1::2], np.float64)


def lattice(ranges, N, k, idx):
    """float32 world points of level k's lattice coordinates idx (..., 3) (fractional allowed)."""
    lo, hi = level_box(ranges, k)
    return (lo + (hi - lo) * (np.asarray(idx, np.float64) / (N - 1))).astype(F32)


def target_cells(N, L):
    """[(level, cell)]: per level, its box's corner cell and a cell that touches the box of the level below (level 0:
    a middle cell)."""
    M = N - 1
    out = []
    for k in range(L):
        out.append((k, (0, 0, 0)))
        if k == 0:
            out.append((k, (M // 2, max(M // 2 - 1, 0), M - 1)))
        else:
            a = cr.inner_range(N, k)[0]
            out.append((k, (max(a - 1, 0), a, a)))
    return out


def one_cell_words(N, L, k, cell):
    M = N - 1
    occ = np.zeros((L, M, M, M), bool)
    occ[k][tuple(cell)] = True
    return cr.pack(occ)


def _ulps(p):
    """p (P, 3) float32 and each coordinate one ulp either way: (27 P, 3)."""
    out = []
    for s in np.ndindex(3, 3, 3):
        q = p.copy()
        for a in range(3):
            if s[a] != 1:
                q[:, a] = np.nextafter(q[:, a], F32(np.inf) if s[a] == 2 else F32(-np.inf))
        out.append(q)
    return np.concatenate(out)


def _rays(o, d, near, far):
    n = len(o)
    return np.concatenate([o, np.broadcast_to(d, (n, 3)), np.broadcast_to(np.asarray(near, F32), (n,))[:, None],
                           np.broadcast_to(np.asarray(far, F32), (n,))[:, None]], 1).astype(F32)


def probes(ranges, N, k, cell):
    """(a) zero-direction rays (near 0, far 1) at the corners, edge midpoints and face centres of the cell and its
    neighbours ({c - 1/2, c, c + 1/2, c + 1, c + 3/2} per axis), each coordinate also one ulp either way."""
    h = np.array([-0.5, 0.0, 0.5, 1.0, 1.5])
    idx = np.array(cell, np.float64) + np.stack(np.meshgrid(h, h, h, indexing="ij"), -1).reshape(-1, 3)
    p = _ulps(lattice(ranges, N, k, idx))
    return _rays(p, np.zeros(3, F32), 0.0, 1.0)


def axis_rays(ranges, N, k, cell, L):
    """(b) rays along each axis, both ways, across the last level's box, in the cell's lattice planes and lines
    (the other two coordinates at c, c + 1/2 or c + 1), each of those one ulp either way."""
    lo, hi = level_box(ranges, L - 1)
    ext = float(np.abs(hi - lo).max())
    mid = 0.5 * (lo + hi)
    out = []
    for a in range(3):
        for sgn in (1.0, -1.0):
            h = np.array([0.0, 0.5, 1.0])
            idx = np.array(cell, np.float64) + np.stack(np.meshgrid(h, h, h, indexing="ij"), -1).reshape(-1, 3)
            idx = idx[idx[:, a] == cell[a]]                     # the 9 transverse positions
            p = _ulps(lattice(ranges, N, k, idx))
            p = p[np.unique(p[:, [b for b in range(3) if b != a]], axis=0, return_index=True)[1]]
            p[:, a] = F32(mid[a] - sgn * ext)
            d = np.zeros(3, F32)
            d[a] = sgn
            out.append(_rays(p, d, 0.0, 2.0 * ext))
    return np.concatenate(out)


def point_rays(ranges, N, k, cell):
    """(c), (d) rays through every corner, edge midpoint and face centre of the cell (and its centre) in each of the
    26 directions of a cell's step, as whole segments (near -2, far 2), segments that start there (0, 2) and
    segments that end there (-2, 0)."""
    lo, hi = level_box(ranges, k)
    step = ((hi - lo) / (N - 1)).astype(F32)
    h = np.array([0.0, 0.5, 1.0])
    idx = np.array(cell, np.float64) + np.stack(np.meshgrid(h, h, h, indexing="ij"), -1).reshape(-1, 3)
    p = lattice(ranges, N, k, idx)
    out = []
    for s in DIRS:
        d = (s * step).astype(F32)
        for near, far in ((-2.0, 2.0), (0.0, 2.0), (-2.0, 0.0)):
            out.append(_rays(p, d, near, far))
    return np.concatenate(out)


def near_misses(ranges, N, k, cell):
    """Rays that pass 1e-3 of a cell outside each face of the cell, along each of the face's two axes and its
    diagonal, and diagonals that pass 1e-3 of a cell outside each corner."""
    lo, hi = level_box(ranges, k)
    step = (hi - lo) / (N - 1)
    c = np.array(cell, np.float64)
    out = []
    for a in range(3):
        for side in (-1e-3, 1.0 + 1e-3):
            for along in range(3):
                if along == a:
                    continue
                o = c + 0.5
                o[a] = c[a] + side
                o[along] -= 3.0
                d = np.zeros(3)
                d[along] = 1.0
                out.append(np.concatenate([lo + o * step, d * step, [0.0, 6.0]]))
            o = c + 0.5
            o[a] = c[a] + side
            b, e = [x for x in range(3) if x != a]
            o[b] -= 3.0
            o[e] -= 3.0
            d = np.zeros(3)
            d[b] = d[e] = 1.0
            out.append(np.concatenate([lo + o * step, d * step, [0.0, 6.0]]))
    for s in np.ndindex(2, 2, 2):
        corner = c + np.array(s, np.float64)
        out_dir = np.where(np.array(s) == 1, 1.0, -1.0)
        o = corner + out_dir * 1e-3 - 3.0 * np.array([1.0, -1.0, 0.0]) * out_dir
        d = np.array([1.0, -1.0, 0.0]) * out_dir
        out.append(np.concatenate([lo + o * step, d * step, [0.0, 6.0]]))
    return np.array(out).astype(F32)


def rounding_rays(ranges, N, k, cell, seed, want=24, tries=20000):
    """(e) a seeded search for rays toward a face of the cell whose exact segment stops short of the face while
    its last float32 sample fl(o + fl(d far)) lands on it: along x (the other coordinates mid-cell) and along x
    with small transverse components, from either side."""
    rng = np.random.default_rng(seed)
    lo, hi = level_box(ranges, k)
    step = (hi - lo) / (N - 1)
    c = np.array(cell, np.float64)
    found = []
    for sgn in (1.0, -1.0):
        face_idx = c[0] if (sgn > 0) == (step[0] > 0) else c[0] + 1.0
        face = F32(lo[0] + face_idx * step[0])
        n = tries
        o = np.zeros((n, 3))
        o[:, 1:] = lo[1:] + (c[1:] + rng.uniform(0.3, 0.7, (n, 2))) * step[1:]
        o[:, 0] = float(face) - sgn * rng.uniform(0.2, 2.0, n) * abs(step[0])
        d = np.zeros((n, 3))
        d[:, 0] = sgn * rng.uniform(0.3, 3.0, n)
        tilt = rng.random(n) < 0.5
        d[tilt, 1:] = rng.uniform(-1e-3, 1e-3, (int(tilt.sum()), 2)) * abs(step[1:])
        o, d = o.astype(F32), d.astype(F32)
        far = ((face.astype(np.float64) - o[:, 0].astype(np.float64)) / d[:, 0].astype(np.float64)).astype(F32)
        # the largest float32 far whose exact end stops short of the face
        for _ in range(4):
            end = o[:, 0].astype(np.float64) + d[:, 0].astype(np.float64) * far.astype(np.float64)
            over = (end - float(face)) * sgn >= 0.0
            far = np.where(over, np.nextafter(far, F32(-np.inf)), far)
        end = o[:, 0].astype(np.float64) + d[:, 0].astype(np.float64) * far.astype(np.float64)
        last = (o[:, 0] + (d[:, 0] * far).astype(F32)).astype(F32)
        hit = ((end - float(face)) * sgn < 0.0) & (last == face) & (far > 0)
        for i in np.nonzero(hit)[0][:want]:
            found.append(np.concatenate([o[i], d[i], [0.0, far[i]]]))
    return np.array(found, F32).reshape(-1, 8)


def touches_any_level(x, words, N, L, ranges):
    """(P,) bool: x lies in the closed box of an occupied cell of some level.  This is what the walk finds for a
    ray with d = 0; the lookup takes the point's own level only, so a point on a finer level's box beside an
    occupied coarser cell is live without being evaluated."""
    w = cr.split(words, N, L)
    x = np.asarray(x).reshape(-1, 3)
    return np.any([cr._evaluated_in_level(x, w[k], N, cr.level_ranges(ranges, k)) for k in range(L)], 0)


FAMILIES = ("probes", "axis", "points", "rounding", "misses")


def family(name, ranges, N, L, k, cell, seed=0):
    if name == "probes":
        return probes(ranges, N, k, cell)
    if name == "axis":
        return axis_rays(ranges, N, k, cell, L)
    if name == "points":
        return point_rays(ranges, N, k, cell)
    if name == "rounding":
        return rounding_rays(ranges, N, k, cell, seed)
    return near_misses(ranges, N, k, cell)
