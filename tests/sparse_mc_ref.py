"""A numpy restatement of the sparse marching cubes (csrc/sparse_mc_kernels.cuh, DESIGN.md §10i).

``candidate_bricks`` is the brick pre-filter of the plan (brick_candidate): per axis the brick's float32 positions
[mn, mx] (NaN left out), per level the cells [floor(v(mn)) - 1, floor(v(mx))] clipped to the level, any occupied bit
there makes a candidate, and so does a range of more than ``PROBE_WORDS`` bit-field words.  ``sparse_march`` is the
march on brick storage: active bricks from the evaluated points, their values per brick and the brick map, march
bricks, the vertex keys 3 q + axis and triangle keys 5 c + t per march brick, sorted, then positions and vertex ids.
"""
import numpy as np

from oracle import mesh_oracle as mo

from . import cascade_ref as cr

BRICK = 8
PROBE_WORDS = 512


def bricks_per_axis(N):
    return -(-int(N) // BRICK)


def _axis_bounds(N, r):
    """(mn, mx, any) per brick of one axis: the least and largest non-NaN float32 position of the brick's points."""
    x = mo.grid_axis(r[0], r[1], N).astype(np.float32).astype(np.float64)
    nb = bricks_per_axis(N)
    pad = np.full(nb * BRICK, np.nan)
    pad[:N] = x
    pad = pad.reshape(nb, BRICK)
    with np.errstate(invalid="ignore"):
        return np.nanmin(np.where(np.isnan(pad), np.inf, pad), 1), np.nanmax(np.where(np.isnan(pad), -np.inf, pad), 1), \
            ~np.isnan(pad).all(1)


def candidate_bricks(N, x_range, y_range, z_range, words, occ_N, occ_ranges, levels=1):
    """bool (nb, nb, nb) indexed [I, J, K] (bricks along i = y, j = x, k = z): the plan's candidates."""
    nb = bricks_per_axis(N)
    M = int(occ_N) - 1
    w = cr.split(words, occ_N, levels)
    mn, mx, ok = zip(*(_axis_bounds(N, r) for r in (x_range, y_range, z_range)))
    out = np.zeros((nb, nb, nb), bool)
    for I in range(nb):
        for J in range(nb):
            for K in range(nb):
                b = (J, I, K)                                  # the brick index of each position axis x, y, z
                if not all(ok[a][b[a]] for a in range(3)):
                    continue
                out[I, J, K] = _candidate(tuple(mn[a][b[a]] for a in range(3)), tuple(mx[a][b[a]] for a in range(3)),
                                          w, M, occ_ranges, levels)
    return out


def _candidate(mn, mx, w, M, occ_ranges, levels):
    for k in range(levels):
        r6 = cr.level_ranges(occ_ranges, k)
        c0, c1 = [], []
        for a in range(3):
            lo, hi = r6[2 * a], r6[2 * a + 1]
            scale = float(M) / (hi - lo)
            v0, v1 = sorted(((mn[a] - lo) * scale, (mx[a] - lo) * scale))
            if not (v1 >= 0.0 and v0 <= M):
                break
            f0, f1 = int(np.floor(max(v0, 0.0))), int(np.floor(min(v1, float(M))))
            c0.append(max(f0 - 1, 0))
            c1.append(min(f1, M - 1))
        else:
            rows = (c1[1] - c0[1] + 1) * (c1[2] - c0[2] + 1)
            if rows * ((c1[0] - c0[0]) // 32 + 2) > PROBE_WORDS:
                return True
            cz, cy, cx = np.meshgrid(np.arange(c0[2], c1[2] + 1), np.arange(c0[1], c1[1] + 1),
                                     np.arange(c0[0], c1[0] + 1), indexing="ij")
            cells = ((cz * M + cy) * M + cx).reshape(-1)
            if (((w[k][cells >> 5] >> (cells & 31).astype(np.uint32)) & 1) == 1).any():
                return True
    return False


def evaluated_points(N, x_range, y_range, z_range, words, occ_N, occ_ranges, levels=1):
    """bool (N, N, N): the evaluated lattice points (tests/mesh_grid_ref.py's rule, by cascade level)."""
    x = mo.grid_positions(N, x_range, y_range, z_range)
    return cr.point_evaluated(x, words, occ_N, levels, occ_ranges).reshape(N, N, N)


def brick_of_points(mask):
    """bool (nb, nb, nb): the bricks holding a True point of an (N, N, N) mask."""
    N = mask.shape[0]
    nb = bricks_per_axis(N)
    pad = np.zeros((nb * BRICK,) * 3, bool)
    pad[:N, :N, :N] = mask
    return pad.reshape(nb, BRICK, nb, BRICK, nb, BRICK).any((1, 3, 5))


def march_bricks(active):
    """An active brick or one with an active neighbour at +1 along any subset of the axes."""
    m = active.copy()
    for d in range(1, 8):
        d0, d1, d2 = d & 1, (d >> 1) & 1, (d >> 2) & 1
        m[:m.shape[0] - d0, :m.shape[1] - d1, :m.shape[2] - d2] |= active[d0:, d1:, d2:]
    return m


def sparse_march(sigma, evaluated, threshold):
    """(vertices (V, 3) float64, triangles (T, 3) int32) of the (N, N, N) grid ``sigma`` at its ``evaluated`` points
    (every other point +0.0), computed the sparse way: brick storage, keys, sort."""
    N = sigma.shape[0]
    nb = bricks_per_axis(N)
    active = brick_of_points(evaluated)
    slots = np.full(nb ** 3, -1, np.int64)
    ids = np.nonzero(active.reshape(-1))[0]
    slots[ids] = np.arange(len(ids))
    store = np.zeros((len(ids), BRICK, BRICK, BRICK), np.float32)
    for s, b in enumerate(ids):
        I, J, K = b // (nb * nb), (b // nb) % nb, b % nb
        blk = np.where(evaluated, sigma, np.float32(0))[I * 8:I * 8 + 8, J * 8:J * 8 + 8, K * 8:K * 8 + 8]
        store[s, :blk.shape[0], :blk.shape[1], :blk.shape[2]] = blk

    def value(i, j, k):
        out = np.zeros(np.broadcast(i, j, k).shape, np.float32)
        ok = (i < N) & (j < N) & (k < N)
        i, j, k = (np.broadcast_to(a, out.shape)[ok] for a in (i, j, k))
        s = slots[((i >> 3) * nb + (j >> 3)) * nb + (k >> 3)]
        v = np.zeros(len(s), np.float32)
        v[s >= 0] = store[s[s >= 0], (i & 7)[s >= 0], (j & 7)[s >= 0], (k & 7)[s >= 0]]
        out[ok] = v
        return out

    thr = float(threshold)
    count, tab = mo.load_table()
    march = np.nonzero(march_bricks(active).reshape(-1))[0]
    a, b, c = np.meshgrid(np.arange(8), np.arange(8), np.arange(8), indexing="ij")
    vkeys, tkeys = [], []
    for br in march:
        I, J, K = br // (nb * nb), (br // nb) % nb, br % nb
        i, j, k = (I * 8 + a).reshape(-1), (J * 8 + b).reshape(-1), (K * 8 + c).reshape(-1)
        inside = value(i, j, k).astype(np.float64) > thr
        pt = (i < N) & (j < N) & (k < N)
        q = (i * N + j) * N + k
        for ax, (di, dj, dk) in enumerate(((1, 0, 0), (0, 1, 0), (0, 0, 1))):
            nxt = np.array([i + di, j + dj, k + dk])
            ok = pt & np.all(nxt < N, 0) & ((value(*nxt).astype(np.float64) > thr) != inside)
            vkeys.append(3 * q[ok] + ax)
        cell = (i < N - 1) & (j < N - 1) & (k < N - 1)
        cube = np.zeros(len(i), np.int64)
        for cc in range(8):
            cube |= (value(i + (cc & 1), j + ((cc >> 1) & 1), k + ((cc >> 2) & 1)).astype(np.float64) > thr) << cc
        lin = (i * (N - 1) + j) * (N - 1) + k
        for t in range(5):
            sel = cell & (count[cube] > t)
            tkeys.append(5 * lin[sel] + t)
    vkeys = np.sort(np.concatenate(vkeys)) if vkeys else np.zeros(0, np.int64)
    tkeys = np.sort(np.concatenate(tkeys)) if tkeys else np.zeros(0, np.int64)
    q, ax = vkeys // 3, vkeys % 3
    pi, pj, pk = q // (N * N), (q // N) % N, q % N
    f0 = value(pi, pj, pk).astype(np.float64)
    f1 = value(pi + (ax == 0), pj + (ax == 1), pk + (ax == 2)).astype(np.float64)
    verts = np.stack([pi, pj, pk], 1).astype(np.float64)
    verts[np.arange(len(q)), ax] += (thr - f0) / (f1 - f0)
    cl, t = tkeys // 5, tkeys % 5
    ci, cj, ck = cl // ((N - 1) ** 2), (cl // (N - 1)) % (N - 1), cl % (N - 1)
    cube = np.zeros(len(cl), np.int64)
    for cc in range(8):
        cube |= (value(ci + (cc & 1), cj + ((cc >> 1) & 1), ck + ((cc >> 2) & 1)).astype(np.float64) > thr) << cc
    geo = np.array([(g[0],) + g[1] for g in (mo.edge_geometry(x) for x in range(12))], np.int64)
    tris = np.zeros((len(cl), 3), np.int64)
    for s in range(3):
        e = geo[tab[cube, 3 * t + s]]
        key = 3 * (((ci + e[:, 1]) * N + cj + e[:, 2]) * N + ck + e[:, 3]) + e[:, 0]
        tris[:, s] = np.searchsorted(vkeys, key)
    return verts, tris.astype(np.int32)
