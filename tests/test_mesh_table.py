"""CPU checks of the coloured-mesh building blocks: the generated marching-cubes table, the numpy marching
cubes, the cv2.remap restatement and the grid-position formula (nerf_pl_b200.mesh; DESIGN.md)."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import gen_mc_table as gen  # noqa: E402
from oracle import mesh_oracle as mo  # noqa: E402

TABLE = gen.build_table()


def test_header_is_generated_from_the_script():
    with open(gen.HEADER) as f:
        assert f.read() == gen.render_header(TABLE)
    count, tab = mo.load_table()
    for c in range(256):
        assert count[c] == len(TABLE[c])
        assert [tuple(tab[c, 3 * t:3 * t + 3]) for t in range(count[c])] == TABLE[c]


def _crossing_edges(case):
    return {e for e in range(12) if ((case >> gen.edge_corners(e)[0]) & 1) != ((case >> gen.edge_corners(e)[1]) & 1)}


@pytest.mark.parametrize("case", range(256))
def test_case_vertices_are_exactly_the_sign_changing_edges(case):
    used = {e for t in TABLE[case] for e in t}
    assert used == _crossing_edges(case)


@pytest.mark.parametrize("case", range(256))
def test_case_boundary_equals_face_segments_and_is_closed(case):
    edges = {}
    for t in TABLE[case]:
        for a, b in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])):
            edges.setdefault(frozenset((a, b)), []).append((a, b))
    segs = {frozenset(s) for s in gen.case_segments(case)}
    # inside the cube every edge is in two triangles (opposite directions) unless it is a face segment
    for k, uses in edges.items():
        if k in segs:
            assert len(uses) == 1, (case, k)
        else:
            assert len(uses) == 2 and uses[0] == uses[1][::-1], (case, k, uses)
    assert segs <= set(edges)
    # the directed boundary is the oriented face segments
    boundary = {uses[0] for k, uses in edges.items() if k in segs}
    assert boundary == set(gen.case_segments(case))


@pytest.mark.parametrize("case", range(256))
def test_face_rule_sees_only_the_face(case):
    """Two cells sharing a face draw the same segments there in opposite directions."""
    for axis in range(3):
        others = [a for a in range(3) if a != axis]
        f_lo = [f for f in gen.FACES if f[0][axis] == -1][0]
        f_hi = [f for f in gen.FACES if f[0][axis] == 1][0]
        # neighbour along +axis: its low face holds our high face's corners
        nb = 0
        for c in range(8):
            if (c >> axis) & 1 and (case >> c) & 1:
                nb |= 1 << (c & ~(1 << axis))
        ours = gen.face_segments(case, f_hi)
        theirs = gen.face_segments(nb, f_lo)

        def shift(e):   # an edge of our high face as the neighbour names it
            a, b = gen.edge_corners(e)
            return gen.EDGE_OF[frozenset((a & ~(1 << axis), b & ~(1 << axis)))]
        assert {(shift(p), shift(q)) for p, q in ours} == {(q, p) for p, q in theirs}, (case, axis, others)


@pytest.mark.parametrize("case", range(1, 255))
def test_orientation_points_from_inside_to_outside(case):
    """Every face segment p -> q has n x (q - p) pointing away from the inside: the face corners behind the
    segment are inside corners.  With the boundary test above this orients every triangle inside -> outside."""
    for n, cyc in gen.FACES:
        for p, q in gen.face_segments(case, (n, cyc)):
            a, b = np.array(gen.edge_mid(p)), np.array(gen.edge_mid(q))
            side = [np.dot(np.cross(n, b - a), np.array(gen.corner_pos(c)) - a) for c in cyc]
            behind = [c for c, s_ in zip(cyc, side) if s_ < 0]
            assert behind and all((case >> c) & 1 for c in behind), (case, n, p, q)


def _brute_mc(sigma, thr):
    """Per cell, straight from the table: the reference the vectorised oracle must reproduce."""
    n0, n1, n2 = sigma.shape
    inside = sigma.astype(np.float64) > thr
    vid = {}
    verts = []
    for i in range(n0):
        for j in range(n1):
            for k in range(n2):
                for a in range(3):
                    q = [i, j, k]
                    q[a] += 1
                    if q[a] < sigma.shape[a] and inside[i, j, k] != inside[tuple(q)]:
                        f0, f1 = float(sigma[i, j, k]), float(sigma[tuple(q)])
                        v = [float(i), float(j), float(k)]
                        v[a] += (thr - f0) / (f1 - f0)
                        vid[(i, j, k, a)] = len(verts)
                        verts.append(v)
    tris = []
    for i in range(n0 - 1):
        for j in range(n1 - 1):
            for k in range(n2 - 1):
                case = sum(int(inside[i + (c & 1), j + ((c >> 1) & 1), k + ((c >> 2) & 1)]) << c for c in range(8))
                for t in TABLE[case]:
                    row = []
                    for e in t:
                        a, d = mo.edge_geometry(e)
                        row.append(vid[(i + d[0], j + d[1], k + d[2], a)])
                    tris.append(row)
    return np.array(verts).reshape(-1, 3), np.array(tris, dtype=np.int32).reshape(-1, 3)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_numpy_marching_cubes_matches_the_table(seed):
    rng = np.random.default_rng(seed)
    sigma = rng.normal(0, 1, (6, 7, 5)).astype(np.float32)
    v, t = mo.marching_cubes(sigma, 0.1)
    bv, bt = _brute_mc(sigma, 0.1)
    assert np.array_equal(v, bv)
    assert np.array_equal(t, bt)


def _sphere(n, r, c=None):
    c = (np.array([n / 2 - 0.3, n / 2 + 0.2, n / 2 + 0.1]) if c is None else np.asarray(c))
    g = np.stack(np.meshgrid(*(np.arange(n),) * 3, indexing="ij"), -1).astype(np.float64)
    return (r - np.linalg.norm(g - c, axis=-1)).astype(np.float32)


def test_numpy_marching_cubes_sphere_is_closed_and_outward():
    sigma = _sphere(14, 4.3)
    v, t = mo.marching_cubes(sigma, 0.0)
    e = np.sort(np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]]), 1)
    _, cnt = np.unique(e, axis=0, return_counts=True)
    assert (cnt == 2).all()
    assert len(v) - len(cnt) + len(t) == 2
    n = np.cross(v[t[:, 1]] - v[t[:, 0]], v[t[:, 2]] - v[t[:, 0]])
    out = v[t].mean(1) - np.array([14 / 2 - 0.3, 14 / 2 + 0.2, 14 / 2 + 0.1])
    assert (np.einsum("ij,ij->i", n, out) > 0).all()


def test_remap_replica_equals_golden_fixture(golden_dir):
    d = np.load(os.path.join(golden_dir, "remap_cv2.npz"))
    assert np.array_equal(mo.remap_bilinear(d["image"], d["xy"][:, 0], d["xy"][:, 1]), d["out"])


@pytest.mark.parametrize("seed", [0, 1])
def test_remap_replica_equals_cv2(seed):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(seed)
    H, W = 37, 53
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    f = np.arange(32, dtype=np.float32) / 32
    fx, fy = np.meshgrid(f, f)
    xy = np.concatenate([
        np.stack([7 + fx.ravel(), 9 + fy.ravel()], 1),
        np.stack([W - 2 + fx.ravel(), H - 2 + fy.ravel()], 1).clip(0, [W - 1, H - 1]),
        rng.uniform(0, 1, (20000, 2)) * [W - 1, H - 1],
        [[W - 1, H - 1], [0, 0], [W - 1, 0], [0, H - 1]]]).astype(np.float32)
    ref = cv2.remap(img, xy[:, 0].copy(), xy[:, 1].copy(), interpolation=cv2.INTER_LINEAR)[:, 0]
    assert np.array_equal(mo.remap_bilinear(img, xy[:, 0], xy[:, 1]), ref)


@pytest.mark.parametrize("N,rng_", [(2, (-1.0, 1.0)), (33, (-1.5, 1.5)), (128, (-1.5, 1.5)), (257, (-0.3, 1.7)),
                                    (100, (0.1, 0.1 + 1e-7))])
def test_grid_formula_equals_linspace_meshgrid(N, rng_):
    """The kernel's x_j = fl32(fl64(fl64(j * step) + lo)), last = hi, equals linspace -> meshgrid -> float32."""
    lo, hi = rng_
    step = (hi - lo) / (N - 1)
    j = np.arange(N, dtype=np.float64)
    ax = (j * step + lo)
    ax[-1] = hi
    ax32 = ax.astype(np.float32)
    assert np.array_equal(ax32, np.linspace(lo, hi, N).astype(np.float32))
    if N <= 33:
        pts = mo.grid_positions(N, (lo, hi), (lo - 0.5, hi), (lo, hi + 0.25))
        ys = np.linspace(lo - 0.5, hi, N).astype(np.float32)
        zs = np.linspace(lo, hi + 0.25, N).astype(np.float32)
        i, jj, k = np.unravel_index(np.arange(N ** 3), (N, N, N))
        assert np.array_equal(pts, np.stack([ax32[jj], ys[i], zs[k]], 1))


def test_to_world_quirks():
    v = np.array([[1.0, 2.0, 3.0], [0.0, 0.0, 0.0]])
    w = mo.to_world(v, 4, (0.0, 1.0), (10.0, 12.0), (-1.0, 1.0))
    assert np.allclose(w[0], [10 + 2 * 0.5, 0.25, -1 + 2 * 0.75])
