"""Sparse marching cubes through an occupancy grid (nb.sparse_marching_cubes, nb.extract_mesh(..., occupancy=);
csrc/sparse_mc_kernels.cuh, DESIGN.md §10i).

Wherever the dense route runs, the sparse mesh is ``marching_cubes(sigma_grid(..., occupancy=grid), threshold)`` bit
for bit and in the same order, independent of the CTA count.  Beyond the dense limit (N_grid 1024 and 1536) it is
held to a windowed oracle (the masked rule, nb.query_sigma and nb.marching_cubes on 48^3 windows), and its largest
cluster to a closed, consistently oriented manifold; its memory stays below the dense sigma grid's."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as mo
from oracle import nerf_oracle as orc
from tests import cases
from tests import mesh_grid_ref as mg

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUBE = ((-1.5, 1.5),) * 3
UNEQUAL = ((-1.5, 1.5), (-1.2, 1.4), (-1.5, 1.3))
REVERSED = ((1.5, -1.5), (-1.2, 1.4), (1.3, -1.5))
INSIDE = ((-0.9, 1.1), (-1.0, 0.8), (-1.1, 0.7))


def _nb():
    import nerf_pl_b200 as nb
    return nb


_M = {}


def _model(kind="random"):
    if kind not in _M:
        w = cases.trained_weights()[1] if kind == "trained" else orc.make_weights(21)
        m = _nb().NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        _M[kind] = m.cuda().eval()
    return _M[kind]


def _grid(words, occ_N, ranges, levels=1):
    bits = torch.from_numpy(np.asarray(words, np.uint32).view(np.int32)).cuda()
    return _nb().OccupancyGrid(bits, occ_N, *ranges, levels=levels)


def _same(a, b):
    (v0, t0), (v1, t1) = a, b
    assert v0.shape == v1.shape and t0.shape == t1.shape, (v0.shape, v1.shape, t0.shape, t1.shape)
    assert torch.equal(v0.view(torch.int64), v1.view(torch.int64)) and torch.equal(t0, t1)


def _dense(model, N, mesh, grid, thr):
    return _nb().marching_cubes(_nb().sigma_grid(model, N, *mesh, occupancy=grid), thr)


def _grids():
    """(name, words, occ_N, occupancy box, levels) of the grids the identity is checked on."""
    cascade = np.concatenate([mg.random_words(9, f, 30 + k) for k, f in enumerate((0.4, 0.2, 0.1))])
    return [("random", mg.random_words(17, 0.2, 1), 17, UNEQUAL, 1),
            ("reversed", mg.random_words(9, 0.3, 2), 9, REVERSED, 1),
            ("inside", mg.random_words(33, 0.1, 3), 33, INSIDE, 1),
            ("single_cell", mg.pack_cells(np.arange(16 ** 3) == (7 * 16 + 9) * 16 + 4), 17, CUBE, 1),
            ("full", mg.random_words(5, 1.0, 0), 5, CUBE, 1),
            ("cascade3", cascade, 9, INSIDE, 3)]


THRESHOLDS = [0.0, 20.0, -1.0, float("nan"), float("inf")]


@pytest.mark.parametrize("N", [2, 9, 17, 64, 127, 256])
@pytest.mark.parametrize("gi", range(6))
def test_identical_to_the_dense_route(N, gi):
    nb = _nb()
    name, words, occ_N, box, levels = _grids()[gi]
    model = _model()
    grid = _grid(words, occ_N, box, levels)
    sigma = nb.sigma_grid(model, N, *CUBE, occupancy=grid)
    vals = sigma[sigma > 0]
    thrs = THRESHOLDS + ([float(vals.median())] if vals.numel() else [])
    nonempty = 0
    for thr in thrs:
        want = nb.marching_cubes(sigma, thr)
        got = nb.sparse_marching_cubes(model, N, *CUBE, thr, occupancy=grid)
        _same(got, want)
        nonempty += len(want[1]) > 0
    if N >= 64 and name != "single_cell":
        assert nonempty >= 1, name


def test_trained_weights_at_512_before_and_after_the_cluster_filter():
    if not cases.have_trained():
        pytest.skip("no trained weights")
    nb = _nb()
    fine = _model("trained")
    grid = nb.occupancy_grid(fine, 128, *CUBE, 1.0, dilate=1)
    want = _dense(fine, 512, CUBE, grid, 20.0)
    got = nb.sparse_marching_cubes(fine, 512, *CUBE, 20.0, occupancy=grid)
    _same(got, want)
    assert len(got[1]) > 100000
    for keep in (False, True):
        w = nb.mesh.keep_largest_cluster(nb.mesh.to_world(want[0], 512, *CUBE), want[1]) if keep else \
            (nb.mesh.to_world(want[0], 512, *CUBE), want[1])
        v, t = nb.extract_mesh(fine, 512, *CUBE, 20.0, keep_largest=keep, occupancy=grid)
        assert torch.equal(v.view(torch.int32), w[0].view(torch.int32)) and torch.equal(t, w[1]), keep


_SUBPROCESS = r"""
import sys
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
import nerf_pl_b200 as nb
from oracle import nerf_oracle as orc
m = nb.NeRF()
m.load_state_dict({k: torch.from_numpy(v) for k, v in orc.make_weights(21).items()})
m = m.cuda().eval()
words = np.load(sys.argv[2])
grid = nb.OccupancyGrid(torch.from_numpy(words.view(np.int32)).cuda(), 17, (1.5, -1.5), (-1.2, 1.4), (1.3, -1.5))
box = ((-1.5, 1.5),) * 3
out = {}
for i, thr in enumerate((0.0, float(sys.argv[4]))):
    v, t = nb.sparse_marching_cubes(m, 83, *box, thr, occupancy=grid)
    out[f"v{i}"], out[f"t{i}"] = v.cpu().numpy(), t.cpu().numpy()
np.savez(sys.argv[3], **out)
"""


def test_independent_of_the_cta_count(tmp_path):
    nb = _nb()
    words = mg.random_words(17, 0.3, 5)
    grid = _grid(words, 17, REVERSED)
    sigma = nb.sigma_grid(_model(), 83, *CUBE, occupancy=grid)
    thr = float(sigma[sigma > 0].median())
    np.save(tmp_path / "w.npy", words)
    env = dict(os.environ, NERFB200_MAX_CTAS="1")
    subprocess.run([sys.executable, "-c", _SUBPROCESS, ROOT, str(tmp_path / "w.npy"), str(tmp_path / "o.npz"),
                    repr(thr)], check=True, env=env, cwd=ROOT)
    z = np.load(tmp_path / "o.npz")
    for i, t in enumerate((0.0, thr)):
        v, tr = nb.sparse_marching_cubes(_model(), 83, *CUBE, t, occupancy=grid)
        assert np.array_equal(z[f"v{i}"].view(np.int64), v.cpu().numpy().view(np.int64))
        assert np.array_equal(z[f"t{i}"], tr.cpu().numpy())
    assert len(z["t1"]) > 0


# ---- beyond the dense limit: the trained weights with the grid of the trained scene ---------------------------------
_BIG = {}


def _trained_big(N):
    if not cases.have_trained():
        pytest.skip("no trained weights")
    nb = _nb()
    if "grid" not in _BIG:
        _BIG["grid"] = nb.occupancy_grid(_model("trained"), 128, *CUBE, 1.0, dilate=1)
    if N not in _BIG:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        mesh = nb.sparse_marching_cubes(_model("trained"), N, *CUBE, 20.0, occupancy=_BIG["grid"])
        torch.cuda.synchronize()
        _BIG[N] = (mesh, torch.cuda.max_memory_allocated() - base)
    return _BIG[N][0], _BIG["grid"]


def _edge_keys(v):
    """(lower endpoint (n, 3) int64, axis (n,)) of index-space vertices: the coordinate off the lattice is the axis."""
    f = np.floor(v)
    frac = v - f
    axis = np.argmax(frac, 1)
    return f.astype(np.int64), axis


def _window_mesh(model, grid, N, o, W):
    nb = _nb()
    ax = [mo.grid_axis(*CUBE[a], N).astype(np.float32) for a in range(3)]
    i, j, k = (np.arange(o[a], o[a] + W) for a in range(3))
    I, J, K = np.meshgrid(i, j, k, indexing="ij")
    x = np.stack([ax[0][J], ax[1][I], ax[2][K]], -1).reshape(-1, 3)
    words = grid.bits.cpu().numpy().view(np.uint32)
    ev = mg.lattice_evaluated(x, words, grid.N, grid.ranges)
    s = np.zeros(len(x), np.float32)
    if ev.any():
        q = nb.query_sigma(model, torch.from_numpy(x[ev]).cuda()).cpu().numpy()
        s[ev] = np.maximum(q, 0)
        s[ev] = np.where(np.isnan(q), q, s[ev])
    v, _ = nb.marching_cubes(torch.from_numpy(s.reshape(W, W, W)).cuda(), 20.0)
    return v.cpu().numpy()


@pytest.mark.parametrize("N", [1024, 1536])
def test_windows_against_the_dense_oracle(N):
    (v, t), grid = _trained_big(N)
    assert len(t) > 0
    vh = v.cpu().numpy()
    W = 48
    rng = np.random.default_rng(N)
    for pick in rng.choice(len(vh), 4, replace=False):
        o = np.clip(np.floor(vh[pick]).astype(np.int64) - W // 2, 0, N - W)
        wv = _window_mesh(_model("trained"), grid, N, o, W)
        lo, ax = _edge_keys(vh)
        up = lo + np.eye(3, dtype=np.int64)[ax]
        inside = np.all((lo >= o) & (up < o + W), 1)
        sv = vh[inside]
        wlo, wax = _edge_keys(wv)
        assert len(wv) == len(sv) > 0
        got = np.lexsort(((lo[inside] - o) @ [W * W, W, 1] * 3 + ax[inside],))
        want = np.lexsort(((wlo) @ [W * W, W, 1] * 3 + wax,))
        gk = ((lo[inside] - o) @ [W * W, W, 1] * 3 + ax[inside])[got]
        wk = (wlo @ [W * W, W, 1] * 3 + wax)[want]
        assert np.array_equal(gk, wk)
        np.testing.assert_allclose(sv[got], wv[want] + o, rtol=0, atol=4 * np.finfo(np.float64).eps * N)


def _defects(v, t, N):
    """Directed edges of the largest cluster used twice (not oriented or not manifold) and without their reverse
    (open), over all directed edges."""
    nb = _nb()
    vw, tw = nb.mesh.keep_largest_cluster(nb.mesh.to_world(v, N, *CUBE), t)
    tt = tw.long()
    V = len(vw)
    d = torch.cat([tt[:, [0, 1]], tt[:, [1, 2]], tt[:, [2, 0]]])
    fwd = torch.unique(d[:, 0] * V + d[:, 1])
    rev = torch.unique(d[:, 1] * V + d[:, 0])
    twice = d.shape[0] - fwd.numel()
    open_ = fwd.numel() - int(torch.isin(fwd, rev).sum())
    return len(tw), twice / d.shape[0], open_ / d.shape[0]


@pytest.mark.parametrize("N", [1024, 1536])
def test_largest_cluster_is_a_closed_oriented_manifold(N):
    """Closed: every directed edge of the largest cluster has its reverse.  Oriented and manifold up to the case
    table's ambiguous faces, which the dense route has too: no more directed edges used twice, relative to its size,
    than the dense route's mesh at N_grid 512."""
    nb = _nb()
    (v, t), grid = _trained_big(N)
    kept, twice, open_ = _defects(v, t, N)
    assert kept > 0.5 * len(t)
    _, twice512, open512 = _defects(*_dense(_model("trained"), 512, CUBE, grid, 20.0), 512)
    print(f"N_grid {N}: {kept} kept triangles, directed edges used twice {twice:.2e} (512: {twice512:.2e}), "
          f"open {open_:.2e} (512: {open512:.2e})")
    assert open_ == 0 == open512                                       # closed
    assert twice <= twice512 and twice < 5e-4                          # oriented, up to the table's ambiguous faces


def test_vertex_count_grows_with_the_surface():
    """Four times the surface area's lattice edges, and more: the 1024 lattice resolves structure of the trained field
    that the 512 one steps over (measured 4.88 on the trained test weights)."""
    nb = _nb()
    (v, t), grid = _trained_big(1024)
    v512, _ = nb.sparse_marching_cubes(_model("trained"), 512, *CUBE, 20.0, occupancy=grid)
    print(f"vertices 512: {len(v512)}, 1024: {len(v)}; ratio {len(v) / len(v512):.3f}")
    assert 3.5 <= len(v) / len(v512) <= 5.0


def test_memory_below_the_dense_sigma_grid():
    _trained_big(1024)
    peak = _BIG[1024][1]
    print(f"N_grid 1024: peak {peak / 2 ** 30:.3f} GiB above the start, dense sigma grid {1024 ** 3 * 4 / 2 ** 30:.3f} GiB")
    assert 0 < peak < 1024 ** 3 * 4


def test_colours_of_the_1024_mesh():
    nb = _nb()
    (v, t), grid = _trained_big(1024)
    vw, tw = nb.mesh.keep_largest_cluster(nb.mesh.to_world(v, 1024, *CUBE), t)
    from tests.test_gpu_mesh_grid import _views
    images, poses, focal, near = _views()
    cols = nb.fuse_vertex_colors(_model("trained"), vw, images[:2], poses[:2], focal, near, occupancy=grid)
    assert cols.shape == (len(vw), 3) and cols.dtype == torch.uint8
    coarse = _nb().NeRF()
    coarse.load_state_dict({k: torch.from_numpy(w) for k, w in cases.trained_weights()[0].items()})
    coarse = coarse.cuda().eval()
    ncols = nb.normal_vertex_colors(coarse, _model("trained"), vw, tw, 2.0, 6.0, occupancy=grid)
    assert ncols.shape == (len(vw), 3) and ncols.dtype == torch.uint8


def test_argument_errors():
    nb = _nb()
    model = _model()
    grid = _grid(mg.random_words(9, 0.5, 0), 9, CUBE)
    for N in (1, 0, -3, 2049, 4096):
        with pytest.raises(ValueError, match=r"\[2, 2048\]"):
            nb.sparse_marching_cubes(model, N, *CUBE, 20.0, occupancy=grid)
        with pytest.raises(ValueError, match=r"\[2, 2048\]"):
            nb.extract_mesh(model, N, *CUBE, 20.0, occupancy=grid)
    for bad in (grid.bits, nb.DensityGrid(9, *CUBE), "grid", None):
        with pytest.raises(ValueError, match="OccupancyGrid"):
            nb.sparse_marching_cubes(model, 9, *CUBE, 20.0, occupancy=bad)
    # an empty grid: an empty mesh
    v, t = nb.sparse_marching_cubes(model, 33, *CUBE, -1.0, occupancy=_grid(mg.random_words(9, 0.0, 0), 9, CUBE))
    assert v.shape == (0, 3) and t.shape == (0, 3) and v.dtype == torch.float64 and t.dtype == torch.int32
