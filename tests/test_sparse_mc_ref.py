"""The sparse marching cubes restated in numpy (tests/sparse_mc_ref.py): the brick pre-filter never drops a brick
with an evaluated point, and the march on brick storage with sorted keys is oracle.mesh_oracle.marching_cubes of the
dense grid with the unevaluated points zeroed."""
import math

import numpy as np
import pytest

from oracle import mesh_oracle as mo
from tests import mesh_grid_ref as mg
from tests import sparse_mc_ref as sm

CUBE = ((-1.5, 1.5),) * 3
UNEQUAL = ((-1.5, 1.5), (-1.2, 1.4), (-1.5, 1.3))
REVERSED = ((1.5, -1.5), (-1.2, 1.4), (1.3, -1.5))
PARTLY_OUTSIDE = ((-0.4, 2.5), (-2.0, 0.9), (-0.7, 1.9))     # the grid box sticks out of CUBE on every axis
SIZES = (2, 3, 8, 9, 17, 33)


def _flat(r):
    return tuple(v for p in r for v in p)


def _check_superset(N, mesh, words, occ_N, occ, levels=1):
    cand = sm.candidate_bricks(N, *mesh, words, occ_N, _flat(occ), levels)
    ev = sm.evaluated_points(N, *mesh, words, occ_N, _flat(occ), levels)
    need = sm.brick_of_points(ev)
    assert not (need & ~cand).any(), np.argwhere(need & ~cand)[:5]
    return cand, need


@pytest.mark.parametrize("N", SIZES)
@pytest.mark.parametrize("box", ["cube", "unequal_reversed", "reversed_unequal", "partly_outside"])
def test_candidates_hold_every_evaluated_brick_random(N, box):
    mesh, occ = {"cube": (CUBE, CUBE), "unequal_reversed": (UNEQUAL, REVERSED), "reversed_unequal": (REVERSED, UNEQUAL),
                 "partly_outside": (CUBE, PARTLY_OUTSIDE)}[box]
    for occ_N, fill, seed in ((5, 0.2, 1), (17, 0.05, 2), (33, 0.01, 3), (2, 1.0, 0)):
        _check_superset(N, mesh, mg.random_words(occ_N, fill, seed), occ_N, occ)


@pytest.mark.parametrize("N", SIZES)
def test_candidates_of_single_cells_on_shared_faces_edges_and_corners(N):
    """Mesh lattice = occupancy lattice (every mesh point a cell corner, on faces, edges and corners of cells) and a
    half-step-shifted one; single occupied cells in turn (the first, the last and random ones)."""
    for occ_N, occ in ((min(N, 9), CUBE), (max(2, (min(N, 17) + 1) // 2), CUBE),
                       (5, ((-1.5, 1.5 + 3 / (2 * (N - 1))),) * 3)):
        M = occ_N - 1
        for c in np.unique(np.random.default_rng(N * occ_N).integers(0, M ** 3, 24).tolist() + [0, M ** 3 - 1]):
            cells = np.zeros(M ** 3, bool)
            cells[c] = True
            _check_superset(N, CUBE, mg.pack_cells(cells), occ_N, occ)


@pytest.mark.parametrize("levels", range(1, 9))
@pytest.mark.parametrize("N", [9, 17, 33])
def test_candidates_in_a_cascade(N, levels):
    occ_N = 5
    words = np.concatenate([mg.random_words(occ_N, 0.3, 100 * levels + k) for k in range(levels)])
    wide = ((-1.5 * 2 ** (levels - 1), 1.5 * 2 ** (levels - 1)),) * 3   # the mesh box over the last level's
    for mesh in (CUBE, wide, REVERSED):
        _check_superset(N, mesh, words, occ_N, ((-0.6, 0.7), (-0.5, 0.5), (0.8, -0.4)), levels)


def test_an_empty_grid_has_no_candidates():
    cand = sm.candidate_bricks(33, *CUBE, mg.random_words(9, 0.0, 0), 9, _flat(CUBE))
    assert not cand.any()


THRESHOLDS = [0.0, 20.0, -1.0, math.nan, math.inf, -math.inf]


def _field(N, seed):
    rng = np.random.default_rng(seed)
    i, j, k = np.meshgrid(*(np.linspace(-1, 1, N),) * 3, indexing="ij")
    s = 40 * np.exp(-3 * (i ** 2 + 0.7 * j ** 2 + 1.3 * k ** 2)) + rng.normal(0, 4, (N, N, N))
    return np.maximum(s, 0).astype(np.float32)


@pytest.mark.parametrize("N", SIZES)
@pytest.mark.parametrize("grid", ["random", "single_cell", "cascade", "full"])
def test_sparse_march_is_the_dense_march_of_the_zeroed_grid(N, grid):
    if grid == "random":
        words, occ_N, occ, L = mg.random_words(9, 0.3, N), 9, UNEQUAL, 1
    elif grid == "single_cell":
        words, occ_N, occ, L = mg.pack_cells(np.arange(27) == 13), 4, CUBE, 1
    elif grid == "cascade":
        words, occ_N, occ, L = np.concatenate([mg.random_words(5, 0.4, k) for k in range(3)]), 5, PARTLY_OUTSIDE, 3
    else:
        words, occ_N, occ, L = mg.random_words(3, 1.0, 0), 3, CUBE, 1
    sigma = _field(N, N)
    ev = sm.evaluated_points(N, *CUBE, words, occ_N, _flat(occ), L)
    zeroed = np.where(ev, sigma, np.float32(0))
    for thr in THRESHOLDS + [float(np.median(sigma))]:
        want_v, want_t = mo.marching_cubes(zeroed, thr)
        got_v, got_t = sm.sparse_march(sigma, ev, thr)
        assert np.array_equal(got_v.view(np.int64), want_v.view(np.int64)), thr
        assert np.array_equal(got_t, want_t), thr
