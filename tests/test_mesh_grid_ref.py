"""The evaluated-point rule of the mesh grids taken through an occupancy grid, on lattice points, in float64
(tests/mesh_grid_ref.py over tests/sample_skip_ref.point_evaluated): one occupied cell, shared faces, points outside
the grid's box, reversed ranges, and the vectorised replica against the per-point one."""
import itertools

import numpy as np
import pytest

from oracle import mesh_oracle as mo
from tests import mesh_grid_ref as mg
from tests import sample_skip_ref as sk

BOX = (-1.0, 1.0, -1.0, 1.0, -1.0, 1.0)


def _lattice(N, ranges):
    """(N^3, 3) positions and (N^3, 3) integer lattice coordinates (j, i, k) -> x, y, z index of each point."""
    pos = mo.grid_positions(N, ranges[0:2], ranges[2:4], ranges[4:6])
    i, j, k = np.meshgrid(np.arange(N), np.arange(N), np.arange(N), indexing="ij")
    return pos, np.stack([j.reshape(-1), i.reshape(-1), k.reshape(-1)], 1)


def _one_cell(occ_N, cell):
    M = occ_N - 1
    cells = np.zeros(M ** 3, bool)
    cx, cy, cz = cell
    cells[(cz * M + cy) * M + cx] = True
    return mg.pack_cells(cells)


@pytest.mark.parametrize("cell", [(0, 0, 0), (1, 2, 3), (3, 3, 3), (2, 0, 3)])
def test_one_occupied_cell_is_its_closed_box(cell):
    """Mesh N = 9 over the occupancy grid's box (N = 5): every cell spans 3 lattice points per axis, the middle one
    inside and two on its faces; exactly the 27 points of the closed box are evaluated."""
    pos, lat = _lattice(9, BOX)
    ev = sk.point_evaluated(pos, _one_cell(5, cell), 5, BOX)
    want = np.all((lat >= 2 * np.array(cell)) & (lat <= 2 * np.array(cell) + 2), 1)
    assert ev.sum() == 27 and np.array_equal(ev, want)
    assert np.array_equal(mg.lattice_evaluated(pos, _one_cell(5, cell), 5, BOX), want)


def test_shared_face_edge_and_corner_points_see_both_sides():
    """Mesh N = occupancy N: every lattice point is a cell corner.  One occupied cell makes its 8 corners evaluated,
    and nothing else; with its neighbour along x also occupied, the 12 corners of both."""
    pos, lat = _lattice(5, BOX)
    ev = sk.point_evaluated(pos, _one_cell(5, (1, 2, 0)), 5, BOX)
    want = np.all((lat >= [1, 2, 0]) & (lat <= [2, 3, 1]), 1)
    assert ev.sum() == 8 and np.array_equal(ev, want)
    M = 4
    cells = np.zeros(M ** 3, bool)
    cells[(0 * M + 2) * M + 1] = cells[(0 * M + 2) * M + 2] = True
    ev = sk.point_evaluated(pos, mg.pack_cells(cells), 5, BOX)
    assert ev.sum() == 12 and np.array_equal(ev, np.all((lat >= [1, 2, 0]) & (lat <= [3, 3, 1]), 1))


def test_points_outside_the_grid_box_are_empty():
    """A full grid over [-0.5, 0.5]^3 inside the mesh box [-1, 1]^3 (N = 9, spacing 0.25): exactly the points with
    every coordinate in [-0.5, 0.5] are evaluated, those on the box's faces included."""
    pos, lat = _lattice(9, BOX)
    inner = (-0.5, 0.5) * 3
    full = mg.pack_cells(np.ones(3 ** 3, bool))
    ev = sk.point_evaluated(pos, full, 4, inner)
    want = np.all((lat >= 2) & (lat <= 6), 1)
    assert ev.sum() == 125 and np.array_equal(ev, want)
    # a NaN and an infinite point are empty whatever the grid holds
    odd = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf]], np.float32)
    assert not sk.point_evaluated(odd, full, 4, inner).any()
    assert not mg.lattice_evaluated(odd, full, 4, inner).any()


def test_reversed_ranges_flip_the_cells():
    """With x_range (1, -1), cell cx = 0 spans x in [0.5, 1]; with every range reversed, cell (0, 0, 0) is the
    corner at (1, 1, 1)."""
    pos, lat = _lattice(9, BOX)
    rev_x = (1.0, -1.0, -1.0, 1.0, -1.0, 1.0)
    ev = sk.point_evaluated(pos, _one_cell(5, (0, 0, 0)), 5, rev_x)
    assert ev.sum() == 27 and np.array_equal(ev, np.all((lat >= [6, 0, 0]) & (lat <= [8, 2, 2]), 1))
    rev = (1.0, -1.0, 1.0, -1.0, 1.0, -1.0)
    ev = sk.point_evaluated(pos, _one_cell(5, (0, 0, 0)), 5, rev)
    assert ev.sum() == 27 and np.array_equal(ev, np.all(lat >= 6, 1))


RANGES = [(-1.5, 1.5) * 3, (-1.5, 1.5, -1.2, 1.4, -1.5, 1.3), (1.5, -1.5, -1.2, 1.4, 1.3, -1.5),
          (-0.9, 1.1, -1.0, 0.8, -1.1, 0.7)]


@pytest.mark.parametrize("mesh_r, occ_r", list(itertools.product(range(4), range(4))))
def test_vectorised_replica_equals_point_evaluated(mesh_r, occ_r):
    mesh, occ = RANGES[mesh_r], RANGES[occ_r]
    for N, occ_N, fill, seed in ((9, 5, 0.3, 0), (11, 4, 0.5, 1), (7, 7, 0.2, 2), (6, 2, 1.0, 3)):
        pos = mo.grid_positions(N, mesh[0:2], mesh[2:4], mesh[4:6])
        words = mg.random_words(occ_N, fill, seed + 10 * mesh_r + 100 * occ_r)
        assert np.array_equal(mg.lattice_evaluated(pos, words, occ_N, occ), sk.point_evaluated(pos, words, occ_N, occ))
