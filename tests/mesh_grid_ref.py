"""The evaluated lattice points of the mesh grids taken through an occupancy grid (``nb.sigma_grid(...,
occupancy=)``, ``nb.rgb_sigma_grid(..., occupancy=)``; DESIGN.md "Grids through an occupancy grid").

A lattice point is evaluated iff its float32 position (``oracle.mesh_oracle.grid_positions``) passes
``tests.sample_skip_ref.point_evaluated``, the rule of ``skip="samples"``.  ``lattice_evaluated`` is the same float64
rule, vectorised so that grids of millions of points can be checked; ``tests/test_mesh_grid_ref.py`` holds it equal to
``point_evaluated``.
"""
import numpy as np

from oracle import mesh_oracle as mo


def lattice_evaluated(x, words, N, ranges):
    """bool (n,) for float32 points x (n, 3): ``point_evaluated(x, words, N, ranges)``, vectorised.  A coordinate
    on a cell boundary takes the cells on both sides (c0 = c1 - 1), so the cells to test are {c0, c1} per axis."""
    x = np.asarray(x, np.float32).reshape(-1, 3)
    M = int(N) - 1
    lo = np.array(ranges[0::2], np.float64)
    hi = np.array(ranges[1::2], np.float64)
    g = (x.astype(np.float64) - lo) * (float(M) / (hi - lo))
    with np.errstate(invalid="ignore"):
        inside = np.all((g >= 0.0) & (g <= M), axis=1)
    g = np.where(inside[:, None], g, 0.0)
    f = np.floor(g)
    fl = f.astype(np.int64)
    c1 = np.minimum(fl, M - 1)
    c0 = np.where((f == g) & (fl > 0), fl - 1, c1)
    w = np.asarray(words).view(np.uint32)
    out = np.zeros(x.shape[0], bool)
    for corner in range(8):
        c = [np.where((corner >> a) & 1, c1[:, a], c0[:, a]) for a in range(3)]
        cell = (c[2] * M + c[1]) * M + c[0]
        out |= ((w[cell >> 5] >> (cell & 31).astype(np.uint32)) & 1) == 1
    return out & inside


def evaluated_points(N, x_range, y_range, z_range, words, occ_N, occ_ranges):
    """bool (N^3,) in flat lattice order: the evaluated points of the N-point mesh grid."""
    return lattice_evaluated(mo.grid_positions(N, x_range, y_range, z_range), words, occ_N, occ_ranges)


def random_words(occ_N, fill, seed):
    """uint32 words of a grid of (occ_N - 1)^3 cells, each occupied with probability ``fill`` (bits past the last
    cell 0)."""
    M = int(occ_N) - 1
    cells = np.random.default_rng(seed).random(M ** 3) < fill
    return pack_cells(cells)


def pack_cells(cells):
    """uint32 words of a flat bool cell array (cell (cz * M + cy) * M + cx, bit c % 32 of word c / 32)."""
    cells = np.asarray(cells, bool).reshape(-1)
    words = np.zeros((cells.size + 31) // 32, np.uint32)
    idx = np.nonzero(cells)[0]
    np.bitwise_or.at(words, idx >> 5, np.left_shift(np.uint32(1), (idx & 31).astype(np.uint32)))
    return words
