"""The float64 restatement of cascaded occupancy grids (tests/cascade_ref.py) at its edges: which level a point
belongs to, which cells are inner, and that the per-level cell walk finds every occupied point of a segment."""
from fractions import Fraction

import numpy as np
import pytest

from . import cascade_ref as cr
from . import occupancy_ref as oc

BOX = (-1.0, 1.0, -0.5, 1.5, 2.0, 3.0)
REVERSED = (1.0, -1.0, -0.5, 1.5, 3.0, 2.0)


def test_level_ranges_double_the_half_extent_around_the_centre():
    assert cr.level_ranges(BOX, 0) == BOX
    assert cr.level_ranges(BOX, 1) == (-2.0, 2.0, -1.5, 2.5, 1.5, 3.5)
    assert cr.level_ranges(BOX, 3) == (-8.0, 8.0, -7.5, 8.5, -1.5, 6.5)
    assert cr.level_ranges(REVERSED, 2) == (4.0, -4.0, -3.5, 4.5, 4.5, 0.5)


@pytest.mark.parametrize("ranges", [BOX, REVERSED], ids=["forward", "reversed"])
def test_level_choice_at_faces_edges_and_corners(ranges):
    """A point on level k's closed box belongs to level k; just outside it, to level k + 1.  Faces, edges and
    corners of every level, the centre, NaN and points beyond the last level."""
    N, L = 9, 4
    c = np.array([0.5 * (ranges[2 * a] + ranges[2 * a + 1]) for a in range(3)])
    for k in range(L):
        r = cr.level_ranges(ranges, k)
        lo = np.minimum(r[0::2], r[1::2])
        hi = np.maximum(r[0::2], r[1::2])
        pts, want = [], []
        for sel in np.ndindex(3, 3, 3):             # 0: low side, 1: centre, 2: high side, per axis
            if sel == (1, 1, 1):
                continue
            on = np.array([(lo, c, hi)[s][a] for a, s in enumerate(sel)])
            pts.append(on)
            want.append(k)                                    # on a face, edge or corner of level k
            out = on + np.array([(-1, 0, 1)[s] for s in sel]) * 1e-9 * (hi - lo)
            pts.append(out)
            want.append(k + 1 if k + 1 < L else -1)           # just outside it
        got = cr.level_of(np.array(pts), N, L, ranges)
        assert got.tolist() == want, k
    assert cr.level_of(c[None], N, L, ranges).tolist() == [0]
    assert cr.level_of(np.array([[np.nan, c[1], c[2]], [c[0], c[1], 1e9]]), N, L, ranges).tolist() == [-1, -1]


def test_a_point_takes_its_own_levels_cells():
    """Level 0 empty, level 1 full: points inside level 0 are empty, points of level 1 are evaluated; a point on
    level 0's boundary belongs to level 0.  Level 1 with only inner cells set: nothing is evaluated."""
    N, L = 9, 2
    M = N - 1
    occ = np.zeros((L, M, M, M), bool)
    occ[1] = ~cr.inner_mask(N, 1)
    words = cr.pack(occ)
    pts = np.array([[0.0, 0.5, 2.5], [1.0, 0.5, 2.5], [1.5, 0.5, 2.5], [-1.9, -1.4, 1.6], [2.1, 0.5, 2.5]])
    assert cr.point_evaluated(pts, words, N, L, BOX).tolist() == [False, False, True, True, False]
    occ[1] = cr.inner_mask(N, 1)
    assert not cr.point_evaluated(pts, cr.pack(occ), N, L, BOX).any()


@pytest.mark.parametrize("M", list(range(1, 14)) + [16, 17, 32])
def test_inner_cells_are_exactly_those_inside_the_level_below(M):
    """The integer rule against exact rational boxes: a level-1 cell is inner iff its closed box lies inside level
    0's closed box, for M = 0 and != 0 mod 4; with M a multiple of 4 that is the middle half of each axis."""
    N = M + 1
    lo, hi = Fraction(-3), Fraction(5)                   # level 0; level 1 is [-7, 9]
    c, h = (lo + hi) / 2, (hi - lo) / 2
    lo1, step = c - 2 * h, 4 * h / M
    a, b = cr.inner_range(N, 1)
    for i in range(M):
        inside = lo <= lo1 + i * step and lo1 + (i + 1) * step <= hi
        assert inside == (a <= i < b), (M, i)
    if M % 4 == 0:
        assert (a, b) == (M // 4, 3 * M // 4)
    assert cr.inner_range(N, 0) == (0, 0)
    assert cr.inner_mask(N, 2).sum() == max(b - a, 0) ** 3


def test_noninner_cells_in_cell_order():
    for N in (2, 5, 9, 10):
        M = N - 1
        for k in (0, 1, 3):
            cells = cr.noninner_cells(N, k)
            a, b = cr.inner_range(N, k)
            assert np.all(np.diff(cells) > 0)
            assert len(cells) == M ** 3 - max(b - a, 0) ** 3
            cx, cy, cz = cells % M, (cells // M) % M, cells // (M * M)
            assert not np.any((cx >= a) & (cx < b) & (cy >= a) & (cy < b) & (cz >= a) & (cz < b))


def test_building_clears_inner_cells_before_and_after_the_dilation():
    """An inner cell marked by the corner rule neither stays occupied nor dilates into its neighbours; a non-inner
    cell dilates within its level only."""
    N, L = 9, 2
    M = N - 1
    cells = np.zeros((L, M, M, M), bool)
    cells[1, 3, 3, 3] = True                          # inner
    occ = cr.occupancy_levels(cells, 1)
    assert not occ.any()
    cells[1, 0, 0, 0] = True
    occ = cr.occupancy_levels(cells, 1)
    assert occ[1].sum() == 8 and occ[1, :2, :2, :2].all() and not occ[0].any()


def _segments(rng, n, ranges, L):
    far_box = np.array(cr.level_ranges(ranges, L - 1))
    c = 0.5 * (far_box[0::2] + far_box[1::2])
    ext = np.abs(far_box[1::2] - far_box[0::2])
    o = c + (rng.random((n, 3)) - 0.5) * ext * 1.4
    d = rng.standard_normal((n, 3))
    near = rng.random(n) * 0.5
    far = near + rng.random(n) * ext.max() * 1.2
    return np.concatenate([o, d, near[:, None], far[:, None]], 1).astype(np.float32)


@pytest.mark.parametrize("seed", range(4))
def test_the_walk_finds_every_occupied_point_of_a_segment(seed):
    """On random sparse cascades, every segment with a densely sampled float64 point that the lookup finds
    occupied is live.  The sampled points use the float32 ray values exactly (the walk's input)."""
    rng = np.random.default_rng(seed)
    N, L = (9, 10, 13, 17)[seed], (2, 3, 4, 2)[seed]
    ranges = (BOX, REVERSED)[seed % 2]
    M = N - 1
    occ = np.stack([(rng.random((M, M, M)) < 0.04) & ~cr.inner_mask(N, k) for k in range(L)])
    words = cr.pack(occ)
    rays = _segments(rng, 300, ranges, L)
    live = cr.ray_live(rays, words, N, L, ranges)
    r = rays.astype(np.float64)
    t = np.linspace(0.0, 1.0, 4001)
    z = r[:, 6:7] + (r[:, 7:8] - r[:, 6:7]) * t
    x = r[:, None, 0:3] + r[:, None, 3:6] * z[:, :, None]
    hit = cr.point_evaluated(x, words, N, L, ranges).any(1)
    assert not np.any(hit & ~live), np.nonzero(hit & ~live)[0]
    assert hit.sum() > 10 and (~live).sum() > 10        # both kinds of segment are there


def test_one_level_restates_the_one_level_rules():
    """With L = 1 the lookup, the packing and the walk are tests/sample_skip_ref's and tests/occupancy_ref's."""
    from . import sample_skip_ref as ss
    rng = np.random.default_rng(7)
    N = 11
    sigma = rng.random((1, N, N, N)).astype(np.float32) * (rng.random((1, N, N, N)) < 0.05)
    words = cr.pack_sigma(sigma, 0.5, 1)
    assert np.array_equal(words, oc.pack_bits(oc.occupancy(sigma[0], 0.5, 1)))
    x = (rng.random((2000, 3)) * 2.4 - 1.2).astype(np.float32) * np.array([1, 1, 0.5], np.float32) + \
        np.array([0, 0.5, 2.5], np.float32)
    assert np.array_equal(cr.point_evaluated(x, words, N, 1, BOX), ss.point_evaluated_vec(x, words, N, BOX))
    rays = _segments(rng, 200, BOX, 1)
    assert np.array_equal(cr.ray_live(rays, words, N, 1, BOX), oc.ray_live(rays, oc.unpack_bits(words, N),
                                                                          cr.pairs(BOX))[0])
