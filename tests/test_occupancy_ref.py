"""The float64 reference of empty-space skipping (tests/occupancy_ref.py) against geometry it can be checked on by
hand: an analytic sphere, the axis order on an asymmetric box, the bit packing at odd sizes, N = 2, and the guards
of the ray walk."""
import numpy as np
import pytest

from tests import occupancy_ref as oc

CUBE = ((-1.5, 1.5),) * 3


def _sigma_of(fn, N, ranges):
    """A sigma grid in nb.sigma_grid's order: sigma[i, j, k] = fn(x_j, y_i, z_k)."""
    x, y, z = (np.linspace(lo, hi, N) for lo, hi in ranges)
    X, Y, Z = np.meshgrid(x, y, z)            # 'xy' indexing, as extract_color_mesh.py builds the grid
    return fn(X, Y, Z).astype(np.float32)


def _rays_through(points, origins, near=0.0, far=20.0):
    d = points - origins
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    n = len(d)
    return np.concatenate([origins, d, np.full((n, 1), near), np.full((n, 1), far)], 1).astype(np.float32)


def test_analytic_sphere_rays_are_live_or_dead_as_geometry_says():
    N, R, r_dil = 49, 0.6, 2
    centre = np.array([0.2, -0.1, 0.3])
    sigma = _sigma_of(lambda X, Y, Z: 50.0 * ((X - centre[0]) ** 2 + (Y - centre[1]) ** 2 + (Z - centre[2]) ** 2 < R * R),
                      N, CUBE)
    occ = oc.occupancy(sigma, 10.0, r_dil)
    h = 3.0 / (N - 1)
    # the occupied set contains the ball and stays inside the ball grown by the dilation plus two cell diagonals
    grown = R + (r_dil + 2) * h * np.sqrt(3.0)
    rng = np.random.default_rng(3)
    n = 4000
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    origins = centre + 4.0 * u
    v = rng.normal(size=(n, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    # aim at a point at distance b from the centre, perpendicular to the viewing direction: b is the ray's miss distance
    perp = v - (v * u).sum(1, keepdims=True) * u
    perp /= np.linalg.norm(perp, axis=1, keepdims=True)
    b = rng.uniform(0.0, 1.4, n)
    rays = _rays_through(centre + b[:, None] * perp, origins)
    flag, _ = oc.ray_live(rays, occ, CUBE)
    inside, outside = b < R - h, b > grown
    assert inside.sum() > 500 and outside.sum() > 500
    assert flag[inside].all()
    assert not flag[outside].any()
    # a segment that ends before the ball, or starts behind it, is dead
    short = rays.copy()
    short[:, 7] = 4.0 - grown - 0.05
    assert not oc.ray_live(short, occ, CUBE)[0].any()
    late = rays.copy()
    late[:, 6] = 4.0 + grown + 0.05
    assert not oc.ray_live(late, occ, CUBE)[0].any()


def test_axis_order_on_an_asymmetric_box_with_one_occupied_cell():
    N = 6
    ranges = ((0.0, 5.0), (10.0, 20.0), (-3.0, -0.5))       # cells of 1 x 2 x 0.5
    cx, cy, cz = 3, 1, 4
    # one point above the threshold: x_3, y_1, z_4 -> sigma[i = 1 (y), j = 3 (x), k = 4 (z)]
    sigma = np.zeros((N, N, N), np.float32)
    sigma[1, 3, 4] = 9.0
    occ = oc.cells_from_sigma(sigma, 1.0)
    want = np.zeros((5, 5, 5), bool)
    want[2:4, 0:2, 3:5] = True                               # the 8 cells that have the point as a corner
    assert np.array_equal(occ, want)
    # a single cell, given directly
    occ = np.zeros((5, 5, 5), bool)
    occ[cx, cy, cz] = True
    words = oc.pack_bits(occ)
    c = (cz * 5 + cy) * 5 + cx
    assert words[c // 32] == np.uint32(1 << (c % 32)) and int(words.astype(np.uint64).sum()) == 1 << (c % 32)
    assert np.array_equal(oc.unpack_bits(words, N), occ)
    # the cell spans x [3, 4], y [12, 14], z [-1, -0.5]: rays along each axis through its centre are live, rays
    # through the centre of the transposed cell (cy, cx) are not
    mid = np.array([3.5, 13.0, -0.75])
    wrong = np.array([1.5, 17.0, -0.75])
    for axis in range(3):
        d = np.zeros(3)
        d[axis] = 1.0
        for centre, live in ((mid, True), (wrong, False)):
            o = centre - 30.0 * d
            ray = np.concatenate([o, d, [0.0, 100.0]]).astype(np.float32)[None]
            assert oc.ray_live(ray, occ, ranges)[0][0] == live, (axis, centre)
            assert oc.ray_live(ray * np.array([1, 1, 1, -1, -1, -1, 1, 1], np.float32) +
                               np.concatenate([60.0 * d, np.zeros(5)]).astype(np.float32), occ, ranges)[0][0] == live


@pytest.mark.parametrize("N", [2, 3, 5, 33, 34, 40])
def test_packing_round_trips_at_sizes_that_are_not_multiples_of_32(N):
    M = N - 1
    rng = np.random.default_rng(N)
    occ = rng.random((M, M, M)) < 0.3
    words = oc.pack_bits(occ)
    assert words.dtype == np.uint32 and len(words) == (M ** 3 + 31) // 32
    assert np.array_equal(oc.unpack_bits(words, N), occ)
    flat = occ.transpose(2, 1, 0).reshape(-1)                # c = (cz * M + cy) * M + cx
    for c in rng.integers(0, M ** 3, 50):
        assert bool((int(words[c // 32]) >> (c % 32)) & 1) == flat[c]
    if M ** 3 % 32:
        assert int(words[-1]) >> (M ** 3 % 32) == 0          # the padding bits are 0


def test_n_equals_two_is_one_cell():
    sigma = np.zeros((2, 2, 2), np.float32)
    assert oc.pack_bits(oc.occupancy(sigma, 0.5, 1)).tolist() == [0]
    sigma[1, 0, 1] = 1.0
    for r in (0, 1, 3):
        assert oc.pack_bits(oc.occupancy(sigma, 0.5, r)).tolist() == [1]
    occ = np.ones((1, 1, 1), bool)
    rays = np.array([[-3, 0.2, 0.1, 1, 0, 0, 0, 10],         # through the cell
                     [-3, 1.2, 0.1, 1, 0, 0, 0, 10],         # beside it
                     [-3, 0.2, 0.1, 1, 0, 0, 0, 1.5]], np.float32)   # ends before it
    assert oc.ray_live(rays, occ, ((-1.0, 1.0),) * 3)[0].tolist() == [True, False, False]


def test_dilation_is_chebyshev():
    occ = np.zeros((9, 9, 9), bool)
    occ[4, 3, 5] = True
    for r in (0, 1, 3):
        d = oc.dilate(occ, r)
        idx = np.indices(occ.shape)
        want = np.maximum.reduce([abs(idx[0] - 4), abs(idx[1] - 3), abs(idx[2] - 5)]) <= r
        assert np.array_equal(d, want)
    assert oc.dilate(occ, 20).all()


def test_ray_walk_guards():
    occ, box, rays, want = oc.guard_cases()
    flag, margin = oc.ray_live(rays, occ, box)
    assert flag.tolist() == want.tolist()
    assert (margin[~np.isfinite(rays).all(1) | (rays[:, 7] <= rays[:, 6])] == np.inf).all()
    # a reversed range names the same cells from the other end
    flag_r, _ = oc.ray_live(rays, occ[::-1], ((2.0, -2.0), (-2.0, 2.0), (-2.0, 2.0)))
    assert flag_r.tolist() == want.tolist()


def test_margin_flags_the_rays_that_graze_an_edge():
    occ = np.zeros((4, 4, 4), bool)
    occ[1, 2, 2] = True                                       # x [-1, 0] x y [0, 1] x z [0, 1]
    box = ((-2.0, 2.0),) * 3
    rays = np.array([[-5, -0.5, -0.5, 1, 0, 0, 0, 10],        # mid-cell all the way, half a cell from the cell
                     [-5, -0.5 - 1e-6, -0.5, 1, 1e-7, 0, 0, 10],
                     [-5, -1.0, -1.0, 1, 0.2, 0.2, 0, 10]],    # touches the cell only at its corner x = y = z = 0
                    np.float32)
    flag, margin = oc.ray_live(rays, occ, box)
    assert flag.tolist() == [False, False, True]
    assert margin[0] >= 0.49 and margin[1] >= 0.49 and margin[2] < 1e-4


def test_vacuum_values_and_scatter():
    keys = oc.result_keys(64, False)
    assert keys == list(oc.RESULT_KEYS)
    assert oc.result_keys(0, True) == ["opacity_coarse"]
    for wb in (False, True):
        v = oc.vacuum_results(5, keys, wb)
        assert (v["rgb_fine"] == (1.0 if wb else 0.0)).all() and v["rgb_fine"].shape == (5, 3)
        assert (v["opacity_fine"] == 0).all() and (v["depth_coarse"] == 0).all()
    compact = {"rgb_fine": np.arange(6, dtype=np.float32).reshape(2, 3), "opacity_fine": np.array([0.5, 0.25], np.float32)}
    out = oc.scatter(compact, np.array([1, 3]), 5, True)
    assert out["opacity_fine"].tolist() == [0, 0.5, 0, 0.25, 0]
    assert out["rgb_fine"].tolist() == [[1, 1, 1], [0, 1, 2], [1, 1, 1], [3, 4, 5], [1, 1, 1]]
