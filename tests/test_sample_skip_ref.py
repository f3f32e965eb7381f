"""CPU checks of skip="samples": the float64 per-point rule (tests/sample_skip_ref.py) on hand cases, the workspace
query, and the argument errors raised before any launch."""
import ctypes

import numpy as np
import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib
from tests import sample_skip_ref as sk


def _words(cells, M):
    """Bit field with the cells (cx, cy, cz) occupied."""
    w = np.zeros((M ** 3 + 31) // 32, np.uint32)
    for cx, cy, cz in cells:
        c = (cz * M + cy) * M + cx
        w[c >> 5] |= np.uint32(1) << np.uint32(c & 31)
    return w.view(np.int32)


# N = 5 points over [0, 4]^3: cell c spans [c, c + 1] on every axis, so grid and world coordinates coincide
N, M, BOX = 5, 4, (0.0, 4.0, 0.0, 4.0, 0.0, 4.0)


def _ev(points, cells, ranges=BOX):
    return sk.point_evaluated(np.asarray(points, np.float32), _words(cells, M), N, ranges)


def test_interior_points():
    assert _ev([[1.5, 2.5, 0.5]], [(1, 2, 0)]).tolist() == [True]
    assert _ev([[1.5, 2.5, 0.5]], [(2, 2, 0)]).tolist() == [False]
    assert _ev([[0.25, 0.25, 0.25]], []).tolist() == [False]


def test_faces_edges_and_corners_touch_every_neighbour():
    occ = [(1, 1, 1)]
    # a point on a face, an edge and a corner of cell (1, 1, 1), seen from its neighbours
    assert _ev([[2.0, 1.5, 1.5], [1.0, 1.5, 1.5], [2.0, 2.0, 1.5], [1.0, 1.0, 1.0], [2.0, 2.0, 2.0]], occ).all()
    # one ulp outside the face is outside the cell
    assert not _ev([[np.nextafter(np.float32(2.0), np.float32(3.0)), 1.5, 1.5]], occ).any()
    assert not _ev([[np.nextafter(np.float32(1.0), np.float32(0.0)), 1.5, 1.5]], occ).any()
    # the corner (2, 2, 2) is shared by 8 cells: any of them will do
    for c in [(2, 2, 2), (1, 2, 2), (2, 1, 1), (1, 1, 2)]:
        assert _ev([[2.0, 2.0, 2.0]], [c]).tolist() == [True], c


def test_box_boundary_and_outside():
    occ = [(0, 0, 0), (3, 3, 3)]
    assert _ev([[0.0, 0.0, 0.0], [4.0, 4.0, 4.0], [0.0, 0.5, 1.0]], occ).tolist() == [True, True, True]
    assert not _ev([[-1e-6, 0.5, 0.5], [4.0000005, 3.5, 3.5], [np.nan, 0.5, 0.5], [np.inf, 3.5, 3.5]], occ).any()


def test_reversed_ranges():
    # y reversed: y = 4 is grid coordinate 0
    rev = (0.0, 4.0, 4.0, 0.0, 0.0, 4.0)
    assert _ev([[0.5, 3.5, 0.5]], [(0, 0, 0)], rev).tolist() == [True]
    assert _ev([[0.5, 0.5, 0.5]], [(0, 0, 0)], rev).tolist() == [False]
    assert _ev([[0.5, 3.0, 0.5]], [(0, 1, 0)], rev).tolist() == [True]      # the boundary y = 3 touches cell 1


def test_a_full_grid_evaluates_the_whole_closed_box():
    every = [(x, y, z) for x in range(M) for y in range(M) for z in range(M)]
    rng = np.random.default_rng(0)
    pts = rng.uniform(0, 4, (200, 3)).astype(np.float32)
    pts[:10] = np.floor(pts[:10])
    assert _ev(pts, every).all()


def test_plain_passes():
    rays = np.array([[0, 0, 0, 0, 0, 1, 2, 6],
                     [np.nan, 0, 0, 0, 0, 1, 2, 6],
                     [0, 0, 0, 0, 0, 1, 6, 2],
                     [0, 0, 0, 0, 0, 1e30, 2, 6]], np.float32)
    z = sk.z_base(rays, 32)
    assert sk.plain_rays(rays).tolist() == [False, True, True, False]
    assert sk.plain_pass(rays, z).tolist() == [False, True, True, True]     # 1e10 * |d| overflows


def test_mask_bits_round_trip():
    ev = np.random.default_rng(1).random((3, 192)) < 0.3
    words = np.zeros((3, 6), np.uint32)
    for r in range(3):
        for i in np.nonzero(ev[r])[0]:
            words[r, i >> 5] |= np.uint32(1) << np.uint32(i & 31)
    assert np.array_equal(sk.mask_bits(words.view(np.int32), 192), ev)


# ---- the C ABI -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


def test_workspace_bytes_and_shape_checks(lib):
    f = lib.nerfb200_samples_workspace_bytes
    assert f(1024, 64, 128) > f(1024, 64, 64) > f(512, 64, 64) > 0
    assert f(0, 64, 64) > 0
    for bad in ((-1, 64, 64), (16, 48, 64), (16, 64, 48), (16, 128, 96), (16, 64, -32), ((1 << 22) + 1, 64, 64)):
        assert f(*bad) == 0, bad


def test_render_samples_argument_checks(lib):
    out = ctypes.c_int64 * 2

    def call(**kw):
        a = dict(rays=256, n_rays=4, packed_coarse=256, packed_fine=256, n_samples=64, n_importance=64, bits=256, N=9,
                 ranges=(ctypes.c_double * 6)(-1, 1, -1, 1, -1, 1), opacity_coarse=256, rgb_fine=256, depth_fine=256,
                 opacity_fine=256, test_time=1)
        a.update(kw)
        return lib.nerfb200_render_samples(ctypes.byref(_lib.SamplesArgs(**a)), ctypes.c_void_p(256), 0, out(), None)

    for bad, msg in ((dict(n_samples=48), b"N_samples"), (dict(n_importance=16), b"N_samples"),
                     (dict(n_rays=-1), b"N_samples"), (dict(N=1), b"N must be"),
                     (dict(ranges=(ctypes.c_double * 6)(1, 1, -1, 1, -1, 1)), b"range"),
                     (dict(bits=None), b"NULL"), (dict(rgb_fine=None), b"fine"),
                     (dict(test_time=0), b"rgb_coarse"), (dict(rays=264), b"aligned"),
                     (dict(), b"workspace smaller")):
        rc = call(**bad)
        assert rc in (-1, -2) and msg in lib.nerfb200_last_error(), (bad, rc, lib.nerfb200_last_error())
    assert call(n_rays=0, rays=None) == 0                 # nothing to do: no pointer is needed


def test_python_argument_errors():
    grid = object.__new__(nb.OccupancyGrid)
    rays = torch.zeros(4, 8)
    with pytest.raises(ValueError, match="inference only"):
        nb.render_rays_culled([], [], rays, grid, perturb=1.0, skip="samples")
    with pytest.raises(ValueError, match="inference only"):
        nb.render_rays_culled([], [], rays, grid, noise_std=1.0, skip="samples")
    with pytest.raises(ValueError, match="skip must be"):
        nb.render_rays_culled([], [], rays, grid, skip="pixels")
    with pytest.raises(ValueError, match="needs an occupancy grid"):
        nb.batched_inference([], [], rays, 64, 64, False, skip="samples")
    with pytest.raises(ValueError, match="needs an occupancy grid"):
        nb.render_image([], [], 4, 4, 1.0, np.eye(3, 4), 2.0, 6.0, skip="samples")
    with pytest.raises(ValueError, match="skip must be"):
        nb.batched_inference([], [], rays, 64, 64, False, skip="none")
    with pytest.raises(ValueError, match="extras=True needs"):
        nb.render_rays_culled([], [], rays, grid, extras=True)
