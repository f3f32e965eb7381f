"""The float64 restatement of the baked-volume render (tests/baked_ref.py, DESIGN.md §10j) against closed forms: a
constant-sigma slab, an empty grid, a field that pins the 'xy' axis order, rays that miss the box, start inside it,
run along a lattice plane or have far <= near, and the early-stop bound."""
import numpy as np
import pytest

from tests import baked_ref as br

BOX = (-1.0, 1.0, -1.0, 1.0, -1.0, 1.0)


def _lattice(N, ranges=BOX):
    """x, y, z of rgb_sigma_grid's lattice (float32 linspace), and the (N, N, N) coordinates in its 'xy' order."""
    ax = [np.linspace(ranges[2 * a], ranges[2 * a + 1], N).astype(np.float32) for a in range(3)]
    X, Y, Z = np.meshgrid(*ax)          # 'xy': X[i, j, k] = x_j, Y[i, j, k] = y_i
    return ax, X, Y, Z


def _grid(N, sigma, rgb=(0.25, 0.5, 0.75)):
    g = np.zeros((N, N, N, 4), np.float32)
    g[..., :3] = rgb
    g[..., 3] = sigma
    return g


def _ray(o, d, near, far):
    return np.array([[*o, *d, near, far]], np.float32)


def test_constant_slab_matches_the_closed_form():
    N, sigma = 17, 3.0
    g = _grid(N, sigma)
    s = br.default_step(N, BOX)
    for d in ((1, 0, 0), (0, 0.6, 0.8), (0.48, -0.6, 0.64)):
        rays = _ray((0.1, -0.2, 0.05), d, 0.0, 0.7)        # inside the box from near to far
        out = br.render(g, BOX, rays)
        K = int(out["K"][0])
        dt = np.float32(np.float32(s) / np.float32(np.linalg.norm(np.float32(d))))
        assert K == int(np.floor(np.float32(0.7) / dt))
        want = 1 - np.exp(-sigma * float(np.float32(s)) * K)
        np.testing.assert_allclose(out["opacity"][0], want, rtol=1e-12)
        np.testing.assert_allclose(out["rgb"][0], np.array([0.25, 0.5, 0.75], np.float32) * want, rtol=1e-6)
        # depth: sum_k w_k t_k with w_k = (1 - a) ^ k a, t_k = (k + 1/2) dt
        a = 1 - np.exp(-sigma * float(np.float32(s)))
        k = np.arange(K)
        np.testing.assert_allclose(out["depth"][0], np.sum(a * (1 - a) ** k * (k + 0.5) * float(dt)), rtol=1e-5)


def test_empty_grid_gives_the_vacuum_value():
    g = _grid(9, 0.0, rgb=(0.9, 0.9, 0.9))
    rays = np.concatenate([_ray((0, 0, -3), (0, 0, 1), 0.0, 6.0), _ray((0.3, 0.2, 0.1), (1, 1, 1), 0.0, 2.0)])
    for wb in (False, True):
        out = br.render(g, BOX, rays, white_back=wb)
        np.testing.assert_array_equal(out["opacity"], 0)
        np.testing.assert_array_equal(out["depth"], 0)
        np.testing.assert_array_equal(out["rgb"], 1.0 if wb else 0.0)


def test_axis_order_is_xy():
    """sigma only where y > 0.5 (axis 0 of the grid); red follows x (axis 1), green y, blue z (axis 2)."""
    N = 33
    _, X, Y, Z = _lattice(N)
    g = np.zeros((N, N, N, 4), np.float32)
    g[..., 0], g[..., 1], g[..., 2] = (X + 1) / 2, (Y + 1) / 2, (Z + 1) / 2
    g[..., 3] = np.where(Y > 0.5, 50.0, 0.0)
    along_x = np.concatenate([_ray((-2, 0.75, 0.0), (1, 0, 0), 0.0, 4.0), _ray((-2, -0.75, 0.0), (1, 0, 0), 0.0, 4.0)])
    out = br.render(g, BOX, along_x)
    assert out["opacity"][0] > 0.999 and out["opacity"][1] == 0
    # a ray along z at (x, y) = (-0.5, 0.75): red (x + 1) / 2 = 0.25, green 0.875, blue the first samples' z (~0)
    out = br.render(g, BOX, _ray((-0.5, 0.75, -2), (0, 0, 1), 0.0, 4.0))
    np.testing.assert_allclose(out["rgb"][0, :2], [0.25, 0.875], atol=1e-6)
    assert out["rgb"][0, 2] < 0.05
    # the same ray along x instead: blue (z + 1) / 2 = 0.5 and red the first samples' x (~0)
    out = br.render(g, BOX, _ray((-2, 0.75, 0.0), (1, 0, 0), 0.0, 4.0))
    np.testing.assert_allclose(out["rgb"][0, 1:], [0.875, 0.5], atol=1e-6)
    assert out["rgb"][0, 0] < 0.05


def test_edge_rays():
    N, sigma = 17, 2.0
    g = _grid(N, sigma)
    s = float(np.float32(br.default_step(N, BOX)))
    rays = np.concatenate([
        _ray((-3, 2, 0), (1, 0, 0), 0.0, 6.0),           # misses the box (y = 2)
        _ray((-3, -3, -3), (-1, 0, 0), 0.0, 6.0),        # points away
        _ray((0, 0, 0), (0, 0, 1), 0.0, 5.0),            # starts inside: samples z = (k + 1/2) s up to the face z = 1
        _ray((-3, 0.125, -0.5), (1, 0, 0), 0.0, 6.0),    # along the lattice plane y = 0.125 (an exact lattice y)
        _ray((0, 0, 0), (0, 0, 1), 1.0, 1.0),            # far == near
        _ray((0, 0, 0), (0, 0, 1), 2.0, 1.0),            # far < near
        _ray((0, 0, 0), (0, 0, 0), 0.0, 1.0),            # |d| = 0
        _ray((0, 0, np.nan), (0, 0, 1), 0.0, 1.0),       # non-finite
        _ray((0, 0, 0), (0, 0, 1), 0.0, np.inf),         # non-finite far
    ])
    out = br.render(g, BOX, rays)
    for r in (0, 1, 4, 5, 6, 7, 8):
        assert out["opacity"][r] == 0 and out["depth"][r] == 0 and not out["rgb"][r].any(), r
    for r in (4, 5, 6, 7, 8):
        assert out["K"][r] == 0, r
    K_in = int(np.floor(1.0 / s - 0.5)) + 1                 # samples with (k + 1/2) s <= 1
    np.testing.assert_allclose(out["opacity"][2], 1 - np.exp(-sigma * s * K_in), rtol=1e-6)
    K_plane = int(np.floor(4.0 / s - 0.5)) - int(np.ceil(2.0 / s - 0.5)) + 1    # x = -3 + (k + 1/2) s in [-1, 1]
    np.testing.assert_allclose(out["opacity"][3], 1 - np.exp(-sigma * s * K_plane), rtol=1e-6)


@pytest.mark.parametrize("eps", [1e-3, 0.05, 0.5, 1.0])
def test_early_stop_bound(eps):
    rng = np.random.default_rng(5)
    N = 17
    g = rng.uniform(0, 1, (N, N, N, 4)).astype(np.float32)
    g[..., 3] = rng.uniform(-5, 40, (N, N, N))
    o = rng.uniform(-3, 3, (300, 3))
    tgt = rng.uniform(-0.7, 0.7, (300, 3))
    d = (tgt - o) / np.linalg.norm(tgt - o, axis=1, keepdims=True)
    rays = np.concatenate([o, d, np.full((300, 1), 0.5), np.full((300, 1), 8.0)], 1).astype(np.float32)
    for wb in (False, True):
        full = br.render(g, BOX, rays, white_back=wb)
        cut = br.render(g, BOX, rays, white_back=wb, early_stop=eps)
        c = cut["cut"]
        assert c.any()
        for k in ("rgb", "depth", "opacity"):
            np.testing.assert_array_equal(cut[k][~c], full[k][~c])
        T = cut["T_cut"][c]
        assert (np.abs(cut["rgb"][c] - full["rgb"][c]).max(1) <= T + 1e-12).all()
        assert (np.abs(cut["opacity"][c] - full["opacity"][c]) <= T + 1e-12).all()
        assert (np.abs(cut["depth"][c] - full["depth"][c]) <= T * full["t_max"][c] + 1e-12).all()
        assert (T < eps).all()
