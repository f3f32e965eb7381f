"""The view-dependent bake's definition (tests/baked_sh_ref.py, DESIGN.md §10k) on the CPU: the fit inverts the basis,
the library's direction table and P are the restatement's bit for bit, and the restated render meets closed forms."""
import ctypes

import numpy as np
import pytest

from nerf_pl_b200 import _lib
from tests import baked_ref as br
from tests import baked_sh_ref as sr

BOX = (-1.0, 1.0, -1.0, 1.0, -1.0, 1.0)


def test_projection_inverts_the_basis():
    Y, P = sr.basis_matrix(), sr.projection()
    assert np.abs(P @ Y - np.eye(9)).max() < 1e-12
    assert np.linalg.cond(Y) < 1.05
    assert 3.5 < np.abs(P).sum(1).max() < 3.6                      # ||P||, the factor of the query's error bar
    d = sr.directions().astype(np.float64)
    assert np.abs(np.linalg.norm(d, axis=1) - 1).max() < 1e-7
    # a colour that does not depend on the direction is all coefficient 0
    f = np.array([0.2, 0.5, 0.9])
    coef = P @ np.broadcast_to(f, (64, 3))
    assert np.abs(coef[0] - f / sr.C0).max() < 1e-12 and np.abs(coef[1:]).max() < 1e-12


def test_fit_host_is_the_restatement_bit_for_bit():
    _lib.build()
    lib = _lib.load()
    dirs, proj = (ctypes.c_float * 192)(), (ctypes.c_float * 576)()
    assert lib.nerfb200_sh_fit_host(dirs, proj) == 0
    got_d = np.frombuffer(dirs, np.float32).reshape(64, 3)
    got_p = np.frombuffer(proj, np.float32).reshape(9, 64)
    assert np.array_equal(got_d.view(np.uint32), sr.directions().view(np.uint32))
    assert np.array_equal(got_p.view(np.uint32), sr.projection().astype(np.float32).view(np.uint32))
    assert lib.nerfb200_sh_fit_host(None, proj) == -1 and lib.nerfb200_sh_fit_host(dirs, None) == -1


def test_slots():
    s = sr.coefficient_slots()
    assert sorted(s.ravel().tolist()) == [i for i in range(28) if i != 3]
    assert s[0].tolist() == [0, 1, 2] and s[1].tolist() == [4, 5, 6] and s[8].tolist() == [25, 26, 27]


def _rays(n, seed):
    rng = np.random.default_rng(seed)
    o = rng.uniform(-2.5, 2.5, (n, 3))
    tgt = rng.uniform(-0.7, 0.7, (n, 3))
    d = (tgt - o) * rng.uniform(0.3, 2.0, (n, 1))
    return np.concatenate([o, d, np.zeros((n, 1)), np.full((n, 1), 6.0)], 1).astype(np.float32)


def _sh_grid(N, seed, c0_only=False):
    rng = np.random.default_rng(seed)
    g = np.zeros((N, N, N, 28))
    coef = rng.uniform(-0.3, 0.3, (N ** 3, 9, 3))
    coef[:, 0] = rng.uniform(0, 1, (N ** 3, 3)) / sr.C0
    if c0_only:
        coef[:, 1:] = 0
    g.reshape(-1, 28)[:] = sr.pack_points(coef, rng.uniform(-3, 12, N ** 3))
    return g


@pytest.mark.parametrize("wb", [False, True])
def test_c0_only_renders_the_direction_free_volume(wb):
    g = _sh_grid(9, 1, c0_only=True)
    dense4 = np.concatenate([g[..., 0:3] * sr.C0, g[..., 3:4]], -1)
    rays = _rays(400, 2)
    a = sr.render(g, BOX, rays, white_back=wb)
    b = br.render(dense4, BOX, rays, white_back=wb)
    for k in ("rgb", "depth", "opacity"):
        assert np.abs(a[k] - b[k]).max() < 1e-12, k
    assert b["opacity"].max() > 0.5


@pytest.mark.parametrize("axis", range(3))
@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_degree_one_field_on_axis_aligned_rays(axis, sign):
    # constant sigma and coefficients: colour = clamp(a C0 + b Y_m(d)), Y_1 = -C1 y, Y_2 = C1 z, Y_3 = -C1 x
    N = 5
    g = np.zeros((N, N, N, 28))
    a, b = np.array([0.4, 0.5, 0.6]), np.array([0.3, -0.2, 0.1])
    m = {0: 3, 1: 1, 2: 2}[axis]
    g[..., 0:3] = a / sr.C0
    g[..., [sr.slot_of(m, c) for c in range(3)]] = b
    g[..., 3] = 2.0
    d = np.zeros(3)
    d[axis] = sign * 0.7
    o = np.array([0.1, -0.2, 0.15])
    o[axis] = -sign * 1.5
    rays = np.array([[*o, *d, 0.0, 6.0]], np.float32)
    r = sr.render(g, BOX, rays)
    y = {0: -sr.C1 * sign, 1: -sr.C1 * sign, 2: sr.C1 * sign}[axis]
    want = np.clip(a + b * y, 0, 1) * r["opacity"][0]
    assert r["opacity"][0] > 0.9
    assert np.abs(r["rgb"][0] - want).max() < 1e-12


def test_clamping_at_zero_and_one():
    N = 5
    g = np.zeros((N, N, N, 28))
    g[..., 0] = 3.0 / sr.C0            # red far above 1
    g[..., 1] = -2.0 / sr.C0           # green far below 0
    g[..., 2] = 0.5 / sr.C0
    g[..., 3] = 1.5
    rays = _rays(200, 5)
    r = sr.render(g, BOX, rays, white_back=True)
    op = r["opacity"]
    assert np.abs(r["rgb"][:, 0] - 1.0).max() < 1e-12                 # op * 1 + (1 - op)
    assert np.abs(r["rgb"][:, 1] - (1 - op)).max() < 1e-12
    assert np.abs(r["rgb"][:, 2] - (0.5 * op + 1 - op)).max() < 1e-12
    assert op.max() > 0.5


@pytest.mark.parametrize("eps", [1e-3, 0.1, 0.6])
def test_early_stop_bound(eps):
    g = _sh_grid(9, 7)
    hi = 8.0 if eps < 0.01 else 3.0                 # dense enough that some rays are cut, thin enough that some are not
    g[..., 3] = np.random.default_rng(9).uniform(-2, hi, g.shape[:3])
    rays = _rays(500, 8)
    full = sr.render(g, BOX, rays)
    cut = sr.render(g, BOX, rays, early_stop=eps)
    c = cut["cut"]
    assert c.any() and (~c).any()
    for k in ("rgb", "depth", "opacity"):
        assert np.array_equal(full[k][~c], cut[k][~c]), k
    T = cut["T_cut"][c]
    assert (T < eps).all()
    assert (np.abs(cut["rgb"] - full["rgb"]).max(1)[c] <= T + 1e-12).all()
    assert (np.abs(cut["opacity"] - full["opacity"])[c] <= T + 1e-12).all()
    assert (np.abs(cut["depth"] - full["depth"])[c] <= T * cut["t_max"][c] + 1e-12).all()
