"""render_rays(..., occupancy=) without a device: the float64 general seed of the sparse compositing backward
(tests/train_skip_seed_ref.py) against the MSE-only restatement and finite differences, the C argument checks of
the structs' appended fields, and the Python errors raised before any device is touched."""
import ctypes

import numpy as np
import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib
from tests import train_skip_ref as tr
from tests import train_skip_seed_ref as seed_ref


def _pass(seed, R=5, S=16):
    rng = np.random.default_rng(seed)
    z = np.sort(rng.uniform(2.0, 6.0, (R, S)), 1)
    sigma = rng.uniform(0.5, 4.0, (R, S)) * rng.choice([-1.0, 1.0], (R, S), p=[0.2, 0.8])
    pre = rng.normal(0.0, 1.0, (R, S, 3))
    ev = rng.random((R, S)) < 0.6
    rays = np.concatenate([rng.normal(0, 1, (R, 3)), rng.normal(0, 1, (R, 3)), np.full((R, 2), 1.0)], 1)
    noise = rng.normal(0.0, 0.05, (R, S))
    return z, sigma, pre, ev, rays, noise


def _sig(x):
    return 1.0 / (1.0 + np.exp(-x))


@pytest.mark.parametrize("white_back", [False, True])
def test_seed_reduces_to_the_mse_backward(white_back):
    z, sigma, pre, ev, rays, noise = _pass(1)
    rng = np.random.default_rng(2)
    rgb_out, target = rng.random((5, 3)), rng.random((5, 3))
    want = tr.backward(z, sigma, _sig(pre), ev, rays[:, 3:6], noise, 1.0, white_back, rgb_out, target, 5)
    got = seed_ref.backward(z, sigma, _sig(pre), ev, rays[:, 3:6], noise, 1.0, white_back,
                            mse=(rgb_out, target, 5, 1.0))
    for a, b in zip(got, want):
        assert np.array_equal(a, b)


def _loss(z, sigma, pre, ev, rays, noise, white_back, gr, gd, go, mse):
    samples = np.concatenate([_sig(pre), sigma[..., None]], -1)
    f = tr.forward(z, samples, ev, rays, noise, 1.0, white_back)
    L = (gr * f["rgb"]).sum() + (gd * f["depth"]).sum() + (go * f["opacity"]).sum()
    if mse is not None:
        target, n_rays, lg = mse
        L += lg * ((f["rgb"] - target) ** 2).sum() / (3.0 * n_rays)
    return L, f


@pytest.mark.parametrize("white_back", [False, True])
@pytest.mark.parametrize("with_mse", [False, True])
def test_seed_matches_finite_differences(white_back, with_mse):
    """Central differences of train_skip_ref.forward (float64, noise, white_back) of L = <g_rgb, rgb> + <g_depth,
    depth> + <g_opacity, opacity> [+ loss_grad * MSE]: d L / d sigma and d L / d rgb_pre at the evaluated samples."""
    z, sigma, pre, ev, rays, noise = _pass(3)
    rng = np.random.default_rng(4)
    gr, gd, go = rng.normal(0, 1, (5, 3)), rng.normal(0, 0.3, 5), rng.normal(0, 1, 5)
    mse = (rng.random((5, 3)), 5, 0.7) if with_mse else None
    L0, f = _loss(z, sigma, pre, ev, rays, noise, white_back, gr, gd, go, mse)
    ds, dp = seed_ref.backward(z, sigma, _sig(pre), ev, rays[:, 3:6], noise, 1.0, white_back, gr, gd, go,
                               None if mse is None else (f["rgb"], mse[0], mse[1], mse[2]))
    h = 1e-6

    def L(sig, pr):
        return _loss(z, sig, pr, ev, rays, noise, white_back, gr, gd, go, mse)[0]

    fd_s, fd_p = np.zeros_like(ds), np.zeros_like(dp)
    for r, i in zip(*np.nonzero(ev)):
        d = np.zeros_like(sigma)
        d[r, i] = h
        fd_s[r, i] = (L(sigma + d, pre) - L(sigma - d, pre)) / (2 * h)
        for ch in range(3):
            d = np.zeros_like(pre)
            d[r, i, ch] = h
            fd_p[r, i, ch] = (L(sigma, pre + d) - L(sigma, pre - d)) / (2 * h)
    assert not ds[~ev].any() and not dp[~ev].any()
    assert np.abs(ds - fd_s).max() <= 1e-6 * max(1.0, np.abs(fd_s).max())
    assert np.abs(dp - fd_p).max() <= 1e-6 * max(1.0, np.abs(fd_p).max())
    assert np.abs(ds).max() > 1e-3 and np.abs(dp).max() > 1e-3
    # dropping any one term of the seed is visible
    for kw in (dict(g_depth=None), dict(g_opacity=None), dict(g_rgb=None)):
        args = {**dict(g_rgb=gr, g_depth=gd, g_opacity=go), **kw}
        bds, bdp = seed_ref.backward(z, sigma, _sig(pre), ev, rays[:, 3:6], noise, 1.0, white_back, **args,
                                     mse=None if mse is None else (f["rgb"], mse[0], mse[1], mse[2]))
        assert np.abs(bds - fd_s).max() + np.abs(bdp - fd_p).max() > 1e-4, kw


# ---- the C ABI -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


def _train_args(**kw):
    a = dict(rays=256, n_rays=4, packed_coarse=256, packed_fine=256, n_samples=64, n_importance=64, bits=256, N=9,
             ranges=(ctypes.c_double * 6)(-1, 1, -1, 1, -1, 1), target=256, loss_out=256, rgb_coarse=256,
             depth_coarse=256, opacity_coarse=256, rgb_fine=256, depth_fine=256, opacity_fine=256)
    a.update(kw)
    return _lib.TrainSamplesArgs(**a)


def test_train_args_without_a_loss_pass_validation(lib):
    """target and loss_out both null (upstream gradients only) get past every argument check to the workspace size;
    exactly one of them null is still a NULL argument, with or without the upstream gradients."""
    live = (ctypes.c_int64 * 2)()
    grads = dict(g_rgb_coarse=256, g_depth_coarse=256, g_opacity_coarse=256, g_rgb_fine=256, g_depth_fine=256,
                 g_opacity_fine=256)
    for kw, msg in ((dict(target=None, loss_out=None), b"workspace smaller"),
                    (dict(target=None, loss_out=None, **grads), b"workspace smaller"),
                    (dict(target=None, **grads), b"NULL"), (dict(loss_out=None, **grads), b"NULL")):
        a = _train_args(**kw)
        rc = lib.nerfb200_train_samples_forward(ctypes.byref(a), ctypes.c_void_p(1024), 0, live, None)
        assert rc == -1 and msg in lib.nerfb200_last_error(), (kw, lib.nerfb200_last_error())
        rc = lib.nerfb200_train_samples_backward(ctypes.byref(a), ctypes.c_void_p(1024), 0, live, None, None, None,
                                                 None, None, None)
        assert rc == -1 and msg in lib.nerfb200_last_error(), (kw, lib.nerfb200_last_error())
        rc = lib.nerfb200_train_samples_backward_dev(ctypes.byref(a), ctypes.c_void_p(1024), 0, None, None, None,
                                                     None, None, None)
        assert rc == -1 and msg in lib.nerfb200_last_error(), (kw, lib.nerfb200_last_error())


def test_samples_args_randoms_checks(lib):
    out = ctypes.c_int64 * 2

    def call(**kw):
        a = dict(rays=256, n_rays=4, packed_coarse=256, packed_fine=256, n_samples=64, n_importance=64, bits=256, N=9,
                 ranges=(ctypes.c_double * 6)(-1, 1, -1, 1, -1, 1), opacity_coarse=256, rgb_fine=256, depth_fine=256,
                 opacity_fine=256, test_time=1)
        a.update(kw)
        return lib.nerfb200_render_samples(ctypes.byref(_lib.SamplesArgs(**a)), ctypes.c_void_p(256), 0, out(), None)

    for bad, msg in ((dict(rng_in_kernel=3), b"rng_in_kernel must be"), (dict(rng_in_kernel=-1), b"rng_in_kernel must be"),
                     (dict(rng_in_kernel=2), b"needs rng_seed"), (dict(perturb=-1.0), b"perturb / noise_std < 0"),
                     (dict(noise_std=float("nan")), b"perturb / noise_std < 0"),
                     (dict(perturb=1.0), b"perturb_rand"), (dict(perturb=1.0, perturb_rand=256), b"u_rand"),
                     (dict(noise_std=1.0), b"noise_coarse"), (dict(noise_std=1.0, noise_coarse=256), b"noise_fine"),
                     (dict(rng_ray_offset=-1), b"rng_ray_offset"), (dict(rng_ray_offset=(1 << 32) - 3), b"rng_ray_offset"),
                     (dict(rng_ray_offset=1 << 62), b"rng_ray_offset")):
        rc = call(**bad)
        assert rc == -1 and msg in lib.nerfb200_last_error(), (bad, rc, lib.nerfb200_last_error())
    # well-formed randoms reach the workspace check
    for ok in (dict(perturb=1.0, perturb_rand=256, u_rand=256, noise_std=1.0, noise_coarse=256, noise_fine=256),
               dict(perturb=1.0, rng_in_kernel=1, rng_seed=5, rng_ray_offset=(1 << 32) - 4),
               dict(perturb=1.0, rng_in_kernel=2, rng_seed=256), dict(perturb=1.0, n_importance=0, perturb_rand=256)):
        rc = call(**ok)
        assert rc == -1 and b"workspace smaller" in lib.nerfb200_last_error(), (ok, lib.nerfb200_last_error())
    assert call(n_rays=0, rays=None, perturb=1.0) == 0       # nothing to do


# ---- Python -----------------------------------------------------------------------------------------------------
def test_python_errors_before_any_device():
    """render_rays(..., occupancy=) refuses what it cannot do before it touches a device (CPU rays and models)."""
    models = [nb.NeRF(), nb.NeRF()]
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    rays = torch.zeros(16, 8)
    grid = object.__new__(nb.OccupancyGrid)
    grid.bits = torch.zeros(1, dtype=torch.int32)
    with pytest.raises(ValueError, match="OccupancyGrid"):
        nb.render_rays(models, emb, rays, 64, N_importance=64, occupancy=object())
    for kw in (dict(test_time=True), dict(extras=True), dict(autograd_impl="torch")):
        with pytest.raises(ValueError, match="gradient graph needs"):
            nb.render_rays(models, emb, rays, 64, N_importance=64, occupancy=grid, **kw)
    for S, K, n in ((48, 64, 16), (64, 16, 16), (64, 160, 16), (64, 64, (1 << 22) + 1)):
        with pytest.raises(ValueError, match="N_samples"):
            nb.render_rays(models, emb, torch.zeros(n, 8, device="meta"), S, N_importance=K, occupancy=grid)
    # the graph path's options are the graph path's: without a graph the call goes on to the device check
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="CUDA"):
            nb.render_rays(models, emb, rays, 64, N_importance=64, occupancy=grid, test_time=True, extras=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        nb.render_rays(models, emb, rays, 64, N_importance=64, occupancy=grid)
