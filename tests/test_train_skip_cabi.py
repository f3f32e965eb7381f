"""The C ABI of the training step with empty samples skipped: the workspace query, and the argument errors the entries
and render_rays_loss(..., occupancy=) raise before any launch."""
import ctypes

import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


def test_workspace_bytes_and_shape_checks(lib):
    f = lib.nerfb200_train_samples_workspace_bytes
    assert f(1024, 64, 128) > f(1024, 64, 64) > f(512, 64, 64) > f(512, 64, 0) > 0
    for bad in ((0, 64, 64), (-1, 64, 64), (16, 48, 64), (16, 64, 48), (16, 128, 96), (16, 64, -32),
                ((1 << 22) + 1, 64, 64)):
        assert f(*bad) == 0, bad


def _args(**kw):
    a = dict(rays=256, n_rays=4, packed_coarse=256, packed_fine=256, n_samples=64, n_importance=64, bits=256, N=9,
             ranges=(ctypes.c_double * 6)(-1, 1, -1, 1, -1, 1), target=256, loss_out=256, rgb_coarse=256,
             depth_coarse=256, opacity_coarse=256, rgb_fine=256, depth_fine=256, opacity_fine=256)
    a.update(kw)
    return _lib.TrainSamplesArgs(**a)


BAD = ((dict(n_samples=48), b"N_samples"), (dict(n_importance=16), b"N_samples"), (dict(n_rays=0), b"n_rays"),
       (dict(n_rays=(1 << 22) + 1), b"n_rays"), (dict(N=1), b"N must be"),
       (dict(ranges=(ctypes.c_double * 6)(1, 1, -1, 1, -1, 1)), b"range"), (dict(bits=None), b"NULL"),
       (dict(target=None), b"NULL"), (dict(loss_out=None), b"NULL"), (dict(rgb_fine=None), b"fine"),
       (dict(perturb=1.0), b"perturb_rand"), (dict(perturb=1.0, perturb_rand=256), b"u_rand"),
       (dict(noise_std=1.0, noise_coarse=256), b"noise_fine"), (dict(perturb=-1.0), b"perturb"),
       (dict(rng_in_kernel=2), b"rng_seed"), (dict(rng_in_kernel=3), b"rng_in_kernel"),
       (dict(rays=264), b"aligned"), (dict(), b"workspace smaller"))


def test_forward_and_backward_argument_checks(lib):
    """Every malformed argument is refused by the host code; nothing here reaches a kernel (no device needed for the
    shape checks, and the device checks come after them)."""
    live = (ctypes.c_int64 * 2)()
    for bad, msg in BAD:
        a = _args(**bad)
        rc = lib.nerfb200_train_samples_forward(ctypes.byref(a), ctypes.c_void_p(1024), 0, live, None)
        assert rc in (-1, -2) and msg in lib.nerfb200_last_error(), (bad, rc, lib.nerfb200_last_error())
        rc = lib.nerfb200_train_samples_backward(ctypes.byref(a), ctypes.c_void_p(1024), 0, live, None, None, None,
                                                 None, None, None)
        assert rc in (-1, -2) and msg in lib.nerfb200_last_error(), (bad, rc, lib.nerfb200_last_error())
    assert lib.nerfb200_train_samples_forward(ctypes.byref(_args()), ctypes.c_void_p(1024), 0, None, None) == -1


def test_python_argument_errors():
    """render_rays_loss(..., occupancy=) checks what it can before touching a device."""
    rays = torch.zeros(4, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        nb.render_rays_loss([], [nb.Embedding(3, 10), nb.Embedding(3, 4)], rays, torch.zeros(4, 3),
                            occupancy=object())
    from nerf_pl_b200 import train_skip
    for n, S, K in ((4, 48, 64), (4, 64, 16), (4, 64, 160), (0, 64, 64), ((1 << 22) + 1, 64, 64)):
        with pytest.raises(ValueError, match="N_samples"):
            train_skip.check_shape(n, S, K)
    train_skip.check_shape(4, 32, 160)
    with pytest.raises(ValueError, match="OccupancyGrid"):
        train_skip.check_grid(object(), rays)
    grid = object.__new__(nb.OccupancyGrid)
    grid.bits = torch.zeros(1, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="occupancy grid is on"):
        train_skip.check_grid(grid, torch.zeros(4, 8, device="meta"))
