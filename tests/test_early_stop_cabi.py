"""Early ray termination without a device: the argument checks of nerfb200_samples_args' early_stop / cut_coarse,
the workspace it needs (no more than a coarse-only render's), and the Python errors raised before any device work."""
import ctypes
import math

import numpy as np
import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib, culling, inference, mesh


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


def _call(lib, ws_bytes=0, **kw):
    a = dict(rays=256, n_rays=4, packed_coarse=256, n_samples=64, n_importance=0, bits=256, N=9,
             ranges=(ctypes.c_double * 6)(-1, 1, -1, 1, -1, 1), opacity_coarse=256, test_time=1)
    a.update(kw)
    out = (ctypes.c_int64 * 2)()
    return lib.nerfb200_render_samples(ctypes.byref(_lib.SamplesArgs(**a)), ctypes.c_void_p(256), ws_bytes, out, None)


@pytest.mark.parametrize("bad,code,msg", [
    (dict(early_stop=float("nan")), -1, b"early_stop must be in [0, 1]"),
    (dict(early_stop=-1e-3), -1, b"early_stop must be in [0, 1]"),
    (dict(early_stop=1.5), -1, b"early_stop must be in [0, 1]"),
    (dict(early_stop=float("inf")), -1, b"early_stop must be in [0, 1]"),
    (dict(early_stop=1e-3, n_importance=64, packed_fine=256, rgb_fine=256, depth_fine=256, opacity_fine=256), -2,
     b"z_vals_fine"),
    (dict(early_stop=1e-3, perturb=1.0, rng_in_kernel=1), -1, b"perturb = 0 and noise_std = 0"),
    (dict(early_stop=1e-3, noise_std=1.0, noise_coarse=256), -1, b"perturb = 0 and noise_std = 0"),
])
def test_argument_checks(lib, bad, code, msg):
    assert _call(lib, **bad) == code
    assert msg in lib.nerfb200_last_error(), lib.nerfb200_last_error()


def test_n_importance_message_gives_the_reason(lib):
    assert _call(lib, early_stop=0.5, n_importance=32, packed_fine=256, rgb_fine=256, depth_fine=256,
                 opacity_fine=256) == -2
    err = lib.nerfb200_last_error()
    assert b"N_importance = 0" in err and b"5 %" in err and b"10f" in err


def test_zero_fields_behave_as_before(lib):
    """The new fields zero: the checks the earlier struct met, in the same order."""
    assert _lib.SamplesArgs().early_stop == 0.0 and _lib.SamplesArgs().cut_coarse is None
    for kw, msg in ((dict(), b"workspace smaller"), (dict(bits=None), b"NULL"), (dict(rays=264), b"aligned"),
                    (dict(n_importance=64), b"fine")):
        assert _call(lib, early_stop=0.0, cut_coarse=None, **kw) == -1
        assert msg in lib.nerfb200_last_error(), (kw, lib.nerfb200_last_error())
    assert _call(lib, n_rays=0, rays=None) == 0


@pytest.mark.parametrize("S", [32, 64, 128])
@pytest.mark.parametrize("n", [1, 75, 4096])
def test_termination_needs_no_more_workspace(lib, S, n):
    need = lib.nerfb200_samples_workspace_bytes(n, S, 0)
    assert need > 0
    assert _call(lib, ws_bytes=need - 1, n_rays=n, n_samples=S, early_stop=1e-3, cut_coarse=256) == -1
    assert b"workspace smaller than nerfb200_samples_workspace_bytes" in lib.nerfb200_last_error()


def test_state_fits_the_unused_fine_part_of_the_carve():
    """T, the state and S/32 row bases per ray (8 + 4 + 8 S/32 bytes) fit in zf's 4 S bytes per ray."""
    for S in (64, 128):
        assert 8 + 4 + 8 * (S // 32) <= 4 * S


def _fail(*a, **k):
    raise AssertionError("device work before the argument checks")


_RENDER_SAMPLES = culling.render_samples      # the entry itself, before the fixture stubs out what it calls
BAD = [(dict(early_stop=float("nan")), "must be in"), (dict(early_stop=-0.1), "must be in"),
       (dict(early_stop=2.0), "must be in")]


@pytest.fixture
def no_device(monkeypatch):
    for mod, name in ((culling, "cull_rays"), (culling, "_check_rays"), (culling, "render_samples"),
                      (inference, "generate_rays"), (inference, "render_culled_samples"), (mesh, "_cuda"),
                      (mesh, "render_rays_culled"), (_lib, "call"), (_lib, "workspace")):
        monkeypatch.setattr(mod, name, _fail)


def test_render_rays_culled_errors(no_device):
    grid, rays = object.__new__(nb.OccupancyGrid), torch.zeros(4, 8)
    for kw, msg in BAD:
        with pytest.raises(ValueError, match=msg):
            nb.render_rays_culled([], [], rays, grid, 64, False, 0, skip="samples", **kw)
    with pytest.raises(ValueError, match="needs skip='samples'"):
        nb.render_rays_culled([], [], rays, grid, 64, False, 0, early_stop=1e-3)
    with pytest.raises(ValueError, match="N_importance = 0.*5 %.*z_vals_fine"):
        nb.render_rays_culled([], [], rays, grid, 64, False, 64, skip="samples", early_stop=1e-3)


def test_batched_inference_and_render_image_errors(no_device):
    grid, rays = object.__new__(nb.OccupancyGrid), torch.zeros(4, 8)
    for kw, msg in BAD:
        with pytest.raises(ValueError, match=msg):
            nb.batched_inference([], [], rays, 64, 0, False, occupancy=grid, skip="samples", **kw)
        with pytest.raises(ValueError, match=msg):
            nb.render_image([], [], 4, 4, 1.0, np.eye(3, 4), 2.0, 6.0, 64, 0, occupancy=grid, skip="samples", **kw)
    with pytest.raises(ValueError, match="needs skip='samples'"):
        nb.batched_inference([], [], rays, 64, 0, False, occupancy=grid, early_stop=1e-3)
    with pytest.raises(ValueError, match="needs skip='samples'"):
        nb.render_image([], [], 4, 4, 1.0, np.eye(3, 4), 2.0, 6.0, 64, 0, occupancy=grid, early_stop=1e-3)
    with pytest.raises(ValueError, match="N_importance = 0"):
        nb.batched_inference([], [], rays, 64, 128, False, occupancy=grid, skip="samples", early_stop=1e-3)
    with pytest.raises(ValueError, match="N_importance = 0"):
        nb.render_image([], [], 4, 4, 1.0, np.eye(3, 4), 2.0, 6.0, 64, 64, occupancy=grid, skip="samples",
                        early_stop=1e-3)


def test_render_samples_errors(no_device):
    grid, rays = object.__new__(nb.OccupancyGrid), torch.zeros(4, 8)
    for kw, msg in BAD:
        with pytest.raises(ValueError, match=msg):
            _RENDER_SAMPLES([], rays, grid, 64, False, 0, False, True, **kw)
        with pytest.raises(ValueError, match=msg):
            culling.render_culled_samples([], rays, grid, 64, False, 0, False, True, **kw)
    with pytest.raises(ValueError, match="N_importance = 0"):
        _RENDER_SAMPLES([], rays, grid, 64, False, 32, False, True, early_stop=0.5)
    with pytest.raises(ValueError, match="N_importance = 0"):
        culling.render_culled_samples([], rays, grid, 64, False, 32, False, True, early_stop=0.5)
    with pytest.raises(ValueError, match="perturb = 0 and noise_std = 0"):
        _RENDER_SAMPLES([], rays, grid, 64, False, 0, False, True, perturb=1.0, early_stop=0.5)
    with pytest.raises(ValueError, match="perturb = 0 and noise_std = 0"):
        _RENDER_SAMPLES([], rays, grid, 64, False, 0, False, True, noise_std=1.0, early_stop=0.5)


def test_fuse_vertex_colors_errors(no_device):
    v, imgs = torch.zeros(4, 3), torch.zeros(1, 4, 4, 3, dtype=torch.uint8)
    grid = object.__new__(nb.OccupancyGrid)
    with pytest.raises(ValueError, match=r"occupancy= for fuse_vertex_colors"):
        nb.fuse_vertex_colors(None, v, imgs, [np.eye(3, 4)], 1.0, 2.0, early_stop=1e-3)
    for kw, msg in BAD:
        with pytest.raises(ValueError, match=msg):
            nb.fuse_vertex_colors(None, v, imgs, [np.eye(3, 4)], 1.0, 2.0, occupancy=grid, **kw)


def test_accepted_values():
    f = culling.check_early_stop
    assert f(0, False, 128) == 0.0 and f(0.0, True, 64, 1.0, 1.0) == 0.0     # zero: no condition applies
    assert f(1, True, 0) == 1.0 and math.isclose(f(0.25, True, 0), 0.25)
