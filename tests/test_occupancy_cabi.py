"""CPU-side checks of the empty-space skipping entries: workspace sizes, the argument checks that need no GPU and the
Python surface (their prototypes are checked with the rest of include/nerf_pl_b200.h in test_cabi.py)."""
import ctypes
import inspect

import pytest

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


def test_occupancy_pack_argument_checks(lib):
    ws = lib.nerfb200_occupancy_workspace_bytes
    assert ws(1) == 0 and ws(0) == 0 and ws(-5) == 0 and ws(1626) == 0
    assert ws(2) >= 2 and ws(65) >= 2 * 64 ** 3 and ws(1625) >= 2 * 1624 ** 3
    one = ctypes.c_void_p(256)      # a non-NULL address that is never dereferenced: every call below fails first
    pack = lib.nerfb200_occupancy_pack
    assert pack(one, 1, 1.0, 0, one, 1 << 30, one, None) == -1
    assert b"N must be in [2, 1625]" in lib.nerfb200_last_error()
    assert pack(one, 1626, 1.0, 0, one, 1 << 40, one, None) == -1
    assert pack(one, 8, 1.0, -1, one, 1 << 30, one, None) == -1
    assert b"dilate" in lib.nerfb200_last_error()
    assert pack(one, 8, float("nan"), 1, one, 1 << 30, one, None) == -1
    assert b"NaN" in lib.nerfb200_last_error()
    for args in ((None, 8, 1.0, 1, one, 1 << 30, one), (one, 8, 1.0, 1, None, 1 << 30, one),
                 (one, 8, 1.0, 1, one, 1 << 30, None)):
        assert pack(*args, None) == -1
        assert b"NULL" in lib.nerfb200_last_error()
    assert pack(one, 8, 1.0, 1, one, ws(8) - 1, one, None) == -1
    assert b"workspace smaller" in lib.nerfb200_last_error()
    pop = lib.nerfb200_occupancy_popcount
    assert pop(None, 8, one, None) == -1 and pop(one, 8, None, None) == -1 and pop(one, 1, one, None) == -1


def test_cull_argument_checks(lib):
    ws = lib.nerfb200_cull_workspace_bytes
    assert ws(-1) == 0
    assert ws(0) > 0 and ws(1) > 0
    assert ws(160000) >= (160000 // 256) * 12 and ws(1 << 24) > ws(160000)
    one = ctypes.c_void_p(256)
    box = (ctypes.c_double * 6)(-1, 1, -1, 1, -1, 1)
    n_live = ctypes.c_int64(77)
    count = lib.nerfb200_cull_count
    # no rays: nothing to do, whatever the pointers
    assert count(None, 0, None, 8, box, None, 0, None, ctypes.byref(n_live), None) == 0 and n_live.value == 0
    assert lib.nerfb200_cull_emit(None, 0, None, None, 0, None, None, None) == 0
    assert count(one, -1, one, 8, box, one, 1 << 20, one, ctypes.byref(n_live), None) == -1
    assert b"n_rays < 0" in lib.nerfb200_last_error()
    assert count(None, 5, one, 8, box, one, 1 << 20, one, ctypes.byref(n_live), None) == -1
    assert b"NULL" in lib.nerfb200_last_error()
    assert count(one, 5, None, 8, box, one, 1 << 20, one, ctypes.byref(n_live), None) == -1
    assert count(one, 5, one, 8, box, one, 1 << 20, None, ctypes.byref(n_live), None) == -1
    assert count(one, 5, one, 8, box, one, 1 << 20, one, None, None) == -1
    assert count(one, 5, one, 8, None, one, 1 << 20, one, ctypes.byref(n_live), None) == -1
    assert count(ctypes.c_void_p(260), 5, one, 8, box, one, 1 << 20, one, ctypes.byref(n_live), None) == -1
    assert b"16-byte aligned" in lib.nerfb200_last_error()
    assert count(one, 5, one, 1, box, one, 1 << 20, one, ctypes.byref(n_live), None) == -1
    assert count(one, 5, one, 1626, box, one, 1 << 20, one, ctypes.byref(n_live), None) == -1
    assert b"N must be in [2, 1625]" in lib.nerfb200_last_error()
    assert count(one, 5, one, 8, box, one, ws(5) - 1, one, ctypes.byref(n_live), None) == -1
    assert b"workspace smaller" in lib.nerfb200_last_error()
    flat = (ctypes.c_double * 6)(-1, 1, 2, 2, -1, 1)
    assert count(one, 5, one, 8, flat, one, 1 << 20, one, ctypes.byref(n_live), None) == -1
    assert b"min != max" in lib.nerfb200_last_error()
    emit = lib.nerfb200_cull_emit
    assert emit(one, 5, None, one, 1 << 20, one, one, None) == -1
    assert emit(one, 5, one, one, 1 << 20, None, one, None) == -1
    assert emit(one, 5, one, one, 1 << 20, one, None, None) == -1
    assert emit(one, 5, one, one, ws(5) - 1, one, one, None) == -1


def test_scatter_argument_checks(lib):
    one = ctypes.c_void_p(256)
    P6 = ctypes.c_void_p * 6
    full, none = P6(*[256] * 6), P6()
    scatter = lib.nerfb200_scatter_results
    assert scatter(none, none, None, 0, 0, 1, None) == 0                  # no rays
    assert scatter(full, full, one, 3, 2, 1, None) == -1                  # more live rays than rays
    assert b"n_live" in lib.nerfb200_last_error()
    assert scatter(full, full, one, -1, 2, 1, None) == -1
    assert scatter(None, full, one, 1, 2, 1, None) == -1
    assert scatter(full, full, None, 1, 2, 1, None) == -1
    assert b"live_idx" in lib.nerfb200_last_error()
    assert scatter(full, P6(256, 256, 256, None, 256, 256), one, 1, 2, 1, None) == -1
    assert b"one side only" in lib.nerfb200_last_error()
    assert scatter(none, none, one, 1, 2, 1, None) == -1
    assert b"no result" in lib.nerfb200_last_error()


def test_python_surface():
    for name in ("OccupancyGrid", "occupancy_grid", "pack_occupancy", "cull_rays", "scatter_results",
                 "render_rays_culled"):
        assert name in nb.__all__ and hasattr(nb, name)
    sig = inspect.signature(nb.occupancy_grid)
    assert list(sig.parameters) == ["model", "N", "x_range", "y_range", "z_range", "sigma_threshold", "dilate", "chunk"]
    assert sig.parameters["dilate"].default == 1 and sig.parameters["chunk"].default == 1 << 21
    sig = inspect.signature(nb.render_rays_culled)
    assert list(sig.parameters)[:9] == ["models", "embeddings", "rays", "occupancy", "N_samples", "use_disp",
                                        "N_importance", "white_back", "test_time"]
    assert sig.parameters["test_time"].default is True
    for fn in (nb.batched_inference, nb.render_image):
        p = inspect.signature(fn).parameters
        assert p["occupancy"].default is None and list(p)[-1] == "occupancy"
    # inference only, whatever the device
    with pytest.raises(ValueError, match="inference only"):
        nb.render_rays_culled([], [], None, None, perturb=1.0)
    with pytest.raises(ValueError, match="inference only"):
        nb.render_rays_culled([], [], None, None, noise_std=1.0)
    with pytest.raises(ValueError, match="OccupancyGrid"):
        nb.render_rays_culled([], [], None, "grid")
