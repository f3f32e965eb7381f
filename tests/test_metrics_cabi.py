"""CPU-side checks of the image-metric entries: workspace sizes, the argument checks that need no GPU and the Python
surface."""
import ctypes
import inspect

import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


def test_workspace_sizes(lib):
    ws = lib.nerfb200_ssim_workspace_bytes
    # one double per 256-pixel tile, rounded up to 256 bytes
    assert ws(1, 3, 800, 800) == ((3 * 800 * 800 + 255) // 256 * 8 + 255) // 256 * 256
    assert ws(2, 5, 7, 9) == 256 and ws(1, 1, 1, 1) == 256
    for bad in ((0, 3, 8, 8), (1, 0, 8, 8), (1, 3, -1, 8), (1, 3, 8, 0), (1 << 20, 1 << 20, 1 << 20, 1)):
        assert ws(*bad) == 0
    dv = lib.nerfb200_visualize_depth_workspace_bytes
    assert dv(1, 1) == 256 and dv(800, 800) == 256 * ((8 * 296 + 255) // 256)
    assert dv(0, 5) == 0 and dv(5, -1) == 0


def test_ssim_argument_checks(lib):
    one = ctypes.c_void_p(256)       # never dereferenced: every call below fails first
    st = (ctypes.c_int64 * 4)(192, 64, 8, 1)
    f = lib.nerfb200_ssim
    big = 1 << 20
    assert f(one, st, one, st, 0, 3, 8, 8, 0, one, big, one, None) == -1
    assert b"must be >= 1" in lib.nerfb200_last_error()
    assert f(one, st, one, st, 1, 3, 8, 8, 3, one, big, one, None) == -1
    assert b"reduction" in lib.nerfb200_last_error()
    for args in ((None, st, one, st), (one, None, one, st), (one, st, None, st), (one, st, one, None)):
        assert f(*args, 1, 3, 8, 8, 0, one, big, one, None) == -1
        assert b"NULL" in lib.nerfb200_last_error()
    assert f(one, st, one, st, 1, 3, 8, 8, 2, None, 0, None, None) == -1
    neg = (ctypes.c_int64 * 4)(192, 64, -8, 1)
    assert f(one, neg, one, st, 1, 3, 8, 8, 2, None, 0, one, None) == -1
    assert b"negative stride" in lib.nerfb200_last_error()
    assert f(one, st, one, st, 1, 3, 8, 8, 0, None, big, one, None) == -1
    assert b"NULL workspace" in lib.nerfb200_last_error()
    assert f(one, st, one, st, 1, 3, 8, 8, 1, one, lib.nerfb200_ssim_workspace_bytes(1, 3, 8, 8) - 1, one, None) == -1
    assert b"workspace smaller" in lib.nerfb200_last_error()


def test_visualize_depth_argument_checks(lib):
    one = ctypes.c_void_p(256)
    f = lib.nerfb200_visualize_depth
    assert f(one, 0, 4, 4, 1, one, 1 << 20, one, None) == -1
    assert b"must be >= 1" in lib.nerfb200_last_error()
    assert f(one, 4, 4, -4, 1, one, 1 << 20, one, None) == -1
    assert b"negative stride" in lib.nerfb200_last_error()
    for args in ((None, one, one), (one, None, one), (one, one, None)):
        assert f(args[0], 4, 4, 4, 1, args[1], 1 << 20, args[2], None) == -1
        assert b"NULL" in lib.nerfb200_last_error()
    assert f(one, 4, 4, 4, 1, one, lib.nerfb200_visualize_depth_workspace_bytes(4, 4) - 1, one, None) == -1
    assert b"workspace smaller" in lib.nerfb200_last_error()


def test_python_surface():
    for name in ("ssim", "visualize_depth"):
        assert name in nb.__all__ and hasattr(nb, name)
    assert list(inspect.signature(nb.ssim).parameters) == ["image_pred", "image_gt", "reduction"]    # metrics.py:15
    assert inspect.signature(nb.ssim).parameters["reduction"].default == "mean"
    p = inspect.signature(nb.visualize_depth).parameters
    assert list(p) == ["depth", "cmap"] and p["cmap"].default == 2                     # cv2.COLORMAP_JET
    x = torch.zeros(1, 3, 4, 4)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        nb.ssim(x, x)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        nb.visualize_depth(torch.zeros(4, 4))
    with pytest.raises(ValueError, match="reduction"):
        nb.ssim(x, x, "max")
    with pytest.raises(ValueError, match="COLORMAP_JET"):
        nb.visualize_depth(torch.zeros(4, 4), cmap=11)
