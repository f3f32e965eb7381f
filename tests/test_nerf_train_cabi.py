"""CPU-side checks of the NeRF.forward training entry points (include/nerf_pl_b200.h, "training a direct
NeRF.forward call"): argument validation without a GPU, workspace size, and the Python switch's default."""
import ctypes

import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib

FAKE = 1 << 30          # a non-NULL, 1024-byte aligned address that is never dereferenced: validation fails first


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


def test_workspace_bytes(lib):
    """bytes(n <= 0) == 0; monotone in n at about the render path's ~9 KiB per sample plus the 128-byte fp16
    direction row the forward fed the tensor core."""
    assert lib.nerfb200_nerf_train_workspace_bytes(0) == 0
    assert lib.nerfb200_nerf_train_workspace_bytes(-5) == 0
    b = [lib.nerfb200_nerf_train_workspace_bytes(n) for n in (1, 128, 129, 196608, 2 * 196608)]
    assert 0 < b[0] == b[1] < b[2] < b[3] < b[4]
    per = (b[4] - b[3]) / 196608
    r1, r2 = (lib.nerfb200_train_workspace_bytes(n, 64, 64) for n in (1024, 2048))
    per_render = (r2 - r1) / (1024 * 192)          # 64 coarse + 128 fine samples per ray
    assert 8000 < per < 11000
    assert 100 < per - per_render < 160, (per, per_render)


def test_argument_validation_without_gpu(lib):
    p24 = (ctypes.c_void_p * 24)(*([FAKE] * 24))
    # init: empty is a no-op, NULL / too small is EINVAL
    assert lib.nerfb200_nerf_train_workspace_init(None, 0, 0, None) == 0
    assert lib.nerfb200_nerf_train_workspace_init(None, 1 << 30, 64, None) == -1
    assert lib.nerfb200_nerf_train_workspace_init(FAKE, 16, 64, None) == -1
    assert b"too small" in lib.nerfb200_last_error()
    need = lib.nerfb200_nerf_train_workspace_bytes(4099)
    assert lib.nerfb200_nerf_train_workspace_init(FAKE, need - 1, 4099, None) == -1
    assert lib.nerfb200_nerf_train_workspace_init(FAKE + 512, need, 4099, None) == -1      # alignment
    # forward
    assert lib.nerfb200_nerf_forward_train(None, 0, 90, None, None, None, None) == 0
    assert lib.nerfb200_nerf_forward_train(None, 4, 90, FAKE, FAKE, FAKE, None) == -1
    assert lib.nerfb200_nerf_forward_train(FAKE, 4, 90, FAKE, None, FAKE, None) == -1
    assert lib.nerfb200_nerf_forward_train(FAKE, 4, 63, FAKE, FAKE, FAKE, None) == -1      # x_stride < 90
    assert lib.nerfb200_nerf_forward_train(FAKE, -1, 90, FAKE, FAKE, FAKE, None) == -1
    # backward
    assert lib.nerfb200_nerf_backward(None, 0, None, None, None, None, None) == 0
    assert lib.nerfb200_nerf_backward(None, 4, FAKE, p24, FAKE, p24, None) == -1
    assert lib.nerfb200_nerf_backward(FAKE, 4, FAKE, None, FAKE, p24, None) == -1
    holes = (ctypes.c_void_p * 24)(*([FAKE] * 23 + [None]))
    assert lib.nerfb200_nerf_backward(FAKE, 4, FAKE, p24, FAKE, holes, None) == -1
    assert b"NULL" in lib.nerfb200_last_error()
    assert lib.nerfb200_nerf_backward(FAKE + 4, 4, FAKE, p24, FAKE, p24, None) == -1      # g_out alignment


def test_autograd_impl_defaults_to_torch_and_cpu_raises():
    m = nb.NeRF()
    assert m.autograd_impl == "torch"
    assert "autograd_impl" not in m.state_dict()
    with pytest.raises(RuntimeError):
        m(torch.zeros(2, 90))
    m.autograd_impl = "fused"
    with pytest.raises(RuntimeError):
        m(torch.zeros(2, 90))
    with pytest.raises(RuntimeError):
        nb.nerf_forward_train(m, torch.zeros(2, 90))
