"""The byte sizes of both training workspaces, pinned at a spread of shapes (no GPU needed).

One layout builder serves the render path and the direct NeRF.forward path; a buffer taken in another order, or
one path given the other's per-ray buffers, changes these sizes.  The wgrad plan sizes its partial-sum slots by the
SM count, so the values hold for the 148-SM plan the library uses when no device is visible."""
import pytest

from nerf_pl_b200 import _lib

RENDER = {
    (1, 32, 0): 8550400, (1, 64, 0): 8550400, (1, 64, 64): 14984192, (1, 128, 64): 21412864,
    (1, 64, 128): 21412864,
    (127, 32, 0): 78739456, (127, 64, 0): 116111360, (127, 64, 64): 264599552, (127, 128, 64): 412921856,
    (127, 64, 128): 339343360,
    (1024, 32, 0): 342521856, (1024, 64, 0): 641497088, (1024, 64, 64): 1838725120, (1024, 128, 64): 3034626048,
    (1024, 64, 128): 2436675584,
    (4096, 32, 0): 1246918656, (4096, 64, 0): 2442819584, (4096, 64, 64): 7231731712,
    (4096, 128, 64): 12015335424, (4096, 64, 128): 9623533568,
    (65536, 32, 0): 19334854656, (65536, 64, 0): 38469269504, (65536, 64, 64): 115091863552,
    (65536, 128, 64): 191629522944, (65536, 64, 128): 153360693248,
}
NERF = {1: 7176192, 128: 7176192, 129: 14147584, 196608: 1860153344, 10 ** 6: 9301867520}


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    lib = _lib.load()
    if lib.nerfb200_sm_count() != 0:
        pytest.skip("the sizes depend on the visible device's SM count")
    return lib


@pytest.mark.parametrize("shape", sorted(RENDER))
def test_render_train_workspace_bytes(lib, shape):
    assert lib.nerfb200_train_workspace_bytes(*shape) == RENDER[shape]


@pytest.mark.parametrize("n", sorted(NERF))
def test_nerf_train_workspace_bytes(lib, n):
    assert lib.nerfb200_nerf_train_workspace_bytes(n) == NERF[n]
