"""The byte sizes of every workspace the library lays out, pinned at a spread of shapes (no GPU needed).

One layout builder serves the render path and the direct NeRF.forward path; a buffer taken in another order, or
one path given the other's per-ray buffers, changes these sizes.  The wgrad plan sizes its partial-sum slots by the
SM count, so the values hold for the 148-SM plan the library uses when no device is visible.  The mesh, volume,
normals, occupancy and cull workspaces end with CUB's temporary storage, which CUB sizes as 0 bytes when no device is
visible: there these values pin the buffers the library carves and their 256-byte rounding.  0 bytes: an unsupported
shape."""
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
    # fine passes of 64, 96, 128, 160 samples from K = 32, 96, 160; the 128-sample coarse pass alone
    (1, 32, 32): 14984192, (1, 64, 32): 14984192, (1, 128, 32): 21412864, (1, 32, 96): 14984192,
    (1, 64, 96): 21412864, (1, 32, 160): 21412864, (1, 128, 0): 8550400,
    (127, 32, 32): 153649152, (127, 64, 32): 228392960, (127, 128, 32): 375549952, (127, 32, 96): 227227648,
    (127, 64, 96): 301971456, (127, 32, 160): 301971456, (127, 128, 0): 189689856,
    (1024, 32, 32): 941799424, (1024, 64, 32): 1539749888, (1024, 128, 32): 2735650816, (1024, 32, 96): 1539749888,
    (1024, 64, 96): 2137700352, (1024, 32, 160): 2137700352, (1024, 128, 0): 1239447552,
    (4096, 32, 32): 3644028928, (4096, 64, 32): 6035830784, (4096, 128, 32): 10819434496,
    (4096, 32, 96): 6035830784, (4096, 64, 96): 8427632640, (4096, 32, 160): 8427632640, (4096, 128, 0): 4834621440,
    (65536, 32, 32): 57688619008, (65536, 64, 32): 95957448704, (65536, 128, 32): 172495108096,
    (65536, 32, 96): 95957448704, (65536, 64, 96): 134226278400, (65536, 32, 160): 134226278400,
    (65536, 128, 0): 76738099200,
}
NERF = {1: 7176192, 128: 7176192, 129: 14147584, 196608: 1860153344, 10 ** 6: 9301867520}
# entry -> {shape: bytes}
MESH = {
    "nerfb200_mc_workspace_bytes": {
        (2, 2, 2): 1024, (2, 3, 5): 1024, (33, 33, 33): 344320, (64, 65, 66): 2683904, (128, 128, 128): 20728320,
        (257, 257, 257): 168760064, (1, 4, 4): 0, (737, 737, 737): 0},
    "nerfb200_mesh_cluster_workspace_bytes": {
        (0, 1): 2816, (3, 1): 2816, (1000, 1): 7424, (100, 200): 19200, (4068, 8000): 701184,
        (292916, 585000): 51190784, (2 ** 20 + 1, 2 ** 21): 183502080, (5, 0): 0, (-1, 3): 0},
    "nerfb200_volume_workspace_bytes": {
        (1,): 0, (2,): 512, (3,): 512, (65,): 1536, (128,): 8704, (256,): 66048, (512,): 524800, (1625,): 16761856,
        (1626,): 0},
    "nerfb200_vertex_normals_workspace_bytes": {
        (0, 0): 256, (10, 0): 256, (3, 1): 1536, (100, 200): 15360, (100, 2000): 144640, (4068, 8000): 576256,
        (2 ** 20 + 1, 2 ** 21): 150995200, (-1, 3): 0},
    "nerfb200_occupancy_workspace_bytes": {
        (1,): 0, (2,): 512, (3,): 512, (65,): 524288, (128,): 4097024, (129,): 4194304, (257,): 33554432,
        (1625,): 8566197248, (1626,): 0},
    "nerfb200_cull_workspace_bytes": {
        (-1,): 0, (0,): 512, (1,): 512, (255,): 512, (256,): 512, (257,): 512, (160000,): 7680, (640000,): 30464,
        (1 << 24,): 786944},
    "nerfb200_sigma_grid_workspace_bytes": {
        (0,): 0, (1,): 256, (21,): 256, (22,): 512, (1000,): 12032, (1 << 21,): 25165824, (1 << 22,): 50331648},
}


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


@pytest.mark.parametrize("entry,shape", [(e, s) for e in MESH for s in MESH[e]])
def test_mesh_and_culling_workspace_bytes(lib, entry, shape):
    assert getattr(lib, entry)(*shape) == MESH[entry][shape]
