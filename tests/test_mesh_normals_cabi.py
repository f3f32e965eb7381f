"""CPU-side checks of the vertex-normal colouring entries: workspace sizes and the argument checks that need no GPU
(their prototypes are checked with the rest of include/nerf_pl_b200.h in test_cabi.py)."""
import pytest

from nerf_pl_b200 import _lib


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


def test_workspace_sizes_and_argument_checks_without_a_gpu(lib):
    ws = lib.nerfb200_vertex_normals_workspace_bytes
    assert ws(-1, 3) == 0 and ws(3, -1) == 0 and ws(2 ** 31 - 1, 1) == 0 and ws(1, 2 ** 31 // 3 + 1) == 0
    assert ws(0, 0) > 0 and ws(10, 0) > 0
    small, big = ws(100, 200), ws(100, 2000)
    assert big > small >= 200 * 3 * 4 * 4 + 200 * 3 * 8   # corner keys / ids (and their sort buffers), triangle normals
    assert ws(2 ** 20 + 1, 2 ** 21) >= 3 * 2 ** 21 * 16 + 3 * 2 ** 21 * 8
    # no triangles on an empty vertex list: nothing to do; triangles on one: every index is out of range
    assert lib.nerfb200_vertex_normals(None, 0, None, 0, None, 0, None, None) == 0
    assert lib.nerfb200_vertex_normals(None, 0, None, 4, None, 0, None, None) == -1
    assert b"outside [0, n_verts)" in lib.nerfb200_last_error()
    assert lib.nerfb200_vertex_normals(None, -1, None, 0, None, 0, None, None) == -1
    assert lib.nerfb200_vertex_normals(None, 5, None, 1, None, 0, None, None) == -1   # NULL pointers
    assert lib.nerfb200_normal_rays(None, None, -1, 2.0, 6.0, 1.0, None, None) == -1
    assert lib.nerfb200_normal_rays(None, None, 0, 2.0, 6.0, 1.0, None, None) == 0
    assert lib.nerfb200_normal_rays(None, None, 3, 2.0, 6.0, 1.0, None, None) == -1
