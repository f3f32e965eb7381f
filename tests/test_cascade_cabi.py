"""CPU-side checks of cascaded occupancy grids at the C ABI (include/nerf_pl_b200.h "cascaded occupancy grids"): the
grid size argument that carries the level count, the grown argument structs, argument checks and workspace sizes,
with no device touched, and the Python surface."""
import ctypes
import inspect
import os
import re
import subprocess

import pytest

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib, culling

from . import test_cabi as tc


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


def test_grid_n_keeps_one_level_values_and_matches_the_header_macro(tmp_path):
    """NERFB200_GRID_N(N, L) == _lib.grid_n(N, L): N itself for one level, L - 1 in the word above N otherwise."""
    assert _lib.grid_n(9) == _lib.grid_n(9, 1) == 9
    assert _lib.grid_n(129, 4) == 129 + (3 << 32)
    src = tmp_path / "g.c"
    src.write_text('#include <stdio.h>\n#include "nerf_pl_b200.h"\nint main(void){\n' +
                   "".join(f'printf("%lld\\n", (long long)NERFB200_GRID_N({n}, {L}));\n'
                           for n, L in ((9, 1), (129, 4), (1625, 8))) + "return 0;}\n")
    exe = tmp_path / "g"
    subprocess.run(["gcc", "-I", os.path.dirname(tc.HEADER), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [_lib.grid_n(9, 1), _lib.grid_n(129, 4), _lib.grid_n(1625, 8)]


def test_argument_structs_grow_by_levels_at_their_ends():
    for name, mirror in (("nerfb200_samples_args", _lib.SamplesArgs),
                         ("nerfb200_train_samples_args", _lib.TrainSamplesArgs)):
        assert tc._struct_fields(name)[-1] == "levels"
        assert mirror._fields_[-1] == ("levels", ctypes.c_int32)
        assert mirror().levels == 0                     # zero-filled: one level


def test_the_header_declares_no_new_entry():
    """The cascade goes through the existing entries: the signature table is unchanged in size."""
    assert len(tc._header_prototypes()) == len(_lib.SIGNATURES) == 75
    assert not any("levels" in n for n in _lib.SIGNATURES)


RANGES = (ctypes.c_double * 6)(-1.0, 1.0, -1.0, 1.0, -1.0, 1.0)
DUMMY = ctypes.c_void_p(16)                              # never dereferenced: every call below fails its checks first


def _calls(lib, grid_N):
    n = ctypes.c_int64()
    return {
        "nerfb200_occupancy_pack": (DUMMY, grid_N, 0.5, 1, DUMMY, 1 << 20, DUMMY, None),
        "nerfb200_occupancy_popcount": (DUMMY, grid_N, DUMMY, None),
        "nerfb200_cull_count": (DUMMY, 0, DUMMY, grid_N, RANGES, DUMMY, 1 << 20, DUMMY, ctypes.byref(n), None),
        "nerfb200_density_points": (grid_N, RANGES, DUMMY, 0, 1, DUMMY, None),
        "nerfb200_density_update": (DUMMY, grid_N, RANGES, 0.5, 0.9, 1, 64, DUMMY, DUMMY, DUMMY, DUMMY, 1 << 20, None),
        "nerfb200_sigma_grid_masked": (DUMMY, 4, RANGES, DUMMY, grid_N, RANGES, 64, DUMMY, 1 << 20, DUMMY,
                                       ctypes.byref(n), None),
        "nerfb200_rgb_sigma_grid_masked": (DUMMY, 4, RANGES, DUMMY, grid_N, RANGES, 64, DUMMY, 1 << 20, DUMMY,
                                           ctypes.byref(n), None),
    }


@pytest.mark.parametrize("levels", [9, 100])
def test_levels_above_8_are_rejected(lib, levels):
    for name, args in _calls(lib, _lib.grid_n(9, levels)).items():
        assert getattr(lib, name)(*args) == -1, name
        assert b"levels must be in [1, 8]" in lib.nerfb200_last_error(), name
    assert lib.nerfb200_occupancy_workspace_bytes(_lib.grid_n(9, levels)) == 0
    assert lib.nerfb200_density_workspace_bytes(_lib.grid_n(9, levels), 64) == 0


@pytest.mark.parametrize("N", [1, 1626, -5])
def test_grid_sizes_outside_2_to_1625_are_rejected_at_every_level_count(lib, N):
    for levels in ((1, 4) if N > 0 else (1,)):
        for name, args in _calls(lib, _lib.grid_n(N, levels)).items():
            assert getattr(lib, name)(*args) == -1, (name, levels)
            assert b"N must be in [2, 1625]" in lib.nerfb200_last_error(), (name, levels)


def test_density_points_number_the_evaluated_cells_of_every_level(lib):
    """N = 9, L = 2: 8^3 cells of level 0, then 8^3 - 4^3 = 448 non-inner cells of level 1."""
    g = _lib.grid_n(9, 2)
    assert lib.nerfb200_density_points(g, RANGES, DUMMY, 0, 512 + 449, DUMMY, None) == -1
    assert b"outside the grid" in lib.nerfb200_last_error()
    assert lib.nerfb200_density_points(g, RANGES, DUMMY, 512 + 448, 0, DUMMY, None) == 0
    huge = (ctypes.c_double * 6)(-1e307, 1e307, -1.0, 1.0, -1.0, 1.0)      # 2^7 h overflows
    assert lib.nerfb200_density_points(_lib.grid_n(9, 8), huge, DUMMY, 0, 1, DUMMY, None) == -1
    assert b"box is not finite" in lib.nerfb200_last_error()
    n = ctypes.c_int64()
    assert lib.nerfb200_cull_count(DUMMY, 0, DUMMY, _lib.grid_n(9, 8), huge, DUMMY, 1 << 20, DUMMY,
                                   ctypes.byref(n), None) == -1


def test_workspaces_are_one_levels(lib):
    """Packing and the density update reuse one level's workspace for every level."""
    for L in (2, 8):
        assert lib.nerfb200_occupancy_workspace_bytes(_lib.grid_n(129, L)) == lib.nerfb200_occupancy_workspace_bytes(129)
        assert lib.nerfb200_density_workspace_bytes(_lib.grid_n(33, L), 1000) == \
            lib.nerfb200_density_workspace_bytes(33, 1000)


def test_samples_args_levels_are_checked(lib):
    """A render whose grid has levels = 9 is refused before anything runs."""
    a = _lib.SamplesArgs(rays=DUMMY, n_rays=1, packed_coarse=DUMMY, n_samples=64, n_importance=0, bits=DUMMY, N=9,
                         ranges=RANGES, levels=9)
    live = (ctypes.c_int64 * 2)()
    assert lib.nerfb200_render_samples(ctypes.byref(a), DUMMY, 1 << 30, live, None) == -1
    assert b"levels must be in [1, 8]" in lib.nerfb200_last_error()


def test_python_surface():
    for name in ("level_ranges", "occupancy_cascade"):
        assert name in nb.__all__ and hasattr(nb, name)
    assert list(inspect.signature(nb.occupancy_cascade).parameters) == [
        "model", "N", "x_range", "y_range", "z_range", "sigma_threshold", "levels", "dilate", "chunk"]
    for fn in (nb.pack_occupancy, nb.OccupancyGrid, nb.DensityGrid):
        p = inspect.signature(fn).parameters
        assert list(p)[-1] == "levels" and p["levels"].default == 1, fn
    for bad in (0, 9, 1.5):
        with pytest.raises(ValueError, match="levels"):
            culling._check_levels(bad, "x")
    assert nb.level_ranges((-1, 1), (0, 2), (2, 3), 2) == ((-4.0, 4.0), (-3.0, 5.0), (0.5, 4.5))
    assert culling.inner_cells(9, 0) == (0, 0) and culling.inner_cells(9, 1) == (2, 6)
    assert culling.inner_cells(10, 3) == (3, 6)
    assert not re.search(r"\blevels\b", str(inspect.signature(nb.occupancy_grid)))
