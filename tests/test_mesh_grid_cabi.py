"""The C ABI of the mesh grids taken through an occupancy grid: the arguments both entries take, the workspace sizes,
and the argument errors the entries return before any launch."""
import ctypes
import math

import pytest

from nerf_pl_b200 import _lib

from .test_cabi import _header_prototypes

BOX = (ctypes.c_double * 6)(-1, 1, -1, 1, -1, 1)


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


def test_both_grid_entries_take_the_same_arguments():
    """The output's name aside."""
    protos = {name: args for name, _, args in _header_prototypes()}
    sigma, rgb = protos["nerfb200_sigma_grid_masked"], protos["nerfb200_rgb_sigma_grid_masked"]
    assert [a.split()[-1] for a in sigma] == [
        "packed", "N", "ranges_host[6]", "bits", "occ_N", "occ_ranges_host[6]", "chunk", "ws", "bytes", "sigma_out",
        "evaluated_host", "stream"]
    assert sigma[:9] + sigma[10:] == rgb[:9] + rgb[10:]


def test_workspace_sizes(lib):
    ws = lib.nerfb200_masked_grid_workspace_bytes
    assert ws(0) == 0 and ws(-1) == 0
    # positions (12 B), index (8 B) and four query channels (16 B) per point, plus the tile counts and CUB's scratch
    for chunk in (1, 127, 4096, 4097, 1 << 21):
        assert ws(chunk) >= 36 * chunk, chunk
    assert ws(1) < ws(127) < ws(4096) < ws(4097) < ws(1 << 21)
    assert ws(1 << 21) < 36 * (1 << 21) + (1 << 20)


def _call(lib, entry, **kw):
    one = ctypes.c_void_p(256)          # never dereferenced: every call below fails before any launch
    a = dict(packed=one, N=17, ranges=BOX, bits=one, occ_N=9, occ_ranges=BOX, chunk=1024, ws=one, nbytes=1 << 40,
             out=one, evaluated=ctypes.byref(ctypes.c_int64(-7)))
    a.update(kw)
    return getattr(lib, entry)(*a.values(), None)


@pytest.mark.parametrize("entry", ["nerfb200_sigma_grid_masked", "nerfb200_rgb_sigma_grid_masked"])
def test_argument_checks(lib, entry):
    cases = [(dict(N=1), b"N"), (dict(N=-5), b"N"), (dict(chunk=0), b"chunk"), (dict(chunk=-1), b"chunk"),
             (dict(packed=None), b"NULL"), (dict(ranges=None), b"NULL"), (dict(bits=None), b"NULL"),
             (dict(occ_ranges=None), b"NULL"), (dict(ws=None), b"NULL"), (dict(out=None), b"NULL"),
             (dict(evaluated=None), b"NULL"),
             (dict(occ_N=1), b"N must be in [2, 1625]"), (dict(occ_N=1626), b"N must be in [2, 1625]"),
             (dict(occ_ranges=(ctypes.c_double * 6)(-1, 1, 0.5, 0.5, -1, 1)), b"finite with min != max"),
             (dict(occ_ranges=(ctypes.c_double * 6)(-1, 1, -1, 1, math.nan, 1)), b"finite with min != max"),
             (dict(occ_ranges=(ctypes.c_double * 6)(-math.inf, 1, -1, 1, -1, 1)), b"finite with min != max"),
             (dict(nbytes=lib.nerfb200_masked_grid_workspace_bytes(1024) - 1), b"workspace smaller"),
             (dict(chunk=4097, nbytes=lib.nerfb200_masked_grid_workspace_bytes(4096)), b"workspace smaller")]
    if entry == "nerfb200_rgb_sigma_grid_masked":
        cases += [(dict(N=1626), b"[2, 1625]"), (dict(out=ctypes.c_void_p(256 + 8)), b"16-byte aligned")]
    for kw, msg in cases:
        assert _call(lib, entry, **kw) == -1, kw
        assert msg in lib.nerfb200_last_error(), (kw, lib.nerfb200_last_error())
