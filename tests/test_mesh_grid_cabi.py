"""The C ABI of the mesh grids taken through an occupancy grid: the companion header
include/nerf_pl_b200_masked_grid.h against _lib.MASKED_GRID_SIGNATURES and the library's exports, the workspace
sizes, and the argument errors the entries return before any launch."""
import ctypes
import math
import os
import re

import pytest

from nerf_pl_b200 import _lib

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "nerf_pl_b200_masked_grid.h")
BOX = (ctypes.c_double * 6)(-1, 1, -1, 1, -1, 1)


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


def _prototypes():
    hdr = re.sub(r"/\*.*?\*/", " ", open(HEADER).read(), flags=re.S)
    hdr = "\n".join(ln for ln in hdr.splitlines() if not ln.lstrip().startswith("#"))
    protos = []
    for decl in hdr.split(";"):
        m = re.search(r"(\w[\w\s\*]*?)\b(nerfb200_\w+)\s*\((.*)\)\s*$", decl.strip(), re.S)
        if m:
            protos.append((m.group(2), " ".join(m.group(1).split()), [" ".join(a.split()) for a in m.group(3).split(",")]))
    return protos


def test_signature_table_matches_the_companion_header(lib):
    protos = _prototypes()
    names = [n for n, _, _ in protos]
    assert names == list(_lib.MASKED_GRID_SIGNATURES) == ["nerfb200_masked_grid_workspace_bytes",
                                                          "nerfb200_sigma_grid_masked",
                                                          "nerfb200_rgb_sigma_grid_masked"]
    others = (_lib.SIGNATURES, _lib.METRICS_SIGNATURES, _lib.VIEWS_SIGNATURES, _lib.SAMPLES_SIGNATURES,
              _lib.TRAIN_SAMPLES_SIGNATURES, _lib.DENSITY_SIGNATURES)
    assert not set(names) & set().union(*others)
    scalars = {"int64_t": ctypes.c_int64, "int32_t": ctypes.c_int32, "size_t": ctypes.c_size_t, "int": ctypes.c_int32,
               "double": ctypes.c_double, "float": ctypes.c_float}
    for name, ret, args in protos:
        restype, argtypes = _lib.MASKED_GRID_SIGNATURES[name]
        assert restype is scalars[ret], (name, ret)
        assert len(argtypes) == len(args), (name, args)
        for decl, t in zip(args, argtypes):
            flat = decl.replace(" ", "")
            if "ranges_host[6]" in flat:
                assert t is ctypes.POINTER(ctypes.c_double), (name, decl)
            elif flat == "int64_t*evaluated_host":
                assert t is ctypes.POINTER(ctypes.c_int64), (name, decl)   # a host pointer
            elif "*" in decl:
                assert t is ctypes.c_void_p, (name, decl, t)               # device pointers
            else:
                assert t is scalars[decl.replace("const ", "").rsplit(" ", 1)[0]], (name, decl, t)
        fn = getattr(lib, name)
        assert fn.restype is restype and list(fn.argtypes) == argtypes, name
    # both grid entries take the same arguments, the output's name aside
    assert [a.split()[-1] for a in protos[1][2]] == [
        "packed", "N", "ranges_host[6]", "bits", "occ_N", "occ_ranges_host[6]", "chunk", "ws", "bytes", "sigma_out",
        "evaluated_host", "stream"]
    assert protos[1][2][:9] + protos[1][2][10:] == protos[2][2][:9] + protos[2][2][10:]
    assert '#include "nerf_pl_b200.h"' in open(HEADER).read()
    assert "nerf_pl_b200_masked_grid.h" in _lib.INCLUDES and "masked_grid_kernels.cuh" in _lib.HEADERS
    assert lib.nerfb200_abi_version() == 3


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
