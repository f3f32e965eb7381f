"""The C ABI of the sparse marching cubes (include/nerf_pl_b200_sparse_mc.h): its prototypes against
_lib.SPARSE_MC_SIGNATURES, the workspace sizes, and the argument errors every entry returns before any launch."""
import ctypes
import math
import os
import re

import pytest

from nerf_pl_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", _lib.SPARSE_MC_INCLUDE)
BOX = (ctypes.c_double * 6)(-1, 1, -1, 1, -1, 1)


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


def _prototypes():
    hdr = re.sub(r"/\*.*?\*/", " ", open(HEADER).read(), flags=re.S)
    hdr = "\n".join(ln for ln in hdr.splitlines() if not ln.lstrip().startswith("#"))
    out = []
    for decl in hdr.split(";"):
        m = re.search(r"(.*?)\b(nerfb200_\w+)\s*\((.*)\)\s*$", decl.strip(), re.S)
        if m:
            ret = " ".join(re.split(r"[{}]", m.group(1))[-1].split())
            out.append((m.group(2), ret, [" ".join(a.split()) for a in m.group(3).split(",")]))
    return out


def test_header_matches_the_signature_table(lib):
    scalars = {"int64_t": ctypes.c_int64, "size_t": ctypes.c_size_t, "double": ctypes.c_double}
    returns = {"int": ctypes.c_int32, "size_t": ctypes.c_size_t}
    protos = _prototypes()
    assert [n for n, _, _ in protos] == list(_lib.SPARSE_MC_SIGNATURES)
    assert not set(_lib.SPARSE_MC_SIGNATURES) & set(_lib.SIGNATURES)
    for name, ret, args in protos:
        restype, argtypes = _lib.SPARSE_MC_SIGNATURES[name]
        assert restype is returns[ret] and len(argtypes) == len(args), name
        for decl, t in zip(args, argtypes):
            m = re.fullmatch(r"(?:const )?(\w+)(\s*\*)?\s*(\w+)(\[\d+\])?", decl)
            assert m, (name, decl)
            base, star, arg, array = m.groups()
            if array or (star and arg.endswith("_host")):
                want = ctypes.POINTER(scalars[base])
            elif star:
                want = ctypes.c_void_p
            else:
                want = scalars[base]
            assert t is want, (name, decl, t)
        fn = getattr(lib, name)
        assert fn.restype is restype and list(fn.argtypes) == argtypes, name


def test_workspace_sizes(lib):
    plan, ws, emit = (lib.nerfb200_sparse_mc_plan_workspace_bytes, lib.nerfb200_sparse_mc_workspace_bytes,
                      lib.nerfb200_sparse_mc_emit_workspace_bytes)
    for N in (1, 0, -1, 2049):
        assert plan(N) == 0 and ws(N, 0, 0) == 0
    for N in (2, 8, 9, 1024, 2048):
        B = (-(-N // 8)) ** 3
        assert 21 * B <= plan(N) < 21 * B + (1 << 22), N
    assert plan(2048) < 360 * 2 ** 20                             # the brick map alone is 64 MiB at N = 2048
    # 2 KiB of values and 16 B of row counts and offsets per active brick, 20 B per march brick, one query's rows
    assert ws(64, 10, 12) >= 10 * 2064 + 12 * 20 + 10 * 512 * 24
    assert ws(2048, 4096, 5000) < ws(2048, 8192, 9000) < ws(2048, 8192, 20000)
    assert ws(2048, 10 ** 6, 10 ** 6) < 10 ** 6 * 2100 + (4096 * 512 * 24) + (1 << 24)
    for bad in ((9, -1, 0), (9, 2, 1), (9, 0, 1), (9, 1, 9), (2049, 1, 1)):   # march >= active, both <= the bricks
        assert ws(*bad) == 0, bad
    assert emit(-1, 0) == 0 and emit(0, -1) == 0 and emit(2 ** 31, 0) == 0 and emit(0, 2 ** 31) == 0
    assert emit(1000, 2000) >= 16 * 3000


def _c(v):
    return (ctypes.c_int64 * 2)(*v)


ONE = ctypes.c_void_p(256)      # never dereferenced: every call below fails before touching the device


def _plan(lib, **kw):
    a = dict(N=17, ranges=BOX, bits=ONE, occ_N=9, occ_ranges=BOX, ws=ONE, nbytes=1 << 40, out=_c((0, 0)))
    a.update(kw)
    return lib.nerfb200_sparse_mc_plan(*a.values(), None)


def _count(lib, **kw):
    a = dict(packed=ONE, N=17, ranges=BOX, bits=ONE, occ_N=9, occ_ranges=BOX, thr=20.0, plan=ONE, plan_bytes=1 << 40,
             bricks=_c((1, 2)), ws=ONE, nbytes=1 << 40, out=_c((0, 0)))
    a.update(kw)
    return lib.nerfb200_sparse_mc_count(*a.values(), None)


def _emit(lib, **kw):
    a = dict(N=17, thr=20.0, plan=ONE, plan_bytes=1 << 40, bricks=_c((1, 2)), ws=ONE, nbytes=1 << 40,
             counts=_c((6, 8)), emit=ONE, emit_bytes=1 << 40, verts=ONE, tris=ONE)
    a.update(kw)
    return lib.nerfb200_sparse_mc_emit(*a.values(), None)


GRID_CASES = [(dict(N=1), b"[2, 2048]"), (dict(N=2049), b"[2, 2048]"), (dict(N=-4), b"[2, 2048]"),
              (dict(ranges=None), b"NULL"), (dict(bits=None), b"NULL"), (dict(occ_ranges=None), b"NULL"),
              (dict(occ_N=1), b"N must be in [2, 1625]"), (dict(occ_N=1626), b"N must be in [2, 1625]"),
              (dict(occ_N=9 + (8 << 32)), b"levels must be in [1, 8]"),
              (dict(occ_ranges=(ctypes.c_double * 6)(-1, 1, 0.5, 0.5, -1, 1)), b"finite with min != max"),
              (dict(occ_ranges=(ctypes.c_double * 6)(-1, 1, -1, 1, math.nan, 1)), b"finite with min != max"),
              (dict(occ_ranges=(ctypes.c_double * 6)(-1e308, 1e308, -1, 1, -1, 1), occ_N=9 + (1 << 32)),
               b"level 1's box")]


def _expect(lib, rc, kw, msg):
    assert rc == -1, kw
    assert msg in lib.nerfb200_last_error(), (kw, lib.nerfb200_last_error())


def test_plan_argument_checks(lib):
    cases = GRID_CASES + [(dict(ws=None), b"NULL"), (dict(out=None), b"NULL"),
                          (dict(nbytes=lib.nerfb200_sparse_mc_plan_workspace_bytes(17) - 1), b"plan workspace smaller"),
                          (dict(N=65, nbytes=lib.nerfb200_sparse_mc_plan_workspace_bytes(64)), b"plan workspace smaller")]
    for kw, msg in cases:
        _expect(lib, _plan(lib, **kw), kw, msg)


def test_count_argument_checks(lib):
    ws = lib.nerfb200_sparse_mc_workspace_bytes(17, 1, 2)
    cases = GRID_CASES + [(dict(packed=None), b"NULL"), (dict(plan=None), b"NULL"), (dict(bricks=None), b"NULL"),
                          (dict(ws=None), b"NULL"), (dict(out=None), b"NULL"),
                          (dict(bricks=_c((2, 1))), b"bricks_host"), (dict(bricks=_c((-1, 2))), b"bricks_host"),
                          (dict(bricks=_c((1, 28))), b"bricks_host"),
                          (dict(plan_bytes=lib.nerfb200_sparse_mc_plan_workspace_bytes(17) - 1), b"plan workspace"),
                          (dict(nbytes=ws - 1), b"workspace smaller"),
                          (dict(bricks=_c((2, 2)), nbytes=ws), b"workspace smaller")]
    for kw, msg in cases:
        _expect(lib, _count(lib, **kw), kw, msg)


def test_emit_argument_checks(lib):
    ws = lib.nerfb200_sparse_mc_workspace_bytes(17, 1, 2)
    em = lib.nerfb200_sparse_mc_emit_workspace_bytes(6, 8)
    cases = [(dict(N=1), b"[2, 2048]"), (dict(N=2049), b"[2, 2048]"),
             (dict(plan=None), b"NULL"), (dict(bricks=None), b"NULL"), (dict(ws=None), b"NULL"),
             (dict(counts=None), b"NULL"), (dict(emit=None), b"NULL"), (dict(verts=None), b"NULL"),
             (dict(tris=None), b"NULL"), (dict(bricks=_c((3, 2))), b"bricks_host"),
             (dict(counts=_c((-1, 0))), b"counts_host"), (dict(counts=_c((0, 4))), b"counts_host"),
             (dict(counts=_c((2 ** 31, 0))), b"counts_host"),
             (dict(plan_bytes=lib.nerfb200_sparse_mc_plan_workspace_bytes(17) - 1), b"plan workspace"),
             (dict(nbytes=ws - 1), b"workspace smaller"), (dict(emit_bytes=em - 1), b"emit workspace smaller"),
             (dict(counts=_c((600, 8)), emit_bytes=em), b"emit workspace smaller")]
    for kw, msg in cases:
        _expect(lib, _emit(lib, **kw), kw, msg)
