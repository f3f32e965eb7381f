"""The C ABI of the view-dependent baked volumes (include/nerf_pl_b200_baked_sh.h): its prototypes against
_lib.BAKED_SH_SIGNATURES, the byte formulas, and the argument errors every entry returns before any launch (no device
needed)."""
import ctypes
import math
import os
import re

import pytest

from nerf_pl_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", _lib.BAKED_SH_INCLUDE)
BOX = (ctypes.c_double * 6)(-1, 1, -1, 1, -1, 1)
ONE = ctypes.c_void_p(256)      # never dereferenced: every call below fails before touching the device
POINT = 729 * 7 * 16            # bytes of one stored brick


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
            args = [] if m.group(3).strip() == "void" else [" ".join(a.split()) for a in m.group(3).split(",")]
            out.append((m.group(2), ret, args))
    return out


def test_header_matches_the_signature_table(lib):
    scalars = {"int64_t": ctypes.c_int64, "int32_t": ctypes.c_int32, "size_t": ctypes.c_size_t,
               "double": ctypes.c_double, "float": ctypes.c_float}
    returns = {"int": ctypes.c_int32, "size_t": ctypes.c_size_t}
    protos = _prototypes()
    assert [n for n, _, _ in protos] == list(_lib.BAKED_SH_SIGNATURES)
    for other in (_lib.SIGNATURES, _lib.SPARSE_MC_SIGNATURES, _lib.BAKED_SIGNATURES):
        assert not set(_lib.BAKED_SH_SIGNATURES) & set(other)
    for name, ret, args in protos:
        restype, argtypes = _lib.BAKED_SH_SIGNATURES[name]
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
    assert lib.nerfb200_abi_version() == 3


def test_byte_formulas(lib):
    vol, ws = lib.nerfb200_baked_sh_bytes, lib.nerfb200_baked_sh_workspace_bytes
    assert POINT == 81648
    for N in (2, 8, 9, 17, 512, 1024):
        B = (-(-N // 8)) ** 3
        for bricks in (0, 1, B // 2, B):
            assert vol(N, bricks) == POINT * bricks + 4 * B, (N, bricks)
        assert vol(N, B + 1) == 0 and vol(N, -1) == 0
    for N in (1, 0, -1, 1025, 2048):
        assert vol(N, 0) == 0 and ws(N, 0, 0) == 0
    # the volume of the counts measured in DESIGN.md §10j, as the table there states
    table = lib.nerfb200_query_rgb_sh_workspace_bytes()
    assert table == (64 * 128 + 64 * 28) * 4
    # one query's rows (12 B of position, 8 of destination, 112 of output per point), 16 B of offsets per brick and
    # the table
    assert ws(64, 10, 12) >= 10 * 512 * 132 + 10 * 16 + table
    assert ws(64, 10, 12) > lib.nerfb200_baked_workspace_bytes(64, 10, 12)
    assert ws(1024, 4096, 5000) == ws(1024, 4096, 9000)
    for bad in ((9, -1, 0), (9, 2, 1), (9, 0, 1), (9, 1, 9), (1025, 1, 1)):
        assert ws(*bad) == 0, bad


def _expect(lib, rc, kw, msg):
    assert rc == -1, kw
    assert msg in lib.nerfb200_last_error(), (kw, lib.nerfb200_last_error())


def _c(*v):
    return (ctypes.c_int64 * len(v))(*v)


def _bake(lib, **kw):
    a = dict(packed=ONE, N=17, ranges=BOX, bits=ONE, occ_N=9, occ_ranges=BOX, plan=ONE, plan_bytes=1 << 40,
             bricks=_c(1, 2), ws=ONE, nbytes=1 << 40, volume=ONE, volume_bytes=lib.nerfb200_baked_sh_bytes(17, 2))
    a.update(kw)
    return lib.nerfb200_baked_sh_bake(*a.values(), None)


def test_bake_argument_checks(lib):
    cases = [(dict(N=1), b"[2, 1024]"), (dict(N=1025), b"[2, 1024]"), (dict(ranges=None), b"NULL"),
             (dict(bits=None), b"NULL"), (dict(occ_ranges=None), b"NULL"), (dict(packed=None), b"NULL"),
             (dict(plan=None), b"NULL"), (dict(bricks=None), b"NULL"), (dict(ws=None), b"NULL"),
             (dict(volume=None), b"NULL"),
             (dict(occ_N=1), b"N must be in [2, 1625]"), (dict(occ_N=9 + (8 << 32)), b"levels must be in [1, 8]"),
             (dict(occ_ranges=(ctypes.c_double * 6)(-1, 1, 0.5, 0.5, -1, 1)), b"finite with min != max"),
             (dict(bricks=_c(2, 1)), b"not a plan's"), (dict(bricks=_c(-1, 0)), b"not a plan's"),
             (dict(bricks=_c(0, 1)), b"not a plan's"), (dict(bricks=_c(1, 28)), b"not a plan's"),
             (dict(plan_bytes=16), b"plan workspace smaller"),
             (dict(nbytes=lib.nerfb200_baked_sh_workspace_bytes(17, 1, 2) - 1), b"nerfb200_baked_sh_workspace_bytes"),
             (dict(volume_bytes=lib.nerfb200_baked_sh_bytes(17, 2) - 1), b"volume_bytes differs"),
             (dict(volume_bytes=lib.nerfb200_baked_bytes(17, 2)), b"nerfb200_baked_sh_bytes")]
    for kw, msg in cases:
        _expect(lib, _bake(lib, **kw), kw, msg)


def test_from_grid_argument_checks(lib):
    count, fill = lib.nerfb200_baked_sh_from_grid_count, lib.nerfb200_baked_sh_from_grid
    out = _c(0)
    for N in (1, 1025):
        _expect(lib, count(ONE, N, ONE, 1 << 40, out, None), N, b"[2, 1024]")
        _expect(lib, fill(ONE, N, ONE, 1 << 40, 0, ONE, lib.nerfb200_baked_sh_bytes(9, 0), None), N, b"[2, 1024]")
    for args in ((None, 9, ONE, 1 << 40, out), (ONE, 9, None, 1 << 40, out), (ONE, 9, ONE, 1 << 40, None)):
        _expect(lib, count(*args, None), args, b"NULL")
    _expect(lib, count(ONE, 9, ONE, 16, out, None), "plan bytes", b"plan workspace smaller")
    good = lib.nerfb200_baked_sh_bytes(17, 5)
    for kw, msg in ((dict(grid=None), b"NULL"), (dict(plan=None), b"NULL"), (dict(volume=None), b"NULL"),
                    (dict(bricks=-1), b"bricks must be in"), (dict(bricks=28), b"bricks must be in"),
                    (dict(volume_bytes=good + 16), b"volume_bytes differs"),
                    (dict(volume_bytes=lib.nerfb200_baked_bytes(17, 5)), b"volume_bytes differs"),
                    (dict(plan_bytes=16), b"plan workspace smaller")):
        a = dict(grid=ONE, N=17, plan=ONE, plan_bytes=1 << 40, bricks=5, volume=ONE, volume_bytes=good)
        a.update(kw)
        _expect(lib, fill(*a.values(), None), kw, msg)


def test_to_dense_argument_checks(lib):
    fn = lib.nerfb200_baked_sh_to_dense
    good = lib.nerfb200_baked_sh_bytes(17, 3)
    for args, msg in (((ONE, good, 1, 3, ONE), b"[2, 1024]"), ((ONE, good, 1025, 3, ONE), b"[2, 1024]"),
                      ((None, good, 17, 3, ONE), b"NULL"), ((ONE, good, 17, 3, None), b"NULL"),
                      ((ONE, good, 17, 28, ONE), b"bricks must be in"),
                      ((ONE, good - 4, 17, 3, ONE), b"volume_bytes differs")):
        _expect(lib, fn(*args, None), args, msg)


def _render(lib, **kw):
    a = dict(volume=ONE, volume_bytes=lib.nerfb200_baked_sh_bytes(17, 3), N=17, ranges=BOX, bricks=3, rays=ONE, n=10,
             step=0.1, white_back=0, eps=0.0, rgb=ONE, depth=ONE, opacity=ONE)
    a.update(kw)
    return lib.nerfb200_baked_sh_render(*a.values(), None)


def test_render_argument_checks(lib):
    cases = [(dict(N=1), b"[2, 1024]"), (dict(N=1025), b"[2, 1024]"), (dict(volume=None), b"NULL"),
             (dict(ranges=None), b"NULL"), (dict(rays=None), b"NULL"), (dict(rgb=None), b"NULL"),
             (dict(depth=None), b"NULL"), (dict(opacity=None), b"NULL"),
             (dict(bricks=-1), b"bricks must be in"), (dict(bricks=28), b"bricks must be in"),
             (dict(volume_bytes=lib.nerfb200_baked_sh_bytes(17, 4)), b"volume_bytes differs"),
             (dict(volume_bytes=lib.nerfb200_baked_bytes(17, 3)), b"volume_bytes differs"),
             (dict(step=0.0), b"step must be"), (dict(step=-1.0), b"step must be"), (dict(step=math.nan), b"step must be"),
             (dict(step=math.inf), b"step must be"), (dict(step=1e-300), b"step must be"), (dict(step=1e300), b"step must be"),
             (dict(eps=-1e-9), b"early_stop must be"), (dict(eps=1.5), b"early_stop must be"),
             (dict(eps=math.nan), b"early_stop must be"), (dict(white_back=2), b"white_back must be"),
             (dict(n=-1), b"n_rays < 0"),
             (dict(ranges=(ctypes.c_double * 6)(-1, 1, 0.5, 0.5, -1, 1)), b"finite with min != max"),
             (dict(ranges=(ctypes.c_double * 6)(-1, 1, -1, 1, math.nan, 1)), b"finite with min != max")]
    for kw, msg in cases:
        _expect(lib, _render(lib, **kw), kw, msg)
    assert _render(lib, n=0, rays=None, rgb=None, depth=None, opacity=None) == 0


def test_query_argument_checks(lib):
    fn = lib.nerfb200_query_rgb_sh
    full = lib.nerfb200_query_rgb_sh_workspace_bytes()
    for args, msg in (((ONE, -1, 3, ONE, ONE, full, ONE), b"n < 0"), ((None, 5, 3, ONE, ONE, full, ONE), b"NULL"),
                      ((ONE, 5, 3, None, ONE, full, ONE), b"NULL"), ((ONE, 5, 3, ONE, None, full, ONE), b"NULL"),
                      ((ONE, 5, 3, ONE, ONE, full, None), b"NULL"), ((ONE, 5, 2, ONE, ONE, full, ONE), b"xyz_stride"),
                      ((ONE, 5, 3, ONE, ONE, full, ctypes.c_void_p(260)), b"16-byte aligned"),
                      ((ONE, 5, 3, ONE, ctypes.c_void_p(260), full, ONE), b"16-byte aligned"),
                      ((ONE, 5, 3, ONE, ONE, full - 1, ONE), b"workspace smaller")):
        _expect(lib, fn(*args, None), args, msg)
    assert fn(None, 0, 3, None, None, 0, None, None) == 0         # empty input is a no-op
