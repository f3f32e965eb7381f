"""CPU-side checks of the companion header include/nerf_pl_b200_mesh_normals.h (the vertex-normal colouring method):
its prototypes against _lib.MESH_NORMALS_SIGNATURES, the library exports them, the main header includes it, and
the argument checks that need no GPU."""
import ctypes
import os
import re

import pytest

from nerf_pl_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "nerf_pl_b200_mesh_normals.h")


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


def _prototypes(path):
    hdr = re.sub(r"/\*.*?\*/", " ", open(path).read(), flags=re.S)
    hdr = "\n".join(ln for ln in hdr.splitlines() if not ln.lstrip().startswith("#"))
    protos = {}
    for decl in hdr.split(";"):
        m = re.search(r"(.*?)\b(nerfb200_\w+)\s*\((.*)\)\s*$", decl.strip(), re.S)
        if m:
            ret = " ".join(re.split(r"[{}]", m.group(1))[-1].split())
            protos[m.group(2)] = (ret, [" ".join(a.split()) for a in m.group(3).split(",")])
    return protos


def test_companion_header_matches_its_signature_table(lib):
    protos = _prototypes(HEADER)
    assert list(protos) == list(_lib.MESH_NORMALS_SIGNATURES)
    assert not set(protos) & set(_lib.SIGNATURES)
    scalars = {"int64_t": ctypes.c_int64, "size_t": ctypes.c_size_t, "float": ctypes.c_float}
    returns = {"int": ctypes.c_int32, "size_t": ctypes.c_size_t}
    for name, (ret, args) in protos.items():
        restype, argtypes = _lib.MESH_NORMALS_SIGNATURES[name]
        assert restype is returns[ret], name
        assert len(argtypes) == len(args), name
        for decl, t in zip(args, argtypes):
            if "*" in decl:
                assert t is ctypes.c_void_p, (name, decl)
            else:
                assert t is scalars[decl.replace("const ", "").rsplit(" ", 1)[0]], (name, decl)
        fn = getattr(lib, name)
        assert fn.restype is restype and list(fn.argtypes) == argtypes


def test_main_header_includes_the_companion():
    main = open(os.path.join(ROOT, "include", "nerf_pl_b200.h")).read()
    assert '#include "nerf_pl_b200_mesh_normals.h"' in main
    assert "#define NERFB200_ABI_VERSION 3" in main


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
