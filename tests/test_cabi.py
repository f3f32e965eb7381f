"""CPU-side checks of the drop-in boundary: the C-ABI library builds for sm_90a, loads, exports
every symbol include/nerf_pl_b200.h declares, validates arguments without touching a GPU, and the
Python mirror keeps the reference's names / signatures / state_dict keys."""
import ctypes
import inspect
import os
import re

import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib
from oracle import nerf_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


HEADER = os.path.join(ROOT, "include", "nerf_pl_b200.h")
# the argument structs the header declares and their ctypes mirrors
MIRRORS = {"nerfb200_render_args": _lib.RenderArgs, "nerfb200_backward_args": _lib.BackwardArgs,
           "nerfb200_samples_args": _lib.SamplesArgs, "nerfb200_train_samples_args": _lib.TrainSamplesArgs}


def test_header_symbols_exported(lib):
    hdr = open(HEADER).read()
    declared = set(re.findall(r"\b(nerfb200_[a-z_0-9]+)\s*\(", hdr)) - set(MIRRORS)
    assert len(declared) == 75
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    assert "#define NERFB200_ABI_VERSION 3" in hdr
    for k, v in (("MEAN", 0), ("SUM", 1), ("NONE", 2)):
        assert f"#define NERFB200_SSIM_{k} {v}" in hdr
    assert _lib.INCLUDES == ["nerf_pl_b200.h"]
    assert sorted(_lib.HEADERS) == sorted(f for f in os.listdir(_lib.CSRC) if f != "capi.cu")
    for name in declared:
        assert hasattr(lib, name), name


def _header_prototypes():
    """[(name, return type, [argument declarations])] of every function include/nerf_pl_b200.h declares, in order."""
    hdr = open(HEADER).read()
    hdr = re.sub(r"/\*.*?\*/", " ", hdr, flags=re.S)
    hdr = "\n".join(ln for ln in hdr.splitlines() if not ln.lstrip().startswith("#"))
    protos = []
    for decl in hdr.split(";"):
        m = re.search(r"(.*?)\b(nerfb200_\w+)\s*\((.*)\)\s*$", decl.strip(), re.S)
        if m:
            ret = " ".join(re.split(r"[{}]", m.group(1))[-1].split())
            args = [] if m.group(3).strip() == "void" else [" ".join(a.split()) for a in m.group(3).split(",")]
            protos.append((m.group(2), ret, args))
    return protos


# Pointer arguments whose memory is read or written on the host although their names do not end in `_host`.
HOST_POINTERS = {("nerfb200_adam_step", "numel"), ("nerfb200_adam_step_dev", "numel"),
                 ("nerfb200_train_samples_forward_dev", "live_samples_dev")}


def test_one_signature_table_matches_all_75_entries_of_the_header(lib):
    """Every prototype of include/nerf_pl_b200.h against _lib.SIGNATURES: the same names, declared once each, in the
    same order, with the same argument counts, argument types and return types (a wrong width would silently corrupt
    the argument); the loaded library's entries carry exactly those types.  A pointer is c_void_p (device memory),
    except: an argument struct is a pointer to its mirror, a table of pointers is POINTER(c_void_p), and host memory
    (an array, a name ending in `_host`, HOST_POINTERS) is a pointer to its scalar type."""
    protos = _header_prototypes()
    names = [name for name, _, _ in protos]
    assert len(names) == 75
    assert len(set(names)) == len(names), sorted(n for n in names if names.count(n) > 1)
    assert names == list(_lib.SIGNATURES) == list(_lib.EXPORTS)          # header order
    scalars = {"int64_t": ctypes.c_int64, "int32_t": ctypes.c_int32, "size_t": ctypes.c_size_t,
               "float": ctypes.c_float, "double": ctypes.c_double}
    returns = {"int": ctypes.c_int32, "size_t": ctypes.c_size_t, "int64_t": ctypes.c_int64,
               "const char*": ctypes.c_char_p}
    host = set()
    for name, ret, args in protos:
        restype, argtypes = _lib.SIGNATURES[name]
        assert restype is returns[ret], (name, ret, restype)
        assert len(argtypes) == len(args), (name, args, argtypes)
        for decl, t in zip(args, argtypes):
            m = re.fullmatch(r"(?:const )?(\w+)((?:\s*\*\s*(?:const\s*)?)*)\s*(\w+)(\[\d+\])?", decl)
            assert m, (name, decl)
            base, stars, arg, array = m.group(1), m.group(2).count("*"), m.group(3), m.group(4)
            if base in MIRRORS:
                want = ctypes.POINTER(MIRRORS[base])
            elif stars + bool(array) >= 2:
                want = ctypes.POINTER(ctypes.c_void_p)
            elif array or (stars and (arg.endswith("_host") or (name, arg) in HOST_POINTERS)):
                want = ctypes.POINTER(scalars[base])
                host.add((name, arg))
            elif stars:
                want = ctypes.c_void_p
            else:
                want = scalars[base]
            assert t is want, (name, decl, t)
        fn = getattr(lib, name)
        assert fn.restype is restype and list(fn.argtypes) == argtypes, name
    assert HOST_POINTERS <= host


def test_call_appends_the_stream_and_maps_return_codes(monkeypatch):
    """_lib.call against a fake library: the stream goes last, 0 returns, -1 / -2 raise ValueError and a positive
    code NerfB200Error, both with the entry's name and the library's message."""
    class Fake:
        rc = 0
        calls = []

        def nerfb200_embed(self, *args):
            self.calls.append(args)
            return self.rc

        def nerfb200_last_error(self):
            return b"what went wrong"

    fake, stream = Fake(), object()
    monkeypatch.setattr(_lib, "load", lambda: fake)
    monkeypatch.setattr(_lib, "_stream_ptr", lambda: stream)
    assert _lib.call("nerfb200_embed", None, 1, 2.5) is None
    assert _lib.call("nerfb200_embed", torch.device("cuda"), 3) is None      # no index: the current device
    assert fake.calls == [(1, 2.5, stream), (3, stream)]
    for rc in (-1, -2):
        fake.rc = rc
        with pytest.raises(ValueError) as e:
            _lib.call("nerfb200_embed", None, 4)
        assert str(e.value) == "nerfb200_embed: what went wrong"
    fake.rc = 700
    with pytest.raises(_lib.NerfB200Error) as e:
        _lib.call("nerfb200_embed", None, 5)
    assert str(e.value) == "nerfb200_embed: what went wrong (code 700)"
    assert fake.calls[-1] == (5, stream)


def test_entries_are_called_through_lib_call():
    """Only _lib.py picks the stream and maps return codes; every other module goes through _lib.call."""
    pkg = os.path.join(ROOT, "nerf_pl_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py") and fn != "_lib.py":
            src = open(os.path.join(pkg, fn)).read()
            assert "_lib.check(" not in src and ".cuda_stream" not in src, fn


def test_abi_basics(lib):
    assert lib.nerfb200_abi_version() == _lib.ABI_VERSION == 3
    # layout.h: 30 x 32 KiB + 5 x 16 KiB fp16 slices + fp32 tail, rounded to 1 KiB, + 30 backward slices
    fwd = 30 * 32768 + 5 * 16384 + 4 * (9 * 256 + 256 + 4 + 384 + 4 + 28 * 128)
    assert lib.nerfb200_packed_bytes() == (fwd + 1023) // 1024 * 1024 + 30 * 32768
    assert lib.nerfb200_launch_count() >= 0
    # the Python mirrors of the argument structs have the C sizes (x86-64 / aarch64 LP64 layout)
    assert ctypes.sizeof(_lib.RenderArgs) == 8 * 5 + 4 * 2 + 4 + 4 * 2 + 4 * 2 + 4 + 8 * 14 + 8 + 8 * 4 + 8 + 8
    assert ctypes.sizeof(_lib.BackwardArgs) == 8 * 13


def test_struct_mirrors_match_the_header(tmp_path):
    """sizeof / offsetof of the argument structs as gcc lays out include/nerf_pl_b200.h == the ctypes mirrors: four
    offsets of nerfb200_render_args and every field of the two skipping structs."""
    import subprocess
    S, T = _lib.SamplesArgs, _lib.TrainSamplesArgs
    exprs = ["sizeof(nerfb200_render_args)", "sizeof(nerfb200_backward_args)",
             "offsetof(nerfb200_render_args, rng_seed)", "offsetof(nerfb200_render_args, rng_in_kernel)",
             "offsetof(nerfb200_render_args, train_workspace)", "offsetof(nerfb200_render_args, perturb_rand)",
             "sizeof(nerfb200_samples_args)", "sizeof(nerfb200_train_samples_args)"]
    exprs += [f"offsetof(nerfb200_samples_args, {f})" for f, _ in S._fields_]
    exprs += [f"offsetof(nerfb200_train_samples_args, {f})" for f, _ in T._fields_]
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nerf_pl_b200.h"\nint main(void){\n' +
                   "".join(f'printf("%zu\\n", (size_t)({e}));\n' for e in exprs) + "return 0;}\n")
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    R = _lib.RenderArgs
    want = [ctypes.sizeof(R), ctypes.sizeof(_lib.BackwardArgs), R.rng_seed.offset, R.rng_in_kernel.offset,
            R.train_workspace.offset, R.perturb_rand.offset, ctypes.sizeof(S), ctypes.sizeof(T)]
    want += [getattr(S, f).offset for f, _ in S._fields_] + [getattr(T, f).offset for f, _ in T._fields_]
    assert got == want


def _struct_fields(name):
    body = re.search(rf"typedef struct {name} \{{(.*?)\}}", open(HEADER).read(), re.S).group(1)
    return [re.sub(r"\[.*\]", "", ln.strip().rstrip(";")).split()[-1].lstrip("*") for ln in body.splitlines()
            if ln.strip()]


def test_samples_args_fields_mirror_the_header():
    assert _struct_fields("nerfb200_samples_args") == [f for f, _ in _lib.SamplesArgs._fields_]


def test_train_samples_args_fields_mirror_the_header():
    assert _struct_fields("nerfb200_train_samples_args") == [f for f, _ in _lib.TrainSamplesArgs._fields_]


def test_training_workspace_layout(lib):
    """Workspace size is a pure function of the shape: monotone in n_rays, ~9 KiB per ray-sample."""
    b1 = lib.nerfb200_train_workspace_bytes(1024, 64, 64)
    b2 = lib.nerfb200_train_workspace_bytes(2048, 64, 64)
    assert 0 < b1 < b2
    per_sample = (b2 - b1) / (1024 * 192)
    assert 8000 < per_sample < 11000
    assert lib.nerfb200_train_workspace_bytes(0, 64, 64) == 0
    a = _lib.RenderArgs(n_rays=4, n_samples=64, n_importance=0)
    b = _lib.BackwardArgs(render=ctypes.pointer(a))
    assert lib.nerfb200_render_backward(ctypes.byref(b), None) == -1      # NULL rays / tables


def test_argument_validation_without_gpu(lib):
    a = _lib.RenderArgs(n_rays=4, n_samples=48, n_importance=0)
    assert lib.nerfb200_render_rays(ctypes.byref(a), None) == -2          # unsupported N_samples
    assert b"N_samples" in lib.nerfb200_last_error()
    a = _lib.RenderArgs(n_rays=4, n_samples=64, n_importance=64)
    assert lib.nerfb200_render_rays(ctypes.byref(a), None) == -1          # NULL rays
    a = _lib.RenderArgs(n_rays=0, n_samples=64, n_importance=0)
    assert lib.nerfb200_render_rays(ctypes.byref(a), None) == 0           # empty input is a no-op
    assert lib.nerfb200_searchsorted(None, None, None, 3, 2, 4, 4, 1, None) == -1   # row mismatch
    assert lib.nerfb200_searchsorted(None, None, None, 0, 0, 4, 4, 1, None) == 0    # empty
    assert lib.nerfb200_composite(None, None, None, None, None, 0.0, 0, 4, 48, None, None, None, None, None) == -2
    assert lib.nerfb200_nerf_forward(None, 0, 90, None, 0, None, None) == 0
    assert lib.nerfb200_embed(None, 5, 10, None, None) == -1


def test_python_mirror_matches_reference_interface():
    sig = inspect.signature(nb.render_rays)
    names = list(sig.parameters)[:11]
    assert names == ["models", "embeddings", "rays", "N_samples", "use_disp", "perturb", "noise_std",
                     "N_importance", "chunk", "white_back", "test_time"]      # models/rendering.py:58-69
    d = {k: v.default for k, v in sig.parameters.items()}
    assert (d["N_samples"], d["use_disp"], d["perturb"], d["noise_std"], d["N_importance"], d["chunk"],
            d["white_back"], d["test_time"]) == (64, False, 0, 1, 0, 1024 * 32, False, False)
    m = nb.NeRF()
    assert list(m.state_dict().keys()) == orc.PARAM_KEYS                    # models/nerf.py:69-81
    assert sum(p.numel() for p in m.parameters()) == 595844
    e = nb.Embedding(3, 10)
    assert e.out_channels == 63 and nb.Embedding(3, 4).out_channels == 27
    assert torch.equal(e.freq_bands, 2 ** torch.arange(10.0))


def test_no_cpu_fallback():
    m = nb.NeRF()
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    with pytest.raises(RuntimeError):
        nb.render_rays([m, m], emb, torch.zeros(4, 8), 64, False, 0, 0, 64)
    with pytest.raises(RuntimeError):
        m(torch.zeros(2, 90))
    with pytest.raises(RuntimeError):
        emb[0](torch.zeros(2, 3))
    with pytest.raises(RuntimeError):
        nb.searchsorted(torch.zeros(1, 3), torch.zeros(1, 3))


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "nerf_pl_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            src = open(os.path.join(pkg, fn)).read()
            assert "oracle" not in src, fn


def test_nerf_parameters_order_matches_state_dict():
    """The packed-image cache reads the 24 parameters through Module._modules / _parameters
    (hot path of every render_rays call); it must see the state_dict order, for this package's
    NeRF and for a module built the way the reference builds its own (models/nerf.py:58-81)."""
    import torch
    from torch import nn

    from nerf_pl_b200.nerf import NeRF, nerf_parameters

    m = NeRF()
    got = nerf_parameters(m)
    want = [p for _, p in m.named_parameters()]
    assert len(got) == 24 and all(a is b for a, b in zip(got, want))

    class RefLike(nn.Module):            # attribute layout of the reference's NeRF
        def __init__(self):
            super().__init__()
            for i in range(8):
                n_in = 63 if i == 0 else (256 + 63 if i == 4 else 256)
                setattr(self, f"xyz_encoding_{i + 1}", nn.Sequential(nn.Linear(n_in, 256), nn.ReLU(True)))
            self.xyz_encoding_final = nn.Linear(256, 256)
            self.dir_encoding = nn.Sequential(nn.Linear(256 + 27, 128), nn.ReLU(True))
            self.sigma = nn.Linear(256, 1)
            self.rgb = nn.Sequential(nn.Linear(128, 3), nn.Sigmoid())

    r = RefLike()
    got = nerf_parameters(r)
    want = [p for _, p in r.named_parameters()]
    assert len(got) == 24 and all(a is b for a, b in zip(got, want))
    assert [tuple(p.shape) for p in got][:2] == [(256, 63), (256,)]
    del torch


def test_bench_b200_arm_does_not_touch_oracle():
    """Only bench.py's cpu_baseline / --impl reference legs may execute oracle/ (it is the thing
    timed there); the measured arm builds its inputs with bench.py's own generators."""
    import ast

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    tree = ast.parse(open(os.path.join(root, "bench.py")).read())
    fns = {n.name: n for n in tree.body if isinstance(n, ast.FunctionDef)}
    for name in ("run_b200", "synthetic_weights", "blender_rays", "main"):
        src = ast.unparse(fns[name])
        # (run_b200 calls cpu_oracle_throughput(): that IS the cpu_baseline leg)
        assert "import oracle" not in src and "from oracle" not in src and "orc." not in src, name
    top = [n for n in tree.body if isinstance(n, (ast.Import, ast.ImportFrom))]
    assert all("oracle" not in ast.unparse(n) for n in top)


def test_bench_reference_arm_prints_one_json_line():
    """bench.py --impl reference (the CPU arm the driver runs next to the GPU arm): exactly one
    JSON line on stdout with the contract's keys."""
    import json
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "bench.py", "--impl", "reference", "--steps", "1", "--warmup", "1"],
                       cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
              "scaling", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    staged = os.path.exists(os.path.join(root, "oracle", "_ref", "models", "rendering.py"))
    assert d["impl"] == "reference" and d["value"] > 0
    assert d["cpu_baseline"]["kind"] == ("reference" if staged else "port")
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0


def test_integration_md_stub_matches_the_struct():
    """The ctypes stub printed in INTEGRATION.md section 4 is the struct the library takes (names, order, size)."""
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    txt = open(os.path.join(root, "INTEGRATION.md")).read()
    block = txt[txt.index("class RenderArgs(ctypes.Structure):"):txt.index("packed = torch.empty(lib.nerfb200_packed_bytes()")]
    assert re.findall(r'\("(\w+)", ctypes\.c_\w+\)', block) == [f[0] for f in _lib.RenderArgs._fields_]
    ns = {}
    exec("import ctypes\n" + block, ns)
    assert ctypes.sizeof(ns["RenderArgs"]) == ctypes.sizeof(_lib.RenderArgs)
