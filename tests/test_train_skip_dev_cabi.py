"""The capturable entries of include/nerf_pl_b200.h (nerfb200_train_samples_forward_dev / _backward_dev):
their declarations, and the argument errors they return before any launch, as tests/test_train_skip_cabi.py checks
the eager entries."""
import ctypes
import re

import pytest
import torch

from nerf_pl_b200 import _lib

from .test_cabi import HEADER
from .test_train_skip_cabi import BAD, _args

DEV_ENTRIES = ("nerfb200_train_samples_forward_dev", "nerfb200_train_samples_backward_dev")


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


def test_capturable_entries_are_declared_in_the_one_header():
    hdr = open(HEADER).read()
    for name in DEV_ENTRIES:
        assert re.search(rf"\bint {name}\(", hdr), name
        assert name in _lib.SIGNATURES
    fwd = _lib.SIGNATURES["nerfb200_train_samples_forward_dev"][1]
    assert fwd[3] is ctypes.POINTER(ctypes.c_int64)           # live_samples_dev: a device int64[2]
    bwd = _lib.SIGNATURES["nerfb200_train_samples_backward_dev"][1]
    assert len(bwd) == 9 and ctypes.POINTER(ctypes.c_int64) not in bwd     # no host counts
    # the eager entries keep their signatures
    assert _lib.SIGNATURES["nerfb200_train_samples_forward"][1][3] is ctypes.POINTER(ctypes.c_int64)
    assert len(_lib.SIGNATURES["nerfb200_train_samples_backward"][1]) == 10


def test_capturable_entries_argument_checks(lib):
    """Every malformed argument the eager entries refuse, the capturable ones refuse with the same message."""
    live = ctypes.cast(ctypes.c_void_p(256), ctypes.POINTER(ctypes.c_int64))
    for bad, msg in BAD:
        a = _args(**bad)
        rc = lib.nerfb200_train_samples_forward_dev(ctypes.byref(a), ctypes.c_void_p(1024), 0, live, None)
        assert rc in (-1, -2) and msg in lib.nerfb200_last_error(), (bad, rc, lib.nerfb200_last_error())
        rc = lib.nerfb200_train_samples_backward_dev(ctypes.byref(a), ctypes.c_void_p(1024), 0, None, None, None,
                                                     None, None, None)
        assert rc in (-1, -2) and msg in lib.nerfb200_last_error(), (bad, rc, lib.nerfb200_last_error())
    assert lib.nerfb200_train_samples_forward_dev(ctypes.byref(_args()), ctypes.c_void_p(1024), 0, None, None) == -1
    assert b"NULL" in lib.nerfb200_last_error()


def test_capturable_backward_needs_both_tables(lib):
    """The capturable backward writes every network's gradients, so a missing table is refused even though the
    eager backward accepts one for a network with no evaluated sample."""
    big = lib.nerfb200_train_samples_workspace_bytes(4, 64, 64)
    ws = ctypes.c_void_p(1 << 20)                   # never dereferenced: the checks come first
    p = (ctypes.c_void_p * 24)(*([256] * 24))
    for tables in ((None, p, p, p), (p, None, p, p), (p, p, None, p), (p, p, p, None)):
        rc = lib.nerfb200_train_samples_backward_dev(ctypes.byref(_args()), ws, big, None, *tables, None)
        assert rc == -1 and b"NULL" in lib.nerfb200_last_error(), tables
    holes = (ctypes.c_void_p * 24)(*([256] * 23 + [None]))
    rc = lib.nerfb200_train_samples_backward_dev(ctypes.byref(_args()), ws, big, None, p, p, holes, p, None)
    assert rc == -1 and b"NULL" in lib.nerfb200_last_error()


def test_python_capturable_mode_checks_the_count_tensor():
    from nerf_pl_b200 import train_skip
    rays = torch.zeros(4, 8, device="meta")
    for bad in (torch.zeros(2, dtype=torch.int32, device="meta"), torch.zeros(3, dtype=torch.int64, device="meta"),
                torch.zeros(2, dtype=torch.int64)):
        with pytest.raises(ValueError, match="live_samples"):
            train_skip.render_rays_train_skip([], rays, 64, False, 0.0, 0.0, 64, False, None, None, None, None,
                                              torch.zeros(4, 3, device="meta"), None, live_samples=bad)

