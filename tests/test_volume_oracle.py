"""The Unity volume (.vol) export without a GPU: the numpy restatement (tests/volume_ref.py) against the reference
notebook's own output (tests/golden/volume_unity.part*.npz, tests/golden/make_volume_golden.py), write_vol's bytes, and
the argument checks of the new C entry points."""
import ctypes

import numpy as np
import pytest

from nerf_pl_b200 import _lib
from nerf_pl_b200.mesh import write_vol
from tests import volume_ref as vr


@pytest.fixture(scope="module")
def golden(golden_dir):
    return vr.load_golden(golden_dir)


def _same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def _within_exp_ulps(a, e64, k=2):
    """a = 1 - e' for an e' within k float32 ulps of the correctly rounded exp term e64."""
    e = np.asarray(e64, np.float32)
    ok = np.zeros(len(e), bool)
    for step in range(-k, k + 1):
        ei = (e.view(np.int32) + step).view(np.float32)
        ok |= _same(np.float32(1) - ei, a)
    return ok


def test_golden_cases_are_what_the_fixture_says(golden):
    cases, meta = golden
    assert set(cases) == {"cube48", "unequal33"}
    for name, c in cases.items():
        N = c["N"]
        assert c["rgbsigma"].shape == (N ** 3, 4) and c["a"].shape == (N ** 3,)
        assert len(c["vol"]) % 8 == 0 and len(c["vol"]) // 8 == meta["cases"][name]["M"] > 0
    assert cases["unequal33"]["ranges"] == [(-1.5, 1.5), (-1.2, 1.4), (-1.5, 1.3)]


@pytest.mark.parametrize("name", ["cube48", "unequal33"])
def test_numpy_exp_choice_reproduces_the_reference_alpha(golden, name):
    cases, meta = golden
    c = cases[name]
    a = vr.alpha(c["rgbsigma"][:, 3], c["ranges"][0], c["N"], exp="numpy")
    diff = ~_same(a, c["a"])
    print(f"\n{name}: local numpy {np.__version__} SIMD {vr.numpy_simd()}; fixture numpy {meta['numpy']} SIMD "
          f"{meta['simd']}; {int(diff.sum())} of {len(a)} alphas differ")
    if diff.any():
        # np.exp on float32 is not correctly rounded and its last bits follow the SIMD path numpy dispatches to:
        # a difference is only acceptable from a machine that dispatches differently, and only by an ulp or two of exp
        assert (vr.numpy_simd(), np.__version__) != (meta["simd"], meta["numpy"]), np.nonzero(diff)[0][:10]
        e64 = vr.exp_term(c["rgbsigma"][:, 3], c["ranges"][0], c["N"], exp="f64")
        assert _within_exp_ulps(a[diff], e64[diff]).all() and _within_exp_ulps(c["a"][diff], e64[diff]).all()


@pytest.mark.parametrize("name", ["cube48", "unequal33"])
def test_reference_alpha_is_within_two_ulps_of_the_correctly_rounded_one(golden, name):
    c = golden[0][name]
    a64 = vr.alpha(c["rgbsigma"][:, 3], c["ranges"][0], c["N"], exp="f64")
    diff = ~_same(a64, c["a"])
    print(f"\n{name}: {int(diff.sum())} of {len(a64)} reference alphas differ from the correctly rounded ones")
    e64 = vr.exp_term(c["rgbsigma"][:, 3], c["ranges"][0], c["N"], exp="f64")
    assert _within_exp_ulps(c["a"][diff], e64[diff]).all()


@pytest.mark.parametrize("name", ["cube48", "unequal33"])
def test_golden_file_equals_the_oracle_except_where_exp_rounds_differently(golden, name, tmp_path):
    c = golden[0][name]
    ref_rows = vr.unpack(c["vol"])
    # the restatement's packing, fed the reference's own alpha, writes the reference's file byte for byte
    assert vr.vol_bytes(vr.pack(c["rgbsigma"], c["a"])) == c["vol"]
    # with the correctly rounded exp, rows differ only at points whose reference alpha is not the correctly rounded one
    a64 = vr.alpha(c["rgbsigma"][:, 3], c["ranges"][0], c["N"], exp="f64")
    amb = ~_same(a64, c["a"])
    ours = vr.pack_volume(c["rgbsigma"], c["ranges"][0], exp="f64")
    path = tmp_path / f"{name}.vol"
    write_vol(str(path), ours)
    assert path.read_bytes() == vr.vol_bytes(ours)
    keep_ref, keep_ours = ~amb[ref_rows[:, 0]], ~amb[ours[:, 0]]
    print(f"\n{name}: {len(ref_rows)} reference rows, {len(ours)} oracle rows, {int(amb.sum())} points with a "
          f"differently rounded alpha ({int((~keep_ref).sum())} / {int((~keep_ours).sum())} rows)")
    assert np.array_equal(ref_rows[keep_ref], ours[keep_ours])
    # at those points: the same kept set up to points at the a > 0 edge, the same rgb, a8 within one
    common, ir, io = np.intersect1d(ref_rows[:, 0], ours[:, 0], return_indices=True)
    only = np.setxor1d(ref_rows[:, 0], ours[:, 0])
    assert amb[only].all()
    sr, so = ref_rows[ir, 1].astype(np.int64), ours[io, 1].astype(np.int64)
    assert np.array_equal(sr >> 8, so >> 8) and np.abs((sr & 255) - (so & 255)).max(initial=0) <= 1
    print(f"  {len(only)} rows kept by one side only, {int(((sr & 255) != (so & 255)).sum())} a8 differ by one")
    if not amb.any():
        assert path.read_bytes() == c["vol"]


def test_alpha_edges():
    N, xr = 512, (-1.2, 1.2)
    s = np.float32([-1.0, -0.0, 0.0, np.inf, np.nan, -np.inf, 1e30])
    a = vr.alpha(s, xr, N)
    assert a[0] == 0 and a[1] == 0 and a[2] == 0 and a[3] == 1 and np.isnan(a[4]) and a[5] == 0 and a[6] == 1
    # the scale is rounded to float32 before the multiply (fl32(fl32(c) sigma), not fl32(c sigma))
    c = -2.4 / 512
    sig = np.float32(np.arange(1, 20001, dtype=np.float32) * np.float32(0.37))
    x_cell = vr.scale(xr, N) * sig
    x_once = (c * sig.astype(np.float64)).astype(np.float32)
    assert (x_cell != x_once).any()
    # a reversed x_range gives a <= 0 everywhere: nothing is kept
    g = np.zeros((8 ** 3, 4), np.float32)
    g[:, 3] = np.linspace(-5, 1e4, 8 ** 3)
    assert len(vr.pack_volume(g, (1.0, -1.0))) == 0
    # the smallest sigma with a > 0 and its predecessor
    sm = vr.smallest_positive_alpha_sigma(xr, N)
    assert vr.alpha(sm, xr, N)[0] > 0 and vr.alpha(np.nextafter(sm, np.float32(0)), xr, N)[0] == 0
    # +inf packs to a8 = 255, rgb 1 to 255
    g = np.zeros((2 ** 3, 4), np.float32)
    g[3] = [1, 0, 1, np.inf]
    assert vr.pack_volume(g, xr).tolist() == [[3, (255 << 24) + (255 << 8) + 255]]


def test_volume_entry_points_reject_bad_arguments_without_a_device():
    _lib.build()
    lib = _lib.load()
    assert lib.nerfb200_volume_workspace_bytes(1) == 0
    assert lib.nerfb200_volume_workspace_bytes(1626) == 0
    assert lib.nerfb200_volume_workspace_bytes(2) > 0
    cnt = ctypes.c_int64(-7)
    fake = 1 << 20                                    # never dereferenced: every call fails its checks first
    big = 1 << 40
    for N in (1, 0, -3, 1626, 1 << 20):
        assert lib.nerfb200_volume_count(fake, N, -1.0, 1.0, fake, big, ctypes.byref(cnt), None) == -1
        assert lib.nerfb200_volume_emit(fake, N, -1.0, 1.0, fake, big, fake, None) == -1
    assert b"1625" in lib.nerfb200_last_error()
    assert lib.nerfb200_volume_count(None, 8, -1.0, 1.0, fake, big, ctypes.byref(cnt), None) == -1
    assert lib.nerfb200_volume_count(fake, 8, -1.0, 1.0, None, big, ctypes.byref(cnt), None) == -1
    assert lib.nerfb200_volume_count(fake, 8, -1.0, 1.0, fake, big, None, None) == -1
    assert lib.nerfb200_volume_count(fake + 4, 8, -1.0, 1.0, fake, big, ctypes.byref(cnt), None) == -1   # alignment
    assert lib.nerfb200_volume_count(fake, 8, -1.0, 1.0, fake, 16, ctypes.byref(cnt), None) == -1       # workspace
    assert b"workspace" in lib.nerfb200_last_error()
    assert lib.nerfb200_volume_emit(fake, 8, -1.0, 1.0, fake, 16, fake, None) == -1
    assert lib.nerfb200_volume_emit(fake, 8, -1.0, 1.0, fake, big, None, None) == -1
    assert lib.nerfb200_volume_emit(fake, 8, -1.0, 1.0, fake, big, fake + 4, None) == -1
    assert cnt.value == -7
    rng = (ctypes.c_double * 6)(-1, 1, -1, 1, -1, 1)
    for N in (1, 1626):
        assert lib.nerfb200_rgb_sigma_grid(fake, N, rng, 1024, fake, big, fake, None) == -1
    assert lib.nerfb200_rgb_sigma_grid(fake, 8, rng, 0, fake, big, fake, None) == -1
    assert lib.nerfb200_rgb_sigma_grid(None, 8, rng, 64, fake, big, fake, None) == -1
    assert lib.nerfb200_rgb_sigma_grid(fake, 8, None, 64, fake, big, fake, None) == -1
    assert lib.nerfb200_rgb_sigma_grid(fake, 8, rng, 64, fake, big, fake + 4, None) == -1
    assert lib.nerfb200_rgb_sigma_grid(fake, 8, rng, 64, fake, 4, fake, None) == -1
    assert lib.nerfb200_query_rgb_sigma(None, 5, 3, fake, fake, None) == -1
    assert lib.nerfb200_query_rgb_sigma(fake, 5, 2, fake, fake, None) == -1
    assert lib.nerfb200_query_rgb_sigma(fake, 5, 3, fake, fake + 4, None) == -1
    assert lib.nerfb200_query_rgb_sigma(fake, -1, 3, fake, fake, None) == -1
    assert lib.nerfb200_query_rgb_sigma(None, 0, 3, None, None, None) == 0      # empty input is a no-op
