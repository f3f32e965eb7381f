"""tests/units_ref.py without a GPU: the emulations and float64 restatements against the oracle and the reference's
goldens, each comparator against the defect it exists for, and the argument checks the Python wrappers make before
anything is launched."""
import os

import numpy as np
import pytest
import torch

import nerf_pl_b200 as nb
from oracle import nerf_oracle as orc
from tests import cases
from tests import render_tape as rt
from tests import units_ref as ur

F32, F64 = np.float32, np.float64


def _raygen():
    g = np.load(os.path.join(cases.GOLDEN, "raygen.npz"))
    return g, int(g["H"]), int(g["W"]), float(g["focal"])


# ------------------------------------------------------------------------------------------------ generate_rays
@pytest.mark.parametrize("ndc", [False, True])
def test_ray_emulation_against_the_reference_golden_and_float64(ndc):
    """The reference's own rays (torch fp32, another matmul order) and the emulation lie within the same few ulps of
    float64 (with the double focal the reference holds); the emulation's NDC rays need its float32 sx, sy."""
    g, H, W, f = _raygen()
    emu = ur.generate_rays32(H, W, f, g["c2w"], 2.0, 6.0, ndc)
    gold = g["ndc" if ndc else "blender"]
    r64, sc = ur.generate_rays64(H, W, f, g["c2w"], 2.0, 6.0, ndc)
    e_emu, e_gold = ur.ray_ulps(emu, r64, sc).max(), ur.ray_ulps(gold, r64, sc).max()
    print(f"\nrays ndc {ndc}: emulation {e_emu:.3g} ulp, reference {e_gold:.3g} ulp of float64")
    bar = 16.0 if ndc else 4.0
    assert e_emu <= bar and e_gold <= bar
    assert ur.bitwise_differ(emu[:, 6:], gold[:, 6:]) == 0
    if not ndc:
        assert ur.bitwise_differ(emu[:, :3], gold[:, :3]) == 0                 # the origin is c2w[:, 3]
    else:
        assert ur.bitwise_differ(emu, ur.generate_rays32(H, W, f, g["c2w"], 2.0, 6.0, True, "sx_f64")) > 0


def test_ray_emulation_edges():
    """1 x 1 and odd sizes (W / 2 = x.5): the pixel direction is exact where it must be."""
    c2w = np.concatenate([np.eye(3), np.zeros((3, 1))], 1).astype(F32)
    r = ur.generate_rays32(1, 1, 2.0, c2w, 2.0, 6.0)
    d = np.array([-0.25, 0.25, -1.0]) / np.sqrt(1.125)
    assert np.all(np.abs(r[0, 3:6] - d) <= 2 * ur.ulp32(d))                  # sqrt and divide: one rounding each
    r = ur.generate_rays32(3, 5, 1.0, c2w, 2.0, 6.0)
    dx = (np.arange(5) - 2.5) / 1.0
    assert np.all(np.sign(r.reshape(3, 5, 8)[0, :, 3]) == np.sign(dx))


def test_bitwise_comparator_rejects_one_ulp():
    g, H, W, f = _raygen()
    emu = ur.generate_rays32(H, W, f, g["c2w"], 2.0, 6.0)
    bad = emu.copy()
    bad[123, 4] = np.nextafter(bad[123, 4], F32(np.inf))
    assert ur.bitwise_differ(bad, emu) == 1
    zero = np.zeros((1, 8), F32)
    assert ur.bitwise_differ(-zero, zero) == 8                                 # -0.0 is not +0.0
    nan = emu.copy()
    nan[0, 0] = np.nan
    assert ur.bitwise_differ(nan, nan.copy()) == 0


# ------------------------------------------------------------------------------------------------ sample_pdf
def test_standalone_emulation_against_the_reference_golden():
    """units.npz holds the reference's own sample_pdf (det and with u); the emulation agrees with it except where
    sample_pdf64 says fp32 may pick another bin, and is within the float64 bar elsewhere."""
    u = np.load(os.path.join(cases.GOLDEN, "units.npz"))
    bins, w = u["pdf_bins"], u["pdf_weights"]
    for K, uu, ref in ((64, np.broadcast_to(orc.linspace01(64), (len(w), 64)), u["pdf_det"]),
                       (48, u["pdf_u"], u["pdf_rand"])):
        emu = rt.inverse_cdf(rt.cdf_standalone(w), bins, uu)
        z64, flagged, bar = rt.sample_pdf64(bins, w, uu, sequential=True)
        ok = ~flagged
        assert np.all(np.abs(emu[ok] - z64[ok]) <= bar[ok])
        assert np.all(np.abs(ref[ok] - z64[ok]) <= bar[ok])


def test_sample_pdf_edges_in_the_emulation():
    nw = 62
    rs = np.random.RandomState(4)
    w = rs.dirichlet(np.ones(nw) * 0.5, 64).astype(F32) * F32(2.7)
    cdf = rt.cdf_standalone(w)
    assert (cdf[:, -1] != 1).any()                                  # cdf[-1] != 1 occurs
    z = rt.inverse_cdf(np.zeros((1, nw + 1), F32) + rt.cdf_standalone(np.zeros((1, nw), F32)),
                       np.arange(nw + 1, dtype=F32)[None], np.array([[0.0, 0.5, 1.0]], F32))
    np.testing.assert_allclose(z[0], [0.0, nw / 2, nw], atol=1e-4)  # all-zero weights: uniform
    bins = np.sort(rs.uniform(2, 6, (64, nw + 1)), 1).astype(F32)
    k = rs.randint(0, nw, 64)
    on = cdf[np.arange(64), k][:, None]
    np.testing.assert_array_equal(rt.inverse_cdf(cdf, bins, on)[:, 0], bins[np.arange(64), k])   # u on a knot


def _pdf_defects(w, bins, u):
    """A neighbouring bin and a cdf built in another order (numpy's cumsum of the whole pdf)."""
    cdf = rt.cdf_standalone(w)
    good = rt.inverse_cdf(cdf, bins, u)
    nw = w.shape[1]
    lo = rt.search_right(cdf, u)
    below = np.clip(lo - 1 + 1, 0, nw)
    above = np.clip(lo + 1, 0, nw)
    rows = np.arange(len(w))[:, None]
    c0, c1 = cdf[rows, below], cdf[rows, above]
    den = np.where((c1 - c0).astype(F32) < rt.EPS_W, F32(1), (c1 - c0).astype(F32))
    neighbour = (bins[rows, below] + (((u - c0).astype(F32) / den).astype(F32)
                                      * (bins[rows, above] - bins[rows, below]).astype(F32)).astype(F32)).astype(F32)
    wp = (w + rt.EPS_W).astype(F32)
    other = np.concatenate([np.zeros((len(w), 1), F32),
                            np.cumsum((wp / wp.sum(1, keepdims=True, dtype=F32)).astype(F32), 1, dtype=F32)], 1)
    return good, {"neighbouring_bin": neighbour, "cdf_order": rt.inverse_cdf(other, bins, u)}


def test_sample_pdf_comparators_reject_each_defect():
    rs = np.random.RandomState(8)
    nw, K = 1000, 64
    w = rs.dirichlet(np.ones(nw) * 0.5, 16).astype(F32)
    bins = np.sort(rs.uniform(2, 6, (16, nw + 1)), 1).astype(F32)
    u = rs.rand(16, K).astype(F32)
    good, bad = _pdf_defects(w, bins, u)
    z64, flagged, bar = rt.sample_pdf64(bins, w, u, sequential=True)
    assert ur.bitwise_differ(good, good) == 0 and not (~(np.abs(good - z64) <= bar) & ~flagged).any()
    for name, z in bad.items():
        assert ur.bitwise_differ(z, good) > 0, name
    z = bad["neighbouring_bin"]
    assert (~(np.abs(z - z64) <= bar) & ~flagged).any()           # float64 sees a wrong bin too


# ------------------------------------------------------------------------------------------------ mse / psnr
@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 5000])
def test_mse_emulation_against_float64_and_the_oracle(n):
    rs = np.random.RandomState(n)
    t = rs.rand(n, 3).astype(F32)
    rc = (t + rs.randn(n, 3).astype(F32) * F32(0.1)).astype(F32)
    rf = (t + rs.randn(n, 3).astype(F32) * F32(0.01)).astype(F32)
    mc, mf, tot, fin = ur.mse_psnr32(rc, rf, t)
    for m, x in ((mc, rc), (mf, rf)):
        m64 = ur.mse64(x, t)
        assert abs(float(m) - m64) <= float(ur.ulp32(m64))        # the double sum is all but exact: one rounding
    assert tot == F32(mc + mf) and fin == mf
    ps = -10 * np.log10(float(fin))
    assert abs(ps - orc.psnr(rf, t)) <= ur.psnr_bar(fin, ps)
    assert ur.mse_psnr32(rc, None, t)[1] == 0 and ur.mse_psnr32(rc, None, t)[3] == mc
    assert ur.mse_psnr32(t, t, t)[3] == 0


def test_mse_comparator_rejects_another_order():
    """The fp32 order the kernel does not use (one float32 running sum) moves the mse by ulps: the bitwise pin sees
    it."""
    rs = np.random.RandomState(1)
    n = 40000
    t = rs.rand(n, 3).astype(F32)
    rc = (t + rs.randn(n, 3).astype(F32) * F32(0.1)).astype(F32)
    mc = ur.mse_psnr32(rc, None, t)[0]
    d = (rc - t).astype(F32).reshape(-1)
    run = F32(0)
    for x in (d * d).astype(F32):
        run = F32(run + x)
    assert F32(run / F32(3 * n)) != mc


# ------------------------------------------------------------------------------------------------ searchsorted
def test_oracle_searchsorted_follows_the_reference_comparisons():
    """orc.searchsorted against a restatement of torchsearchsorted's CUDA search on ties, +-0, +-inf and NaN: equal
    everywhere except that search's own slip (rows of 1 or 2 columns, 'left', v == a[-1]), which returns ncol where
    a count of a < v gives ncol - 1."""
    a = np.array([-np.inf, -1, -0.0, 0.0, 0.0, 1, 1, 2, np.inf], F32)
    v = np.array([np.nan, -np.inf, -1, -0.0, 0.0, 0.5, 1, 2, np.inf, 3, -7], F32)
    for side in ("left", "right"):
        np.testing.assert_array_equal(orc.searchsorted(a[None], v[None], side)[0], ur.searchsorted_bisect(a, v, side))
    rs = np.random.RandomState(0)
    for ncol in (3, 4, 7, 50):
        for _ in range(20):
            row = np.sort(np.round(rs.randn(ncol), 0)).astype(F32)
            vv = np.concatenate([row, rs.choice(row, 5), [np.nan, 0.0, -0.0, np.inf, -np.inf]]).astype(F32)
            for side in ("left", "right"):
                np.testing.assert_array_equal(orc.searchsorted(row[None], vv[None], side)[0],
                                              ur.searchsorted_bisect(row, vv, side))
    for ncol in (1, 2):
        row = np.arange(1, ncol + 1, dtype=F32)
        assert ur.searchsorted_bisect(row, row[-1:], "left")[0] == ncol
        assert orc.searchsorted(row[None], row[None, -1:], "left")[0, 0] == ncol - 1
    assert orc.searchsorted(a[None], np.full((3, 2), np.nan, F32), "right").sum() == 0    # broadcast rows


# ------------------------------------------------------------------------------------------------ Embedding
def test_embed_comparator_rejects_swapped_sin_cos_and_a_wrong_frequency():
    rs = np.random.RandomState(2)
    x = (rs.uniform(-1, 1, (300, 3)) * 10.0 ** rs.uniform(-3, 4, (300, 1))).astype(F32)
    ref = ur.embed64(x, 10)
    good = ref.astype(F32)                                            # correctly rounded: 0.5 ulp
    assert ur.embed_ulps(good[:, 3:], ref[:, 3:]).max() <= 0.5
    swapped = good.copy().reshape(300, 1 + 2 * 10, 3)
    swapped[:, 1::2], swapped[:, 2::2] = good.reshape(300, 21, 3)[:, 2::2], good.reshape(300, 21, 3)[:, 1::2]
    assert ur.embed_ulps(swapped.reshape(300, 63)[:, 3:], ref[:, 3:]).max() > ur.EMBED_ULPS
    shifted = ur.embed64(x, 11)[:, np.r_[0:3, 9:69]].astype(F32)     # frequencies 2^(k+1)
    assert ur.embed_ulps(shifted[:, 3:], ref[:, 3:]).max() > ur.EMBED_ULPS
    specials = np.array([[np.inf, np.nan, -0.0]], F32)
    r = ur.embed64(specials, 2)
    assert np.isnan(r[0, 3:5]).all() and np.signbit(r[0, 5]) and r[0, 8] == 1.0


def test_embed_restatement_against_the_reference_golden():
    u = np.load(os.path.join(cases.GOLDEN, "units.npz"))
    for key, x, k in (("embed10", u["x3"], 10), ("embed4", (u["x3"] / F32(6)).astype(F32), 4)):
        e = ur.embed_ulps(u[key][:, 3:], ur.embed64(x, k)[:, 3:])
        print(f"\nreference {key}: worst {e.max():.3g} ulp of float64")
        assert e.max() <= ur.EMBED_ULPS


# ------------------------------------------------------------------------------------------------ packed image
@pytest.mark.parametrize("kind", ["random", "trained"])
def test_pack_restatement_passes_its_comparator(kind):
    ws = cases.trained_weights() if kind == "trained" else cases.weights()
    rep = ur.check_packed(ur.pack_image(ws[0]), ws[0])
    assert rep["plain_differ"] == 0 and rep["fold_outside"] == 0 and rep["fold_twins_differ"] == 0, rep
    assert rep["fold_worst"] <= 1.0


@pytest.mark.parametrize("defect", ur.PACK_DEFECTS)
def test_pack_comparator_rejects_each_defect(defect):
    w = cases.weights()[0]
    rep = ur.check_packed(ur.pack_image(w, defect), w)
    assert rep["plain_differ"] + rep["fold_outside"] + rep["fold_twins_differ"] > 0, (defect, rep)


def test_pack_layout_sizes():
    assert ur.PACKED_BYTES == 2_074_624 and ur.HALF_BYTES == 1_064_960 and ur.OFF_BWD % 1024 == 0
    n, k = np.meshgrid(np.arange(256), np.arange(64), indexing="ij")
    offs = ur.sw128_off(n, k)
    assert len(np.unique(offs)) == 256 * 64 and offs.max() == 256 * 128 - 2     # a permutation of the slice


# ------------------------------------------------------------------------------------------------ argument checks
def _raises(fn, match):
    """The call raises ValueError with `match` in its message (anything else fails the assertion)."""
    try:
        fn()
    except Exception as e:          # noqa: BLE001 - the type is part of what is checked
        assert type(e) is ValueError and match in str(e), f"{type(e).__name__}: {e}"
        return
    raise AssertionError("no exception")


def test_sample_pdf_checks_shapes_before_any_launch():
    """CPU tensors: a check that ran after the device check would raise RuntimeError instead."""
    b, w = torch.zeros(5, 9), torch.zeros(5, 8)
    _raises(lambda: nb.sample_pdf(b, w, 16, u=torch.zeros(5, 15)), "u must be (N_rays, N_importance)")
    _raises(lambda: nb.sample_pdf(b, w, 16, u=torch.zeros(4, 16)), "u must be (N_rays, N_importance)")
    _raises(lambda: nb.sample_pdf(b, w, 16, u=torch.zeros(80)), "u must be (N_rays, N_importance)")
    _raises(lambda: nb.sample_pdf(torch.zeros(5, 8), w, 16), "bins must be")
    _raises(lambda: nb.sample_pdf(b, torch.zeros(40), 16), "weights must be")


def test_volume_render_checks_shapes_before_any_launch():
    n, S = 4, 32
    s, z, d = torch.zeros(n, S), torch.zeros(n, S), torch.zeros(n, 3)
    rgb = torch.zeros(n, S, 3)
    _raises(lambda: nb.volume_render(s, torch.zeros(n, S, 4), z, d), "rgbs must be")
    _raises(lambda: nb.volume_render(s, torch.zeros(n - 1, S, 3), z, d), "rgbs must be")
    _raises(lambda: nb.volume_render(s, rgb, torch.zeros(n, S - 32), d), "z_vals must be")
    _raises(lambda: nb.volume_render(s, None, z, torch.zeros(n + 1, 3)), "dirs must be")
    _raises(lambda: nb.volume_render(s, rgb, z, d, torch.zeros(n, S + 1), 1.0), "noise must be")
    _raises(lambda: nb.volume_render(torch.zeros(n * S), rgb, z, d), "sigmas must be")


def test_mse_psnr_checks_shapes_before_any_launch():
    t = torch.zeros(10, 3)
    _raises(lambda: nb.mse_psnr({"rgb_coarse": torch.zeros(10, 3), "rgb_fine": torch.zeros(9, 3)}, t),
            "rgb_fine must have the shape of targets")
    _raises(lambda: nb.mse_psnr({"rgb_coarse": torch.zeros(11, 3)}, t), "rgb_coarse must have the shape of targets")
    _raises(lambda: nb.mse_psnr({"rgb_coarse": torch.zeros(30)}, torch.zeros(30)), "targets must be (N_rays, 3)")
