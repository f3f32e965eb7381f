"""The resampling emulation and float64 references of tests/render_tape.py, without a GPU.

Hand cases pin the emulation's exact output where it is known in closed form; a scalar lane-by-lane replica of
pdf_to_cdf_ray pins the vectorised one at per = 1, 2 and 4 samples per lane; the emulation agrees with the fp32
oracle (whose cumsum runs in another order) except where float64 says fp32 may legitimately differ; and each defect
of DEFECTS injected into the emulation is rejected by the comparator tests/test_gpu_render_stages.py applies to
the device's depths."""
import numpy as np
import pytest

from oracle import nerf_oracle as orc
from tests import render_tape as rt

F32, F64 = np.float32, np.float64


def _cdf_scalar(w):
    """pdf_to_cdf_ray of ONE ray, lane by lane and shuffle by shuffle with float32 scalars."""
    S = len(w)
    nw = S - 2
    w = [F32(x) for x in w]
    part = [F32(0)] * 32
    for lane in range(32):
        for i in range(lane, nw, 32):
            part[lane] = F32(part[lane] + F32(w[1 + i] + F32(1e-5)))
    for o in (16, 8, 4, 2, 1):
        part = [F32(part[l] + part[l ^ o]) for l in range(32)]
    total = part[0]
    per = (nw + 31) >> 5
    loc = [[F32(0)] * per for _ in range(32)]
    run = [F32(0)] * 32
    for lane in range(32):
        for p in range(per):
            i = lane * per + p
            pdf = F32(F32(w[1 + i] + F32(1e-5)) / total) if i < nw else F32(0)
            run[lane] = F32(run[lane] + pdf)
            loc[lane][p] = run[lane]
    incl = list(run)
    for o in (1, 2, 4, 8, 16):
        incl = [F32(incl[l] + incl[l - o]) if l >= o else incl[l] for l in range(32)]
    cdf = np.zeros(S - 1, F32)
    for lane in range(32):
        excl = incl[lane - 1] if lane else F32(0)
        for p in range(per):
            i = lane * per + p
            if i < nw:
                cdf[i + 1] = F32(excl + loc[lane][p])
    return cdf


def _weights(kind, R, S, seed):
    rs = np.random.RandomState(seed)
    if kind == "random":
        return rs.dirichlet(np.ones(S) * 0.5, R).astype(F32)
    # trained-like: a sharp surface, empty space elsewhere (exact zeros and 1e-9-level residue); opaque rays (an
    # empty bin's pdf 1e-5 / (1 + nw 1e-5) is just under the threshold) and every other ray semi-transparent
    w = np.where(rs.rand(R, S) < 0.5, 0.0, rs.rand(R, S) * 1e-9)
    c = rs.randint(2, S - 4, R)
    for r in range(R):
        w[r, c[r]:c[r] + 3] = rs.dirichlet(np.ones(3)) * (1.0 if r % 2 == 0 else rs.uniform(0.5, 1.0))
    return w.astype(F32)


def _depths(R, S, seed):
    rs = np.random.RandomState(seed)
    rays = orc.make_rays(R, seed)
    return orc.coarse_depths(rays, S, False, 1.0, rs.rand(R, S).astype(F32))


# ------------------------------------------------------------------------------------------ hand cases
@pytest.mark.parametrize("S", [32, 64, 128])
@pytest.mark.parametrize("kind", ["random", "trained"])
def test_cdf_matches_the_scalar_lane_replica(S, kind):
    """nw = 30, 62, 126: per = 1, 2, 4 samples per lane (the last lane partly or wholly empty)."""
    w = _weights(kind, 6, S, S)
    got = rt.cdf_fused(w)
    for r in range(len(w)):
        np.testing.assert_array_equal(got[r], _cdf_scalar(w[r]))


def test_zero_weights_give_a_uniform_cdf():
    for S in (32, 64, 128):
        nw = S - 2
        cdf = rt.cdf_fused(np.zeros((1, S), F32))[0]
        assert cdf[0] == 0 and np.all(np.diff(cdf) > 0)
        np.testing.assert_allclose(cdf, np.arange(nw + 1) / nw, rtol=0, atol=8 * 2.0 ** -24)
        # linspace u on a uniform cdf over evenly spaced bins: the identity map up to the lerp's roundings
        zc = rt.linspace01(S)[None, :] * F32(4) + F32(2)
        u = rt.linspace01(64)[None, :]
        z = rt.inverse_cdf(cdf[None, :], rt.bins_from_depths(zc), u)[0]
        b = rt.bins_from_depths(zc)[0]
        np.testing.assert_allclose(z, b[0] + u[0] * (b[-1] - b[0]), rtol=0, atol=1e-5)


def test_one_hot_weights_take_the_denom_branch():
    S, j = 64, 20
    w = np.zeros((1, S), F32)
    w[0, 1 + j] = 1                       # pdf index j: the jump cdf[j] -> cdf[j + 1]
    cdf = rt.cdf_fused(w)
    bins = rt.bins_from_depths(_depths(1, S, 3))
    d = np.diff(cdf[0])
    # below the jump every bin is under the threshold; above it (cdf near 1, ulp 6e-8) rounding puts the
    # differences on both sides of 1e-5: the conditioning sample_pdf64 flags
    assert np.all(d[:j] < 1e-5) and d[j] > 0.99
    assert (d[j + 1:] < 1e-5).any() and (d[j + 1:] >= 1e-5).any()
    u = np.array([[0.0, 0.5 * cdf[0, 5], cdf[0, j] * F32(0.999), 0.5, 0.9]], F32)
    z = rt.inverse_cdf(cdf, bins, u)[0]
    for k in range(3):                    # empty space: denom -> 1, z = b0 + (u - c0) (b1 - b0), a hair above b0
        lo = int(np.searchsorted(cdf[0], u[0, k], side="right"))
        b0, b1, c0 = bins[0, lo - 1], bins[0, lo], cdf[0, lo - 1]
        assert z[k] == F32(b0 + F32(F32(u[0, k] - c0) * F32(b1 - b0)))
        assert b0 <= z[k] < b0 + 1e-4 * (b1 - b0)
    assert np.all((z[3:] >= bins[0, j]) & (z[3:] <= bins[0, j + 1]))     # the surface bin


def test_u_on_a_knot_takes_the_right_side_and_the_end_points():
    S = 64
    w = _weights("random", 4, S, 5)
    cdf = rt.cdf_fused(w)
    bins = rt.bins_from_depths(_depths(4, S, 5))
    k = np.array([3, 17, 40, 61])
    u = cdf[np.arange(4), k][:, None]
    z = rt.inverse_cdf(cdf, bins, u)[:, 0]
    np.testing.assert_array_equal(z, bins[np.arange(4), k])          # below = k, t = 0: exactly bin k
    z0 = rt.inverse_cdf(cdf, bins, np.zeros((4, 1), F32))[:, 0]
    np.testing.assert_array_equal(z0, bins[:, 0])
    z1 = rt.inverse_cdf(cdf, bins, np.ones((4, 1), F32))[:, 0]
    for r in range(4):
        if cdf[r, -1] <= 1:           # searchsorted(right) = nw + 1: both clamps on the last bin
            assert z1[r] == bins[r, -1]
        else:
            assert bins[r, -2] <= z1[r] <= bins[r, -1]


def test_standalone_cdf_is_sequential():
    w = _weights("random", 3, 100, 6)
    cdf = rt.cdf_standalone(w)
    for r in range(3):
        wp = (w[r] + F32(1e-5)).astype(F32)
        part = np.zeros(32, F32)
        for i in range(100):
            part[i % 32] = F32(part[i % 32] + wp[i])
        total = rt._butterfly_total(part[None, :])[0]
        run, ref = F32(0), [F32(0)]
        for i in range(100):
            run = F32(run + F32(wp[i] / total))
            ref.append(run)
        np.testing.assert_array_equal(cdf[r], np.array(ref, F32))


# ------------------------------------------------------------------------------------------ oracle agreement
@pytest.mark.parametrize("S,K", [(32, 32), (64, 64), (64, 128), (128, 64)])
@pytest.mark.parametrize("kind", ["random", "trained"])
def test_emulation_agrees_with_the_oracle_except_on_flagged_samples(S, K, kind):
    R = 200
    w = _weights(kind, R, S, S + K)
    zc = _depths(R, S, S + K)
    u = np.sort(np.random.RandomState(K).rand(R, K).astype(F32), 1)
    u[:, 0] = 0.0
    bins = rt.bins_from_depths(zc)
    emu = rt.inverse_cdf(rt.cdf_fused(w), bins, u)
    ora = orc.sample_pdf(bins, w[:, 1:-1], K, u=u)
    z64, flagged, bar = rt.sample_pdf64(bins, w[:, 1:-1], u)
    ok = ~flagged
    assert np.all(np.abs(emu[ok] - z64[ok]) <= bar[ok])
    assert np.all(np.abs(ora[ok] - z64[ok]) <= bar[ok])
    assert np.all(np.abs(emu[ok].astype(F64) - ora[ok]) <= 2 * bar[ok])
    print(f"S={S} K={K} {kind}: flagged {flagged.sum()} of {flagged.size}, emulation != oracle on "
          f"{(emu != ora).sum()} ({(emu[ok] != ora[ok]).sum()} unflagged, all within the bar)")
    if kind == "trained":
        assert flagged.any()          # the threshold flag does occur with empty space


# ------------------------------------------------------------------------------------------ defect injection
def _defect_case(S=64, K=64, seed=9):
    R = 64
    w = np.concatenate([_weights("random", R // 2, S, seed), _weights("trained", R // 2, S, seed + 1)])
    zc = _depths(R, S, seed)
    u = np.random.RandomState(seed).rand(R, K).astype(F32)
    u[:, 0] = 0.0
    u[:, 1:9] = rt.cdf_fused(w)[:, 4:60:7]                 # on knots (empty space of the trained-like rays)
    u[:, 9:12] = [3e-5, 1.5e-4, 4e-4]                      # below a trained-like ray's surface
    return w, zc, u


def test_correct_emulation_passes_the_comparator():
    w, zc, u = _defect_case()
    z, _, _ = rt.z_fine(w, zc, u)
    rep = rt.check_resampling(z, w, zc, u)
    assert rep["differ"] == 0 and rep["f64_bad"] == 0 and rep["nonfinite_mismatch"] == 0, rep


@pytest.mark.parametrize("defect", rt.DEFECTS)
def test_each_injected_defect_is_rejected(defect):
    """The device's depths are compared bit for bit with the emulation; a kernel with one of these defects would
    return the defective emulation's depths.  The float64 comparison must also see every defect that moves an
    unflagged depth: all but the dropped coarse depth (only the merge sees it) and searchsorted 'left' (it differs
    from 'right' only for u on a knot, which is a flagged sample)."""
    w, zc, u = _defect_case()
    z_bad, _, _ = rt.z_fine(w, zc, u, defect)
    rep = rt.check_resampling(z_bad, w, zc, u)
    assert rep["differ"] > 0, (defect, rep)
    if defect not in ("drop_coarse", "side_left"):
        bad = rt.check_resampling(z_bad, w, zc, u, defect)
        assert bad["differ"] == 0
        assert bad["f64_bad"] + bad["nonfinite_mismatch"] > 0, (defect, bad)


# ------------------------------------------------------------------------------------------ compositing references
def test_composite64_against_the_fp32_oracle():
    rs = np.random.RandomState(2)
    R, S = 50, 64
    sig = (rs.randn(R, S) * 3).astype(F32)
    sig[0, :] = 1e30                          # alpha = 1 everywhere
    sig[1, :] = -5                            # alpha = 0
    rgb = rs.rand(R, S, 3).astype(F32)
    z = np.sort(rs.uniform(2, 6, (R, S)), 1).astype(F32)
    z[2, 10:12] = z[2, 10]                    # zero delta
    d = rs.randn(R, 3).astype(F32)
    noise = rs.randn(R, S).astype(F32)
    w64, c64, d64, o64 = rt.composite64(sig, z, d, rgb, noise, 1.0, True)
    w32, c32, d32, o32 = orc.volume_render(sig, rgb, z, d, noise, 1.0, True)
    assert np.abs(w64 - w32).max() < 2e-6 and np.abs(c64 - c32).max() < 5e-6 and np.abs(d64 - d32).max() < 2e-5
    assert w64[0, 0] == 1 and np.all(w64[0, 1:] <= 1e-10) and np.all(w64[1] == 0)     # 1 - alpha + 1e-10
    np.testing.assert_allclose(o64, w64.sum(1))


def test_exhaustive_merge_branch_needs_an_inverted_list():
    """Coarse depths that decrease (far below near) invert the coarse list; increasing ones with random and
    trained-like weights give sorted lists."""
    w, zc, u = _defect_case()
    assert not rt.z_fine(w, zc, u)[2].any()
    near = np.full((4, 1), 2.0, F32)
    zdec = orc.coarse_depths(np.concatenate([np.zeros((4, 6), F32), near, near - F32(1e-3)], 1), 64)
    assert rt.z_fine(w[:4], zdec, u[:4])[2].all()
