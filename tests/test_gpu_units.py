"""The stand-alone kernels of csrc/aux_kernels.cuh (the reference's unit-level API) against tests/units_ref.py at the
shapes, types and edges the C ABI accepts (pytest -m gpu).

Bit for bit: generate_rays (blender and NDC), sample_pdf, mse_psnr's MSEs, searchsorted and the plain slices of
the packed weight image.  Bounded against float64: Embedding (2-ulp sinf / cosf), generate_rays against the
reference's double-focal formulas, sample_pdf (tests/render_tape.py sample_pdf64), volume_render (render_tape's
compositing bars), PSNR (log10f) and the folded W' / b' of the packed image (fmaf chain bound).  The worst values
measured on an H100 stand in BARS below.
"""
import subprocess

import numpy as np
import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200.nerf import packed_weights_pair
from oracle import nerf_oracle as orc
from tests import cases
from tests import render_tape as rt
from tests import units_ref as ur

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
WAVE_RAYS = 148 * 8 * 4          # sample_pdf / composite: 4 rays per CTA, at most 148 * 8 CTAs per launch

# Worst values measured on one H100 80GB HBM3 (700 W power limit) over the cases below.  Every bitwise comparison
# found 0 differences.  volume_render uses render_tape.BARS: weights 0.084, last weight 0.11, sums 0.56 of their
# bars; the packed image's folded W' / b' reach 0.95 of ur.check_packed's bound (units of the fmaf-chain bound plus
# half an fp16 ulp).  The ray bars are a few ulps over the emulation's own distance from float64, which is the
# device's distance (the two are equal bit for bit); the others are derived bounds.
BARS = {
    "embed_ulps": ur.EMBED_ULPS,    # sinf / cosf against float64, ulps of the result; worst 1.45 (N_freqs 16, n C > 2^31)
    "rays_blender_ulps": 4.0,       # generate_rays vs float64 with a double focal, ulps of the triple's magnitude; 2.57
    "rays_ndc_ulps": 16.0,          # same for NDC; worst 8.15 (camera 2.3 from the near plane: a long shift o + t d)
    "psnr": 1.0,                    # |psnr - float64| / ur.psnr_bar; worst 0.54
}


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def card(dev):
    name = torch.cuda.get_device_name(dev)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(dev.index)],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    print(f"\ncard: {name}, power limit {pl}")


def T(a, dev):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev)


# ------------------------------------------------------------------------------------------------ Embedding
def _embed_inputs(n, seed):
    rs = np.random.RandomState(seed)
    mag = 10.0 ** rs.uniform(-3, 4, (n, 1))
    x = (rs.uniform(-1, 1, (n, 3)) * mag).astype(F32)
    specials = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e4, -1e4, 3.1415927, 1e-30, 65504.0], F32)
    k = min(len(specials), n)
    x[:k, 0] = specials[:k]
    return x


def _embed_check(got, x, n_freqs, freqs=None):
    ref = ur.embed64(x, n_freqs, freqs)
    c = x.shape[1]
    assert got.shape == ref.shape
    np.testing.assert_array_equal(got[:, :c].view(np.uint32), np.asarray(x, F32).view(np.uint32))   # x copied
    g, r = got[:, c:], ref[:, c:]
    e = ur.embed_ulps(g, r) if r.size else np.zeros(1)
    zero = np.isfinite(r) & (r == 0)
    return float(e.max()), np.array_equal(np.signbit(g[zero]), np.signbit(r[zero]))     # sin(-0) = -0


@pytest.mark.parametrize("n_freqs", list(range(17)))
def test_embedding_every_frequency_count(n_freqs, dev):
    """embed_kernel at N_freqs 0 .. 16, |x| up to 1e4 (arguments 2^15 1e4 ~ 3.3e8 take sinf's slow reduction),
    +-0, +-inf, NaN, n = 1000 (not a multiple of 256)."""
    x = _embed_inputs(1000, n_freqs)
    emb = nb.Embedding(3, n_freqs)
    with torch.no_grad():
        got = emb(T(x, dev)).cpu().numpy()
    worst, signs_ok = _embed_check(got, x, n_freqs)
    xt = T(x, dev)
    parts = [xt]
    for k in range(n_freqs):
        a = float(2.0 ** k) * xt
        parts += [torch.sin(a), torch.cos(a)]
    tor = torch.cat(parts, -1).cpu().numpy()
    vs_torch = ur.bitwise_differ(got, tor)
    print(f"\nembed N_freqs {n_freqs}: worst {worst:.3g} ulp (bar {BARS['embed_ulps']}); "
          f"{vs_torch} of {got.size} differ from torch.sin / torch.cos")
    assert worst <= BARS["embed_ulps"] and signs_ok


def test_embedding_past_2_31_elements(dev):
    """n * C > 2^31 (N_freqs = 16, C = 99): sampled rows, those around the 2^31-th element and the last."""
    C = 99
    n = (1 << 31) // C + 4099
    x = torch.empty(n, 3, device=dev).uniform_(-30, 30)
    with torch.no_grad():
        out = nb.Embedding(3, 16)(x)
    assert out.shape == (n, C)
    cross = (1 << 31) // C
    rows = np.unique(np.concatenate([np.arange(256), cross + np.arange(-300, 300), n - 1 - np.arange(256),
                                     np.random.RandomState(0).randint(0, n, 2048)]))
    ri = torch.from_numpy(rows).to(dev)
    got, xs = out[ri].cpu().numpy(), x[ri].cpu().numpy()
    del out
    torch.cuda.empty_cache()
    worst, _ = _embed_check(got, xs, 16)
    print(f"\nembed n {n} (n C = {n * C}): worst {worst:.3g} ulp over {len(rows)} rows")
    assert worst <= BARS["embed_ulps"]


def test_embedding_of_a_wider_input(dev):
    """An (N, 6) input to Embedding(3, 10), the module the fused kernel serves, gives (N, 126) as the reference's
    torch ops do; the kernel reads rows of 3, and taking it here returned (N, 63) of wrong values.  Embedding(6, 10)
    on the same input agrees bit for bit."""
    x6 = np.random.RandomState(3).uniform(-3, 3, (257, 6)).astype(F32)
    with torch.no_grad():
        got = nb.Embedding(3, 10)(T(x6, dev)).cpu().numpy()
        got66 = nb.Embedding(6, 10)(T(x6, dev)).cpu().numpy()
    assert got.shape == (257, 126)
    worst, _ = _embed_check(got, x6, 10)
    print(f"\nEmbedding(3, 10) on (N, 6): worst {worst:.3g} ulp")
    assert worst <= BARS["embed_ulps"] and ur.bitwise_differ(got66, got) == 0


def test_embedding_of_more_than_16_frequencies(dev):
    """Embedding(3, N > 16) under no_grad (the kernel takes at most 16 frequencies) goes through torch ops, at the
    reference's shape and values."""
    x3 = np.random.RandomState(4).uniform(-3, 3, (257, 3)).astype(F32)
    e20 = nb.Embedding(3, 20)
    with torch.no_grad():
        got = e20(T(x3, dev)).cpu().numpy()
    assert got.shape == (257, 123)
    worst, _ = _embed_check(got, x3, 20, e20.freq_bands.tolist())
    print(f"\nEmbedding(3, 20): worst {worst:.3g} ulp")
    assert worst <= BARS["embed_ulps"]


# ------------------------------------------------------------------------------------------------ generate_rays
def _pose(kind):
    if kind == "golden_like":
        return np.array([[0.7648422, 0.0, 0.64421767, 1.5], [0.2, 0.96, -0.1, -0.3], [-0.64421767, 0.1, 0.7648422, 3.2]])
    rs = np.random.RandomState(7)
    q = np.linalg.qr(rs.randn(3, 3))[0]
    t = {"rotated": [0.3, -1.2, 2.5], "near_plane": [0.1, -0.05, -1.0 + 1e-3], "on_plane": [0.2, 0.1, -1.0]}[kind]
    if kind != "rotated":              # forward-facing: the camera looks down -z, slightly rotated
        q = np.array([[0.995, -0.0998, 0.0], [0.0998, 0.995, 0.0], [0.0, 0.0, 1.0]])
    return np.concatenate([q, np.array(t)[:, None]], 1).astype(F32)


RAY_CASES = [(1, 1, 0.7, "rotated", False), (7, 5, 3.3, "rotated", False), (24, 36, 41.5, "golden_like", False),
             (401, 399, 555.5, "rotated", False), (3024, 4032, 3260.5, "rotated", False),
             (1, 1, 0.7, "near_plane", True), (7, 5, 3.3, "near_plane", True), (24, 36, 41.5, "golden_like", True),
             (37, 801, 1111.1, "near_plane", True), (64, 48, 60.0, "on_plane", True),
             (3024, 4032, 3260.5, "near_plane", True)]


@pytest.mark.parametrize("H,W,focal,pose,ndc", RAY_CASES)
def test_generate_rays_bitwise(H, W, focal, pose, ndc, dev):
    """generate_rays equals the float32 emulation bit for bit (odd W and H: W / 2 = x.5; 3024 x 4032 = 12.2 M rays,
    LLFF's full resolution), and the float64 reference formulas with a double focal within BARS."""
    c2w = _pose(pose)
    got = nb.generate_rays(H, W, focal, c2w, 2.0, 6.0, ndc=ndc, device=dev).cpu().numpy()
    emu = ur.generate_rays32(H, W, focal, c2w, 2.0, 6.0, ndc)
    diff = ur.bitwise_differ(got, emu)
    del emu
    sel = np.arange(H * W) if H * W <= 1 << 20 else np.unique(np.r_[np.arange(0, H * W, 97), H * W - 1])
    r64, sc = ur.generate_rays64(H, W, focal, c2w, 2.0, 6.0, ndc, sel)
    e = ur.ray_ulps(got[sel], r64, sc)
    bar = BARS["rays_ndc_ulps" if ndc else "rays_blender_ulps"]
    print(f"\nrays {H}x{W} {pose} ndc {ndc}: {diff} differ from the emulation; float64 worst {e.max():.3g} ulp")
    assert diff == 0 and e.max() <= bar


# ------------------------------------------------------------------------------------------------ sample_pdf
def _pdf_case(R, nw, K, seed, edge):
    rs = np.random.RandomState(seed)
    w = rs.dirichlet(np.ones(nw) * 0.5, R).astype(F32) * rs.uniform(0.2, 3, (R, 1)).astype(F32)   # cdf[-1] != 1 too
    bins = np.sort(rs.uniform(2, 6, (R, nw + 1)), 1).astype(F32)
    u = rs.rand(R, K).astype(F32)
    if edge:
        w[0] = 0                                      # all-zero weights: uniform cdf
        if R > 1:
            w[1] = 0
            w[1, nw // 2] = 5                         # one dominant weight: the denom < eps branch elsewhere
        if R > 2:
            w[2, rs.rand(nw) < 0.8] = 0               # flat runs
        cdf = rt.cdf_standalone(w)
        u[:, 0] = 0.0
        if K > 1:
            u[:, 1] = 1.0
        if K > 4:
            k = rs.randint(0, nw + 1, (R, K - 4))
            u[:, 4:] = np.where(rs.rand(R, K - 4) < 0.5, cdf[np.arange(R)[:, None], k], u[:, 4:])   # on knots
    return bins, w, u


@pytest.mark.parametrize("nw", [1, 31, 32, 33, 62, 63, 1000, 4096])
@pytest.mark.parametrize("K", [1, 31, 33, 200])
def test_sample_pdf_bitwise(nw, K, dev):
    """sample_pdf_kernel against cdf_standalone + inverse_cdf bit for bit; float64 sample_pdf64: no unflagged sample
    outside its bar."""
    R = 9 if nw >= 1000 else 131
    bins, w, u = _pdf_case(R, nw, K, 1000 * nw + K, True)
    got = nb.sample_pdf(T(bins, dev), T(w, dev), K, u=T(u, dev)).cpu().numpy()
    emu = rt.inverse_cdf(rt.cdf_standalone(w), bins, u)
    diff = ur.bitwise_differ(got, emu)
    z64, flagged, bar = rt.sample_pdf64(bins, w, u, sequential=True)
    far = int((~(np.abs(got - z64) <= bar) & ~flagged).sum())
    print(f"\nsample_pdf nw {nw} K {K}: {diff} differ from the emulation; float64 {far} unflagged outside the bar, "
          f"{int(flagged.sum())} flagged")
    assert diff == 0 and far == 0


@pytest.mark.parametrize("R", [1, 3, 4, 5, WAVE_RAYS - 1, WAVE_RAYS + 1, 3 * WAVE_RAYS + 7])
@pytest.mark.parametrize("det", [False, True])
def test_sample_pdf_ray_counts(R, det, dev):
    """Ray counts around the 4-warp block and past one grid wave (each CTA then walks several rays), det u too."""
    nw, K = 62, 64
    bins, w, u = _pdf_case(R, nw, K, R, True)
    bt, wt = T(bins, dev), T(w, dev)
    if det:
        got = nb.sample_pdf(bt, wt, K, det=True).cpu().numpy()
        u = np.broadcast_to(torch.linspace(0, 1, K, device=dev).cpu().numpy(), (R, K))
    else:
        got = nb.sample_pdf(bt, wt, K, u=T(u, dev)).cpu().numpy()
    emu = rt.inverse_cdf(rt.cdf_standalone(w), bins, u)
    assert ur.bitwise_differ(got, emu) == 0


def test_sample_pdf_rejects_more_than_4096_weights(dev):
    w = torch.ones(2, 4097, device=dev)
    b = torch.ones(2, 4098, device=dev)
    with pytest.raises(ValueError, match="sample_pdf: bad sizes"):
        nb.sample_pdf(b, w, 8, u=torch.rand(2, 8, device=dev))


# ------------------------------------------------------------------------------------------------ mse_psnr
@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 640_000, 4_000_000])
@pytest.mark.parametrize("mode", ["coarse_only", "fine", "equal"])
def test_mse_psnr(n, mode, dev):
    """MSEs bit for bit against the kernel's fixed order; PSNR within log10f's bound of float64."""
    rs = np.random.RandomState(n % 1000)
    tgt = rs.rand(n, 3).astype(F32)
    rc = (tgt + rs.randn(n, 3).astype(F32) * F32(0.05)).astype(F32)
    rf = None if mode == "coarse_only" else (tgt + rs.randn(n, 3).astype(F32) * F32(0.01)).astype(F32)
    if mode == "equal":
        rf = tgt.copy()
    res = {"rgb_coarse": T(rc, dev)}
    if rf is not None:
        res["rgb_fine"] = T(rf, dev)
    out = nb.mse_psnr(res, T(tgt, dev))
    got = {k: float(v) for k, v in out.items()}
    mc, mf, tot, fin = ur.mse_psnr32(rc, rf, tgt)
    assert got["mse_coarse"] == mc and got["mse_fine"] == mf
    assert got["loss"] == (tot if rf is not None else mc)
    m64 = ur.mse64(rf if rf is not None else rc, tgt)
    if m64 == 0:
        assert got["psnr"] == np.inf                  # the reference's -10 log10(0) = +inf
        err = 0.0
    else:
        err = abs(got["psnr"] - (-10 * np.log10(m64))) / ur.psnr_bar(fin, got["psnr"])
    print(f"\nmse_psnr n {n} {mode}: psnr {got['psnr']:.6g}, error {err:.3g} of the bar")
    assert err <= BARS["psnr"]


# ------------------------------------------------------------------------------------------------ searchsorted
def _ss_check(a, v, dev):
    for side in ("left", "right"):
        got = nb.searchsorted(T(a, dev), T(v, dev), side=side).cpu().numpy()
        np.testing.assert_array_equal(got, orc.searchsorted(a, v, side))


def _edge_values(rs, a, n):
    v = rs.choice(a.reshape(-1), n).astype(F32)                    # exact ties
    v[::7] = np.nan
    v[1::7] = 0.0
    v[2::7] = -0.0
    v[3::7] = np.inf
    v[4::7] = -np.inf
    return v


@pytest.mark.parametrize("A", [100_000, 1 << 20])
def test_searchsorted_long_rows(A, dev):
    rs = np.random.RandomState(A % 97)
    a = np.sort(np.round(rs.randn(2, A) * 4, 1), 1).astype(F32)    # ties everywhere
    a[0, :5], a[0, -3:] = -np.inf, np.inf
    a[1, A // 2 - 2:A // 2 + 2] = [-0.0, 0.0, -0.0, 0.0]
    a = np.sort(a, 1)
    v = np.stack([_edge_values(rs, a[r], 3000) for r in range(2)])
    _ss_check(a, v, dev)


def test_searchsorted_broadcast_rows(dev):
    """A one-row a against 10^6 rows of v, and 10^6 rows of a against a one-row v."""
    rs = np.random.RandomState(5)
    a1 = np.sort(np.round(rs.randn(1, 100), 1), 1).astype(F32)
    v = _edge_values(rs, a1, 1_000_000 * 3).reshape(1_000_000, 3)
    _ss_check(a1, v, dev)
    a = np.sort(np.round(rs.randn(1_000_000, 6), 1), 1).astype(F32)
    v1 = np.array([[np.nan, -np.inf, -0.0, 0.0, 0.1, 1.0, np.inf]], F32)
    _ss_check(a, v1, dev)


# ------------------------------------------------------------------------------------------------ volume_render
def _vr_case(n, S, seed, edge):
    rs = np.random.RandomState(seed)
    sig = (rs.randn(n, S) * 3).astype(F32)
    rgb = rs.rand(n, S, 3).astype(F32)
    z = np.sort(rs.uniform(2, 6, (n, S)).astype(F32), -1)
    d = (rs.randn(n, 3) * rs.uniform(0.2, 3, (n, 1))).astype(F32)
    noise = rs.randn(n, S).astype(F32)
    if edge and n >= 6:
        d[0] = 0                                      # zero-norm direction: every delta 0
        d[1] = [1e18, -3e17, 2e17]                    # huge direction (|d|^2 still finite in fp32)
        z[2, 4:12] = z[2, 4]                          # repeated depths: delta 0
        sig[3, 5] = 1e4                               # alpha = 1 exactly: the transmittance at the 1e-10 floor
        sig[3, 9] = 3e4
        sig[4] = 1e4
        z[5] = z[5, 0]                                # one depth for the whole ray
    return sig, rgb, z, d, noise


@pytest.mark.parametrize("S", [32, 96, 160, 192])
@pytest.mark.parametrize("n", [1, 3, 4, 5, 97, 3 * WAVE_RAYS + 5])
def test_volume_render_shapes(S, n, dev):
    sig, rgb, z, d, noise = _vr_case(n, S, S + n, True)
    for nz, ns, wb, with_rgb in ((None, 0.0, False, True), (noise, 0.0, True, True), (noise, 1.0, True, False)):
        r = rgb if with_rgb else None
        w, c, dp, op = [None if x is None else x.cpu().numpy()
                        for x in nb.volume_render(T(sig, dev), T(r, dev), T(z, dev), T(d, dev), T(nz, dev), ns, wb)]
        assert (c is None) == (not with_rgb) and (dp is None) == (not with_rgb)
        e = rt.composite_errors(sig, r, z, d, nz, ns, wb, w, c, dp, op)
        print(f"\nvolume_render S {S} n {n} noise_std {ns} wb {wb} rgb {with_rgb}: "
              + " ".join(f"{k} {v:.3g}" for k, v in e.items()))
        assert np.all(np.isfinite(w))
        assert not rt.composite_violations(e), rt.composite_violations(e)
    if n >= 6:
        assert np.all(w[0] == 0) and np.all(w[5, :-1] == 0)


def test_volume_render_nan_sigma_is_empty_space(dev):
    """composite_ray clamps sigma with fmaxf(s, 0), so a NaN sigma gives weight 0 and the rest of the ray is composited
    as if that sample were empty.  The reference's torch.relu (and the oracle's np.maximum) keep the NaN, which then
    spreads to every later weight.  Pinned here; DESIGN.md section 5 records the divergence."""
    S, n = 64, 8
    sig, rgb, z, d, _ = _vr_case(n, S, 11, False)
    sig[:, 10] = np.nan
    sig[3, :] = np.nan
    w, c, dp, op = [x.cpu().numpy() for x in nb.volume_render(T(sig, dev), T(rgb, dev), T(z, dev), T(d, dev))]
    assert np.all(w[:, 10] == 0) and np.all(w[3] == 0) and op[3] == 0
    clean = np.where(np.isnan(sig), F32(0), sig)
    e = rt.composite_errors(clean, rgb, z, d, None, 0.0, False, w, c, dp, op)
    assert not rt.composite_violations(e), rt.composite_violations(e)
    ow, _, _, _ = orc.volume_render(sig, rgb, z, d)
    assert np.isnan(ow[:, 10:]).all()                 # the reference's semantics


# ------------------------------------------------------------------------------------------------ packed weights
SENTINEL = 0xA5                  # fill byte (fp16 -0.0222, fp32 -2.9e-16): a region a launch leaves unwritten keeps it


def _model(w, dev):
    m = nb.NeRF()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
    return m.to(dev)


@pytest.mark.parametrize("kind", ["random", "trained"])
def test_packed_weight_image(kind, dev):
    """Every written element of nb.packed_weights: the plain slices (zero columns of slices 0 and 34 and the
    transposed backward slices included) and the fp32 region bit for bit, the folded W' / b' within the fmaf chain's
    bound of float64, and W' identical in its forward and backward copies."""
    ws = cases.trained_weights() if kind == "trained" else cases.weights()
    for w in ws:
        m = _model(w, dev)
        nb.packed_weights(m).fill_(SENTINEL)              # the allocator may hand back a blob that holds this image
        blob = nb.packed_weights(m)                       # trainable: every call re-packs into the same blob
        assert blob.numel() == ur.PACKED_BYTES
        rep = ur.check_packed(blob.cpu().numpy(), w)
        print(f"\npacked {kind}: {rep}")
        assert rep["plain_differ"] == 0 and rep["fold_outside"] == 0 and rep["fold_twins_differ"] == 0


def test_pack_pair_equals_two_single_packs(dev):
    """Each blob is filled with a sentinel before each launch, so every compared byte was written by that launch."""
    ws = cases.weights()
    ma, mb = _model(ws[0], dev), _model(ws[1], dev)       # trainable: every call re-packs, the pair in one launch

    def fill():
        for m in (ma, mb):
            nb.packed_weights(m).fill_(SENTINEL)         # allocates / re-packs the cached blob, then overwrites it

    fill()
    pa, pb = [b.clone() for b in packed_weights_pair(ma, mb)]
    fill()
    sa = nb.packed_weights(ma).clone()
    fill()
    sb = nb.packed_weights(mb).clone()
    for x, y, w in ((pa, sa, ws[0]), (pb, sb, ws[1])):
        assert torch.equal(x[:ur.FWD_BYTES], y[:ur.FWD_BYTES]) and torch.equal(x[ur.OFF_BWD:], y[ur.OFF_BWD:])
        rep = ur.check_packed(x.cpu().numpy(), w)
        assert rep["plain_differ"] == 0 and rep["fold_outside"] == 0 and rep["fold_twins_differ"] == 0
