"""GPU parity tests (pytest -m gpu): the sm_90a kernels, called through the C ABI, against
(a) the committed outputs of the reference's own Python path (tests/golden) and (b) the numpy
oracle on the same seeded inputs.

Tolerances (floating-point path, BASELINE.json north_star: "rgb_fine within 1e-3 abs"):
  rgb_*      1e-3 absolute      (MLP in fp16 operands / fp32 accumulate, rest fp32)
  opacity_*  1e-3 absolute
  depth_*    4e-3 absolute      (depths are 2..6: 1e-3 relative); 2e-2 when noise_std > 0:
             with sigma noise of std 1 the ReLU kink at sigma+noise = 0 makes depth (a weighted
             sum of z in [2,6]) ill-conditioned - the fp32 oracle itself moves by 1.05e-2 when only
             its WEIGHTS are rounded to fp16 (measured, DESIGN.md section "Precision").
Integer/index work (searchsorted) is bit-exact.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib
from oracle import nerf_oracle as orc
from tests import cases

pytestmark = pytest.mark.gpu

TOL = {"rgb": 1e-3, "opacity": 1e-3, "depth": 4e-3}


def tol_for(key, noise_std=0.0):
    kind = key.split("_")[0]
    if kind == "depth" and noise_std > 0:
        return 2e-2
    return TOL[kind]


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def ws():
    return cases.weights()


@pytest.fixture(scope="module")
def models(ws, dev):
    out = []
    for w in ws:
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        out.append(m.to(dev).eval())
    return out


@pytest.fixture(scope="module")
def emb():
    return [nb.Embedding(3, 10), nb.Embedding(3, 4)]


def _fp16_error_model():
    import importlib.util
    spec = importlib.util.spec_from_file_location("fp16_error_model", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "fp16_error_model.py"))
    em = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(em)
    return em


def to_dev(d, dev):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in d.items()}


@pytest.mark.parametrize("name", list(cases.CASES))
def test_render_rays_vs_reference_golden(name, models, emb, ws, dev):
    n, kind, rseed, S, K, disp, perturb, noise, wb, tt = cases.CASES[name]
    rays, randoms, ref = cases.load_case(name)
    with torch.no_grad():
        out = nb.render_rays(models, emb, torch.from_numpy(rays).to(dev), S, disp, perturb, noise, K, 1024 * 32,
                             wb, test_time=tt, randoms=to_dev(randoms, dev))
    torch.cuda.synchronize()
    assert set(out) == set(ref)                                   # result keys (models/rendering.py:209-242)
    oracle = orc.render_rays(ws, rays, S, disp, perturb, noise, K, wb, tt, randoms)
    for k, v in ref.items():
        got = out[k].cpu().numpy()
        assert got.shape == v.shape and got.dtype == np.float32
        mx, p999, mean = cases.error_stats(got, v)
        mxo, _, _ = cases.error_stats(got, oracle[k])
        print(f"{name}/{k}: vs reference max {mx:.2e} p99.9 {p999:.2e} mean {mean:.2e}; vs oracle max {mxo:.2e}")
        assert mx < tol_for(k, noise), f"{name}/{k} vs reference: max {mx:.3e}"
        assert mxo < tol_for(k, noise), f"{name}/{k} vs oracle: max {mxo:.3e}"
    if "rgb_fine" in ref:
        assert orc.psnr(out["rgb_fine"].cpu().numpy(), ref["rgb_fine"]) > 60.0


def test_units_vs_reference_golden(models, emb, dev):
    u = np.load(os.path.join(cases.GOLDEN, "units.npz"))
    x3 = torch.from_numpy(u["x3"]).to(dev)
    np.testing.assert_allclose(emb[0](x3).cpu().numpy(), u["embed10"], atol=2e-6, rtol=0)   # a2
    np.testing.assert_allclose(emb[1](x3 / 6).cpu().numpy(), u["embed4"], atol=2e-6, rtol=0)
    with torch.no_grad():
        full = models[0](torch.from_numpy(u["nerf_in"]).to(dev)).cpu().numpy()              # a4
        sig = models[1](torch.from_numpy(u["embed10"]).to(dev), sigma_only=True).cpu().numpy()
    assert full.shape == (64, 4) and sig.shape == (64, 1)
    assert np.abs(full[:, :3] - u["nerf_full"][:, :3]).max() < 1e-3
    assert (np.abs(full[:, 3] - u["nerf_full"][:, 3]) / (1 + np.abs(u["nerf_full"][:, 3]))).max() < 2e-3
    assert (np.abs(sig - u["nerf_sigma"]) / (1 + np.abs(u["nerf_sigma"]))).max() < 2e-3
    bins, wts = torch.from_numpy(u["pdf_bins"]).to(dev), torch.from_numpy(u["pdf_weights"]).to(dev)
    det = nb.sample_pdf(bins, wts, 64, det=True).cpu().numpy()                               # a8
    np.testing.assert_allclose(det[:, :-1], u["pdf_det"][:, :-1], atol=1e-4, rtol=0)
    last_bin = u["pdf_bins"][:, -1] - u["pdf_bins"][:, -2]
    assert np.all(np.abs(det[:, -1] - u["pdf_det"][:, -1]) <= last_bin + 1e-5)
    rnd = nb.sample_pdf(bins, wts, 48, det=False, u=torch.from_numpy(u["pdf_u"]).to(dev)).cpu().numpy()
    np.testing.assert_allclose(rnd, u["pdf_rand"], atol=1e-4, rtol=0)


@pytest.mark.parametrize("side", ["left", "right"])
def test_searchsorted_reference_grid(side, dev):
    """torchsearchsorted/test/test_searchsorted.py:27-44 grid, exact integer equality (a9)."""
    rs = np.random.RandomState(0)
    for Ba, Bv in ((1, 1), (100, 100), (200, 200), (1, 100), (100, 1)):
        for A in (1, 50, 500):
            for V in (1, 12, 120):
                a = np.sort(rs.rand(Ba, A).astype(np.float32), -1)
                v = rs.rand(Bv, V).astype(np.float32)
                if A > 4:
                    v[:, 0] = a[0, 3] if Ba == 1 else a[:Bv, 3] if Bv <= Ba else a[0, 3]   # exact ties
                got = nb.searchsorted(torch.from_numpy(a).to(dev), torch.from_numpy(v).to(dev), side=side)
                assert got.dtype == torch.long and got.is_cuda
                np.testing.assert_array_equal(got.cpu().numpy(), orc.searchsorted(a, v, side))
    # hot-path shape: cdf (R,63), deterministic u with ties at 0 and 1
    cdf = np.sort(rs.rand(4096, 63).astype(np.float32), -1)
    cdf[:, 0], cdf[:, -1] = 0.0, 1.0
    uu = np.broadcast_to(orc.linspace01(64), (4096, 64)).copy()
    got = nb.searchsorted(torch.from_numpy(cdf).to(dev), torch.from_numpy(uu).to(dev), side=side)
    np.testing.assert_array_equal(got.cpu().numpy(), orc.searchsorted(cdf, uu, side))


def test_searchsorted_errors(dev):
    with pytest.raises(AssertionError):
        nb.searchsorted(torch.zeros(3, 4, device=dev), torch.zeros(2, 4, device=dev))
    with pytest.raises(AssertionError):
        nb.searchsorted(torch.zeros(4, device=dev), torch.zeros(2, 4, device=dev))
    assert nb.searchsorted(torch.zeros(2, 0, device=dev), torch.zeros(2, 3, device=dev)).sum().item() == 0


@pytest.mark.parametrize("S,with_rgb,wb", [(64, True, True), (128, True, False), (192, False, False), (64, False, True)])
def test_volume_render_vs_oracle(S, with_rgb, wb, dev):
    rs = np.random.RandomState(S)
    n = 257
    sig = (rs.randn(n, S) * 3).astype(np.float32)
    rgb = rs.rand(n, S, 3).astype(np.float32) if with_rgb else None
    z = np.sort(rs.uniform(2, 6, (n, S)).astype(np.float32), -1)
    d = rs.randn(n, 3).astype(np.float32)
    noise = rs.randn(n, S).astype(np.float32)
    w, c, dp, op = nb.volume_render(torch.from_numpy(sig).to(dev), None if rgb is None else torch.from_numpy(rgb).to(dev),
                                    torch.from_numpy(z).to(dev), torch.from_numpy(d).to(dev),
                                    torch.from_numpy(noise).to(dev), 0.7, wb)
    ow, oc, od, oo = orc.volume_render(sig, rgb, z, d, noise, 0.7, wb)
    np.testing.assert_allclose(w.cpu().numpy(), ow, atol=2e-6, rtol=1e-5)
    np.testing.assert_allclose(op.cpu().numpy(), oo, atol=5e-6, rtol=1e-5)
    if with_rgb:
        np.testing.assert_allclose(c.cpu().numpy(), oc, atol=5e-6, rtol=1e-5)
        np.testing.assert_allclose(dp.cpu().numpy(), od, atol=2e-5, rtol=1e-5)


def test_full_image_properties(models, emb, ws, dev):
    """BASELINE.json configs[2]: one 400x400 view (160,000 rays) in eval.py's 32768-ray chunks,
    test_time=True.  Size-independent properties + a random 384-ray subset against the oracle."""
    import bench
    n = 160000
    rays_np = bench.blender_rays(n, 5)
    rays = torch.from_numpy(rays_np).to(dev)
    with torch.no_grad():
        chunks = [nb.render_rays(models, emb, rays[i:i + 32768], 64, False, 0, 0, 64, 32768, True,
                                 test_time=True, extras=True) for i in range(0, n, 32768)]
        whole = nb.render_rays(models, emb, rays, 64, False, 0, 0, 64, 32768, True, test_time=True, extras=True)
        again = nb.render_rays(models, emb, rays, 64, False, 0, 0, 64, 32768, True, test_time=True, extras=True)
    torch.cuda.synchronize()
    assert set(whole) - {"z_vals_fine", "weights_fine", "weights_coarse"} == {
        "opacity_coarse", "rgb_fine", "depth_fine", "opacity_fine"}
    for k in whole:
        cat = torch.cat([c[k] for c in chunks], 0)
        assert torch.equal(cat, whole[k]), f"chunking changed {k}"          # rays are independent units
        assert torch.equal(again[k], whole[k]), f"non-deterministic {k}"
        assert torch.isfinite(whole[k]).all()
    z = whole["z_vals_fine"]
    assert z.shape == (n, 128) and bool((z[:, 1:] >= z[:, :-1]).all())       # sorted merge (:229)
    t = torch.from_numpy(orc.linspace01(64)).to(dev)
    zc = rays[:, 6:7] * (1 - t) + rays[:, 7:8] * t
    pos = torch.searchsorted(z.contiguous(), zc.contiguous())
    assert torch.allclose(torch.gather(z, 1, pos.clamp(max=127)), zc, atol=1e-6)   # coarse depths are kept
    assert bool((z >= rays[:, 6:7] - 1e-6).all()) and bool((z <= rays[:, 7:8] + 1e-6).all())
    for k in ("opacity_coarse", "opacity_fine"):
        assert float(whole[k].min()) >= 0.0 and float(whole[k].max()) <= 1.0 + 1e-5
    assert torch.allclose(whole["weights_fine"].sum(1), whole["opacity_fine"], atol=1e-5)
    assert float(whole["rgb_fine"].min()) >= -1e-5 and float(whole["rgb_fine"].max()) <= 1.0 + 1e-4
    idx = np.random.RandomState(0).choice(n, 384, replace=False)
    ref = orc.render_rays(ws, rays_np[idx], 64, False, 0.0, 0.0, 64, True, True)
    for k, v in ref.items():
        mx, p999, mean = cases.error_stats(whole[k][torch.from_numpy(idx).to(dev)].cpu().numpy(), v)
        print(f"full-image subset {k}: max {mx:.2e} p99.9 {p999:.2e} mean {mean:.2e}")
        assert mx < tol_for(k)


def test_llff_view_with_noise_properties(models, emb, ws, dev):
    """BASELINE.json configs[3]: one LLFF-fern-shaped view, 504x378 = 190,512 NDC rays (near 0, far 1,
    non-unit directions; datasets/llff.py:236-241), the README recipe's perturb=1 / noise_std=1,
    white_back=False, training-mode forward.  Size-independent properties (bit-exact determinism and
    chunk invariance with the same random tensors, ranges, weights sum) + a 256-ray subset against
    the oracle on the same random draws."""
    H, W, focal = 378, 504, 407.0
    c2w = np.array([[1, 0, 0, 0.05], [0, 1, 0, -0.02], [0, 0, 1, 0.1]], np.float32)
    rays = nb.generate_rays(H, W, focal, c2w, 0.0, 1.0, ndc=True, device=dev)
    n = H * W
    assert rays.shape == (n, 8) and n == 190512
    g = torch.Generator(device=dev).manual_seed(11)
    rnd = {"perturb_rand": torch.rand(n, 64, device=dev, generator=g), "noise_coarse": torch.randn(n, 64, device=dev, generator=g),
           "u_rand": torch.rand(n, 64, device=dev, generator=g), "noise_fine": torch.randn(n, 128, device=dev, generator=g)}
    with torch.no_grad():
        a = nb.render_rays(models, emb, rays, 64, False, 1.0, 1.0, 64, 32768, False, randoms=rnd, extras=True)
        b = nb.render_rays(models, emb, rays, 64, False, 1.0, 1.0, 64, 32768, False, randoms=rnd, extras=True)
        lo, hi = 70001, 70001 + 4097
        part = nb.render_rays(models, emb, rays[lo:hi], 64, False, 1.0, 1.0, 64, 32768, False,
                              randoms={k: v[lo:hi] for k, v in rnd.items()}, extras=True)
    torch.cuda.synchronize()
    for k in a:
        assert torch.isfinite(a[k]).all(), k
        assert torch.equal(a[k], b[k]), f"non-deterministic {k}"
        assert torch.equal(a[k][lo:hi], part[k]), f"chunking changed {k}"
    z = a["z_vals_fine"]
    assert bool((z[:, 1:] >= z[:, :-1]).all()) and float(z.min()) >= -1e-6 and float(z.max()) <= 1 + 1e-6
    for k in ("opacity_coarse", "opacity_fine"):
        assert float(a[k].min()) >= 0.0 and float(a[k].max()) <= 1.0 + 1e-5
    assert torch.allclose(a["weights_fine"].sum(1), a["opacity_fine"], atol=1e-5)
    idx = np.random.RandomState(1).choice(n, 256, replace=False)
    ti = torch.from_numpy(idx).to(dev)
    sub_args = (ws, rays[ti].cpu().numpy(), 64, False, 1.0, 1.0, 64, False, False,
                {k: v[ti].cpu().numpy() for k, v in rnd.items()})
    ref = orc.render_rays(*sub_args)
    with _fp16_error_model().rounded_operands("wa"):
        fp16 = orc.render_rays(*sub_args)       # the fp32 oracle with the kernel's fp16 roundings, same draws
    for k, v in ref.items():
        got = a[k][ti].cpu().numpy()
        mx, p999, mean = cases.error_stats(got, v)
        print(f"llff subset {k}: max {mx:.2e} p99.9 {p999:.2e} mean {mean:.2e}")
        # NDC depths are in [0,1]; under noise a sign flip of sigma+noise at the far plane moves depth/opacity
        # by the remaining transmittance (DESIGN.md section 5): bound the bulk, and rgb by the north-star bar.
        # Which rays flip depends on the draws (a CUDA generator's stream depends on the device's SM count): a
        # ray the fp16 format itself puts over the bar on these draws is bounded by the format's own error, as
        # for ray 16 of grad_trained below, and every ray must agree with the error model.
        if k.startswith("rgb"):
            err = np.abs(got - v).max(-1)
            bar = np.maximum(1e-3, np.abs(fp16[k] - v).max(-1) + 1e-4)
            assert (err < bar).all() and mx < 5e-3, (k, mx, [(int(i), float(err[i]), float(bar[i])) for i in np.argsort(-err)[:3]])
            assert float(np.abs(got - fp16[k]).max()) < 2e-4, (k, float(np.abs(got - fp16[k]).max()))
        else:
            assert mean < 1e-3, (k, mean)


def test_800x800_view(models, emb, ws, dev):
    """BASELINE.json configs[4]'s image: 640,000 rays in one launch (the single-GPU leg of the sharded
    render), test_time=True: finite, deterministic, oracle-checked subset."""
    import bench
    rays_np = bench.blender_rays(0, 7, 800, 800, pixels="all")
    rays = torch.from_numpy(rays_np).to(dev)
    with torch.no_grad():
        a = nb.render_rays(models, emb, rays, 64, False, 0, 0, 64, 32768, True, test_time=True, match_reference_rng=False)
        b = nb.render_rays(models, emb, rays, 64, False, 0, 0, 64, 32768, True, test_time=True, match_reference_rng=False)
    torch.cuda.synchronize()
    assert a["rgb_fine"].shape == (640000, 3)
    for k in a:
        assert torch.isfinite(a[k]).all() and torch.equal(a[k], b[k]), k
    idx = np.random.RandomState(2).choice(640000, 256, replace=False)
    ref = orc.render_rays(ws, rays_np[idx], 64, False, 0.0, 0.0, 64, True, True)
    for k, v in ref.items():
        mx, _, _ = cases.error_stats(a[k][torch.from_numpy(idx).to(dev)].cpu().numpy(), v)
        assert mx < tol_for(k), (k, mx)


@pytest.mark.parametrize("K,test_time,perturb,use_disp,white_back", [
    (128, False, 1.0, False, True),     # three fine tiles per group, training-mode coarse pass, rank-sorted u
    (64, False, 1.0, True, False),      # disparity sampling
    (0, False, 0.0, False, True),       # coarse only: every tile is a coarse tile
    (64, True, 0.0, False, False),
])
def test_tile_pipeline_is_invisible(K, test_time, perturb, use_disp, white_back, models, emb, ws, dev):
    """The render kernel pipelines tiles of different ray groups (C(g+1) before F(g), helper warps
    working one tile ahead, double-buffered hand-over).  None of that may show: a launch in which
    every CTA walks 7-8 groups (odd counts end in single-ray groups) must equal, bit for bit, the
    same rays rendered in launches so small that every CTA has a single group - and the oracle."""
    import bench
    n = 148 * 14 + 3
    rays_np = bench.blender_rays(n, 9)
    rays = torch.from_numpy(rays_np).to(dev)
    g = torch.Generator(device="cpu").manual_seed(4)
    rnd = {}
    if perturb > 0:
        rnd["perturb_rand"] = torch.rand(n, 64, generator=g).to(dev)
        if K > 0:
            rnd["u_rand"] = torch.rand(n, K, generator=g).to(dev)

    def run(lo, hi):
        r = {k: v[lo:hi] for k, v in rnd.items()}
        return nb.render_rays(models, emb, rays[lo:hi], 64, use_disp, perturb, 0.0, K, 32768, white_back,
                              test_time=test_time, randoms=r, extras=True)
    with torch.no_grad():
        whole = run(0, n)
        step = 290           # <= 2 rays per CTA: one group per CTA, nothing to pipeline
        parts = [run(i, min(i + step, n)) for i in range(0, n, step)]
    torch.cuda.synchronize()
    for k in whole:
        cat = torch.cat([p_[k] for p_ in parts], 0)
        assert torch.isfinite(whole[k]).all()
        assert torch.equal(cat, whole[k]), f"tile pipelining changed {k}"
    idx = np.arange(0, n, 29)
    rn = {k: v[torch.from_numpy(idx).to(dev)].cpu().numpy() for k, v in rnd.items()}
    ref = orc.render_rays(ws, rays_np[idx], 64, use_disp, perturb, 0.0, K, white_back, test_time, randoms=rn)
    for k, v in ref.items():
        mx, p999, mean = cases.error_stats(whole[k][torch.from_numpy(idx).to(dev)].cpu().numpy(), v)
        print(f"pipeline K={K} {k}: max {mx:.2e}")
        assert mx < tol_for(k)


def test_host_buffer_entry_matches_device_path(models, emb, dev):
    """nerfb200_render_rays_host (host pointers, copies inside) == device-pointer path, bitwise."""
    lib = _lib.load()
    n = 777
    rays = orc.make_rays(n, 9)
    with torch.no_grad():
        ref = nb.render_rays(models, emb, torch.from_numpy(rays).to(dev), 64, False, 0, 0, 64, 32768, True)
    torch.cuda.synchronize()
    bufs = {k: np.zeros(tuple(v.shape), np.float32) for k, v in ref.items()}
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    args = _lib.RenderArgs(rays=p(rays), n_rays=n, ray_stride=8,
                           packed_coarse=nb.packed_weights(models[0]).data_ptr(),
                           packed_fine=nb.packed_weights(models[1]).data_ptr(),
                           n_samples=64, n_importance=64, use_disp=0, perturb=0.0, noise_std=0.0, white_back=1,
                           test_time=0, rgb_coarse=p(bufs["rgb_coarse"]), depth_coarse=p(bufs["depth_coarse"]),
                           opacity_coarse=p(bufs["opacity_coarse"]), rgb_fine=p(bufs["rgb_fine"]),
                           depth_fine=p(bufs["depth_fine"]), opacity_fine=p(bufs["opacity_fine"]))
    assert lib.nerfb200_render_rays_host(ctypes.byref(args), None) == 0, lib.nerfb200_last_error()
    for k, v in ref.items():
        np.testing.assert_array_equal(bufs[k], v.cpu().numpy())
    # the Python face of the same entry: CPU (pinned) rays in, CPU tensors out
    got = nb.render_rays_host(models, emb, torch.from_numpy(rays).pin_memory(), 64, False, 0, 0, 64, 32768, True)
    assert set(got) == set(ref)
    for k, v in ref.items():
        assert not got[k].is_cuda and torch.equal(got[k], v.cpu()), k
        assert got[k].is_pinned()          # pinned in -> pinned out: the mapped-memory (zero-copy) path ran
    # pageable rays through the Python face: the staged path
    got = nb.render_rays_host(models, emb, torch.from_numpy(rays), 64, False, 0, 0, 64, 32768, True)
    for k, v in ref.items():
        assert torch.equal(got[k], v.cpu()), k
    # strided pinned rays (a column slice of a wider pinned tensor) and caller-supplied pinned outputs
    wide = torch.zeros(n, 11).pin_memory()
    wide[:, :8] = torch.from_numpy(rays)
    outs = {k: torch.empty(tuple(v.shape)).pin_memory() for k, v in ref.items()}
    got = nb.render_rays_host(models, emb, wide[:, :8], 64, False, 0, 0, 64, 32768, True, out=outs)
    for k, v in ref.items():
        assert got[k] is outs[k] and torch.equal(got[k], v.cpu()), k


def test_in_kernel_random_numbers(models, emb, ws, dev):
    """rng_in_kernel (randoms={'seed': s}): the kernel's Philox numbers are exactly those of the host replica
    (tests/philox.py, itself pinned to the published known-answer vectors): feeding the replica's arrays as TENSORS
    gives bit-identical results, and the oracle on the same numbers agrees within the float tolerance."""
    from tests import philox
    n, seed = 333, 0x1234_5678_9ABC_DEF0
    rays = orc.make_rays(n, 17)
    r = torch.from_numpy(rays).to(dev)
    for K, tt in ((64, False), (128, True)):
        rnd = philox.randoms(seed, n, 64, K)
        with torch.no_grad():
            a = nb.render_rays(models, emb, r, 64, False, 1.0, 0.0, K, 32768, True, test_time=tt, randoms={"seed": seed},
                               extras=True)
            b = nb.render_rays(models, emb, r, 64, False, 1.0, 0.0, K, 32768, True, test_time=tt, randoms=to_dev(rnd, dev),
                               extras=True)
        torch.cuda.synchronize()
        assert set(a) == set(b)
        for k in a:
            assert torch.equal(a[k], b[k]), k
        ref = orc.render_rays(ws, rays, 64, False, 1.0, 0.0, K, True, tt, rnd)
        for k, v in ref.items():
            assert cases.error_stats(a[k].cpu().numpy(), v)[0] < tol_for(k), k
    # 'kernel': a fresh seed per call, deterministic under torch.manual_seed
    with torch.no_grad():
        torch.manual_seed(5)
        x1 = nb.render_rays(models, emb, r, 64, False, 1.0, 0.0, 64, 32768, True, randoms="kernel")["rgb_fine"]
        x2 = nb.render_rays(models, emb, r, 64, False, 1.0, 0.0, 64, 32768, True, randoms="kernel")["rgb_fine"]
    assert not torch.equal(x1, x2)
    # the host entry takes the same option (no device tensors at all: rays and results are host memory)
    got = nb.render_rays_host(models, emb, torch.from_numpy(rays).pin_memory(), 64, False, 1.0, 0.0, 64, 32768, True,
                              randoms={"seed": seed})
    with torch.no_grad():
        dev_res = nb.render_rays(models, emb, r, 64, False, 1.0, 0.0, 64, 32768, True, randoms={"seed": seed})
    for k in got:
        assert torch.equal(got[k], dev_res[k].cpu()), k


def test_weight_cache_tracks_parameter_updates(ws, emb, dev):
    m = []
    for w in ws:                  # pseudo-trained weights: non-zero opacity, so colours matter
        net = nb.NeRF()
        net.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        m.append(net.to(dev))
    rays = torch.from_numpy(orc.make_rays(64, 1)).to(dev)
    with torch.no_grad():
        a = nb.render_rays(m, emb, rays, 64, False, 0, 0, 64)["rgb_fine"].clone()
        m[1].rgb[0].bias.add_(1.0)            # in-place update bumps _version, like an optimizer step
        b = nb.render_rays(m, emb, rays, 64, False, 0, 0, 64)["rgb_fine"]
    assert float((a - b).abs().max()) > 1e-2


def test_training_path_produces_gradients(ws, emb, dev):
    """Autograd drop-in (train.py:103-117): loss.backward() fills .grad of both NeRFs."""
    m = [nb.NeRF().to(dev), nb.NeRF().to(dev)]
    rays = torch.from_numpy(orc.make_rays(128, 2)).to(dev)
    torch.manual_seed(0)
    out = nb.render_rays(m, emb, rays, 64, False, 1.0, 1.0, 64, 32768, True)
    loss = ((out["rgb_coarse"] - 0.5) ** 2).mean() + ((out["rgb_fine"] - 0.5) ** 2).mean()   # losses.py:9-14
    loss.backward()
    for net in m:
        for name, p in net.named_parameters():
            assert p.grad is not None and torch.isfinite(p.grad).all(), name
    assert float(m[0].xyz_encoding_1[0].weight.grad.abs().sum()) > 0
    assert float(m[1].rgb[0].weight.grad.abs().sum()) > 0


def test_unsupported_shapes_fail_loudly(models, emb, dev):
    rays = torch.from_numpy(orc.make_rays(8, 1)).to(dev)
    with pytest.raises(ValueError):
        nb.render_rays(models, emb, rays, 48, False, 0, 0, 0)
    with pytest.raises(ValueError):
        nb.render_rays(models, [nb.Embedding(3, 6), nb.Embedding(3, 4)], rays, 64, False, 0, 0, 0)
    with pytest.raises(ValueError):
        nb.render_rays(models[:1], emb, rays, 64, False, 0, 0, 64)
    out = nb.render_rays(models[:1], emb, rays[:0], 64, False, 0, 0, 0)          # empty input
    assert out["rgb_coarse"].shape == (0, 3)


@pytest.mark.parametrize("S,K,test_time,perturb", [(32, 0, False, 0.0), (32, 32, False, 1.0), (64, 32, True, 0.0),
                                                   (64, 96, False, 1.0), (128, 64, True, 0.0), (32, 160, False, 1.0),
                                                   (128, 0, False, 1.0)])
def test_general_sample_counts(S, K, test_time, perturb, models, emb, ws, dev):
    """N_samples in {32, 64, 128}, N_importance any multiple of 32 with N_samples + N_importance <= 192
    (opt.py:19-22 lets the user choose them) against the oracle on the same inputs; odd ray count."""
    n = 75
    rays = orc.make_rays(n, 50 + S + K)
    rs = np.random.RandomState(S * 7 + K)
    randoms = {}
    if perturb > 0:
        randoms = {"perturb_rand": rs.rand(n, S).astype(np.float32)}
        if K > 0:
            randoms["u_rand"] = rs.rand(n, K).astype(np.float32)
    ref = orc.render_rays(ws, rays, S, False, perturb, 0.0, K, True, test_time, randoms)
    with torch.no_grad():
        out = nb.render_rays(models, emb, torch.from_numpy(rays).to(dev), S, False, perturb, 0.0, K, 32768, True,
                             test_time=test_time, randoms=to_dev(randoms, dev))
    assert set(out) == set(ref)
    for k in ref:
        mx, p999, mean = cases.error_stats(out[k].cpu().numpy(), ref[k])
        # 32 coarse samples: the resampling bins are twice as wide (0.13) and sample_pdf's (u - cdf) / denom is as
        # ill-conditioned as ever (models/rendering.py:50-54), so depths move more per flipped bin
        tol = 2e-2 if (k.startswith("depth") and S == 32) else tol_for(k)
        assert mx < tol, f"S={S} K={K} {k}: max {mx:.3e} p99.9 {p999:.3e}"


def test_ray_generation_and_image_driver(models, emb, ws, dev):
    """SURVEY section 8f rows 1-2: on-GPU rays (vs reference ray_utils golden), one-launch image render,
    uint8 conversion (eval.py:58-86, 119-128)."""
    g = np.load(os.path.join(cases.GOLDEN, "raygen.npz"))
    H, W, focal = int(g["H"]), int(g["W"]), float(g["focal"])
    r = nb.generate_rays(H, W, focal, g["c2w"], 2.0, 6.0, device=dev)
    np.testing.assert_allclose(r.cpu().numpy(), g["blender"], atol=2e-6, rtol=0)
    rn = nb.generate_rays(H, W, focal, g["c2w"], 2.0, 6.0, ndc=True, device=dev)
    np.testing.assert_allclose(rn.cpu().numpy(), g["ndc"], atol=5e-6, rtol=1e-5)
    out = nb.render_image(models, emb, H, W, focal, g["c2w"], 2.0, 6.0, 64, 64, white_back=True, device=dev)
    assert out["rgb"].shape == (H, W, 3) and out["rgb_uint8"].dtype == torch.uint8
    ref = orc.render_rays(ws, g["blender"], 64, False, 0.0, 0.0, 64, True, True)
    assert np.abs(out["rgb"].reshape(-1, 3).cpu().numpy() - ref["rgb_fine"]).max() < 1e-3
    exp8 = orc.to_uint8(out["rgb"].cpu().numpy())
    assert np.abs(out["rgb_uint8"].cpu().numpy().astype(int) - exp8.astype(int)).max() <= 1
    bi = nb.batched_inference(models, emb, r, 64, 64, False, 32768, True)
    assert set(bi) == {"opacity_coarse", "rgb_fine", "depth_fine", "opacity_fine"}
    assert torch.equal(bi["rgb_fine"].view(H, W, 3), out["rgb"])


def test_sigma_query_and_loss_epilogue(models, emb, ws, dev):
    """SURVEY section 8f rows 3-4: dense sigma query (extract_color_mesh.py:127-140) and MSE/PSNR
    (losses.py:9-14, metrics.py:4-13)."""
    rs = np.random.RandomState(5)
    xyz = rs.uniform(-1.5, 1.5, (3000, 3)).astype(np.float32)
    got = nb.query_sigma(models[1], torch.from_numpy(xyz).to(dev)).cpu().numpy()
    x = np.concatenate([orc.embed(xyz, 10), orc.embed(np.zeros_like(xyz), 4)], -1)
    ref = orc.nerf_forward(ws[1], x)[:, -1]
    assert got.shape == (3000,)
    assert (np.abs(got - ref) / (1 + np.abs(ref))).max() < 2e-3
    # drop-in two-step path gives the same numbers to the same tolerance
    with torch.no_grad():
        two = models[1](torch.cat([emb[0](torch.from_numpy(xyz).to(dev)), emb[1](torch.zeros(3000, 3, device=dev))], 1))
    assert (np.abs(two[:, -1].cpu().numpy() - ref) / (1 + np.abs(ref))).max() < 2e-3
    rays = torch.from_numpy(orc.make_rays(500, 4)).to(dev)
    with torch.no_grad():
        res = nb.render_rays(models, emb, rays, 64, False, 0, 0, 64, 32768, True)
    tgt = torch.rand(500, 3, device=dev)
    m = nb.mse_psnr(res, tgt)
    mc = float(((res["rgb_coarse"] - tgt) ** 2).mean())
    mf = float(((res["rgb_fine"] - tgt) ** 2).mean())
    assert abs(float(m["loss"]) - (mc + mf)) < 1e-5 * (mc + mf) + 1e-9
    assert abs(float(m["psnr"]) - (-10 * np.log10(mf))) < 1e-4


def _build_trainable(ws, dev):
    out = []
    for w in ws:
        net = nb.NeRF()
        net.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        out.append(net.to(dev))
    return out


def _named_grads(models):
    return {f"{tag}.{k}": p.grad.detach().cpu().numpy() for tag, m in zip(("coarse", "fine"), models)
            for k, p in m.named_parameters()}


@pytest.mark.parametrize("name", list(cases.GRAD_CASES))
@pytest.mark.parametrize("fused_loss", [False, True])
def test_training_step_gradients_vs_reference_golden(name, fused_loss, ws, emb, dev):
    """The fused training step (forward with activation capture + sm_90a backward: compositing
    backward, wgmma dgrad chain, wgmma wgrad) against the 48 .grad tensors of the UNMODIFIED
    reference's loss.backward() (tests/golden/grad_*.npz, train.py:103-117 / losses.py:9-14), on the
    same rays, targets and replayed random draws.  Bar: per-tensor relative L2 error < 5e-2 and
    cosine > 0.998 (16-bit operands vs fp32), loss within 1e-3 relative."""
    from oracle import nerf_oracle_grad as og
    n, kind, rseed, K, perturb, noise, wb = cases.GRAD_CASES[name]
    rays, target, randoms, ref_loss, ref_out, ref_grads = cases.load_grad_case(name)
    m = _build_trainable(ws, dev)
    rnd = to_dev(randoms, dev)
    r, t = torch.from_numpy(rays).to(dev), torch.from_numpy(target).to(dev)
    if fused_loss:
        out = nb.render_rays_loss(m, emb, r, t, 64, False, perturb, noise, K, 32768, wb, randoms=rnd)
        loss = out["loss"]
        assert abs(float(out["psnr"]) + 10 * np.log10(float(out["mse_fine"]))) < 1e-4
    else:
        out = nb.render_rays(m, emb, r, 64, False, perturb, noise, K, 32768, wb, randoms=rnd)
        loss = ((out["rgb_coarse"] - t) ** 2).mean() + ((out["rgb_fine"] - t) ** 2).mean()
    loss.backward()
    torch.cuda.synchronize()
    assert abs(float(loss.detach()) - ref_loss) < 1e-3 * ref_loss, (float(loss.detach()), ref_loss)
    for k in ("rgb_coarse", "rgb_fine"):
        # under sigma noise a sign flip of sigma+noise at the far plane (delta = 1e10) moves single rays by
        # their remaining transmittance (DESIGN.md section 5 (ii), (iii)): bound the bulk there
        mx, p999, mean = cases.error_stats(out[k].detach().cpu().numpy(), ref_out[k])
        assert (mx < 1e-3) if noise == 0 else (mx < 5e-3 and mean < 1e-4), (k, mx, mean)
    grads = _named_grads(m)
    assert set(grads) == set(ref_grads)
    rows, (rel, cos) = og.grad_compare(grads, ref_grads)
    worst = max(rows.items(), key=lambda kv: kv[1][0])
    print(f"{name} fused_loss={fused_loss}: global rel {rel:.3e} cos {cos:.6f}; worst {worst[0]} rel {worst[1][0]:.3e}")
    # Bars.  Whole gradient: relative L2 error < 5e-3, cosine > 0.9999.  Per tensor: < 8e-2 / > 0.997 - the fp16
    # forward flips the ReLU mask of the ~1e-4 of pre-activations that lie within fp16 rounding of zero, each flip
    # is an O(1) error in that element's gradient, i.e. ~1e-2 relative L2 per layer, accumulating towards layer 1.
    # The kernels themselves are pinned much tighter by tests/test_gpu_train_stages.py: every stage against float64
    # on the device's own stored inputs (same masks), every element of every .grad tensor.
    assert rel < 5e-3 and cos > 0.9999, (rel, cos)
    for k, (rr, cc) in rows.items():
        assert np.isfinite(grads[k]).all(), k
        assert rr < 8e-2 and cc > 0.997, f"{k}: rel {rr:.3e} cos {cc:.5f}"


@pytest.fixture(scope="module")
def trained_ws():
    if not cases.have_trained():
        pytest.skip("tests/golden/trained_weights.npz not generated")
    return cases.trained_weights()


@pytest.mark.parametrize("name", list(cases.TRAINED_CASES))
def test_trained_weights_render_vs_reference_golden(name, trained_ws, emb, dev):
    """TRAINED weights (8000 steps of this repository's own training step on a procedural scene: larger norms,
    sharp density, high positional frequencies in use - what the fp16 MLP and the final.dir folding are most
    sensitive to) through the fused kernel against the unmodified reference's outputs."""
    n, rseed, K, perturb, noise, tt = cases.TRAINED_CASES[name]
    rays, randoms, ref = cases.load_case(name)
    m = []
    for w in trained_ws:
        net = nb.NeRF()
        net.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        m.append(net.to(dev).eval())
    with torch.no_grad():
        out = nb.render_rays(m, emb, torch.from_numpy(rays).to(dev), 64, False, perturb, noise, K, 32768, True,
                             test_time=tt, randoms=to_dev(randoms, dev))
    torch.cuda.synchronize()
    assert set(out) == set(ref)
    for k, v in ref.items():
        mx, p999, mean = cases.error_stats(out[k].cpu().numpy(), v)
        print(f"{name}/{k}: vs reference max {mx:.2e} p99.9 {p999:.2e} mean {mean:.2e}")
        # rgb: the north-star bar (1e-3 abs).  opacity / depth on TRAINED weights: the density is sharp
        # (sigma of tens per unit length), so the fp16 rounding of the hidden activations (2^-11 relative)
        # moves single alphas by ~1e-3; rounding ONLY the activations of the fp32 oracle to fp16 gives
        # opacity 1.3e-3 / depth 4.8e-3 max on trained_test (tools/fp16_error_model.py), means are 2e-5 / 8e-5.
        bar = {"rgb": 1e-3, "opacity": 2.5e-3, "depth": 1e-2 if noise == 0 else 2e-2}[k.split("_")[0]]
        assert mx < bar, f"{name}/{k}: max {mx:.3e}"
        assert mean < {"rgb": 1e-4, "opacity": 1e-4, "depth": 5e-4}[k.split("_")[0]], f"{name}/{k}: mean {mean:.3e}"
    assert orc.psnr(out["rgb_fine"].cpu().numpy(), ref["rgb_fine"]) > 60.0


def test_trained_weights_gradients_vs_reference_golden(trained_ws, emb, dev):
    """The training step on trained weights against the reference's loss.backward() (grad_trained.npz)."""
    from oracle import nerf_oracle_grad as og
    name, n, rseed, K, perturb, noise = cases.TRAINED_GRAD
    rays, target, randoms, ref_loss, ref_out, ref_grads = cases.load_grad_case(name)
    m = _build_trainable(trained_ws, dev)
    out = nb.render_rays_loss(m, emb, torch.from_numpy(rays).to(dev), torch.from_numpy(target).to(dev), 64, False,
                              perturb, noise, K, 32768, True, randoms=to_dev(randoms, dev))
    out["loss"].backward()
    torch.cuda.synchronize()
    assert abs(float(out["loss"].detach()) - ref_loss) < 1e-3 * ref_loss
    for k in ("rgb_coarse", "rgb_fine"):
        # ray 16 of this batch grazes a sphere: the fp32 oracle with fp16-rounded big-layer operands is off by
        # 1.58e-3 there (tools/fp16_error_model.py on this case; the kernel: 1.59e-3), the other 63 rays stay
        # below 4e-4.  The bar for this batch is therefore the error model's, not 1e-3: see DESIGN.md section 5.
        mx, p999, mean = cases.error_stats(out[k].detach().cpu().numpy(), ref_out[k])
        srt = np.sort(np.abs(out[k].detach().cpu().numpy() - ref_out[k]).max(-1))
        print(f"{name}/{k}: max {mx:.2e} second-worst ray {srt[-2]:.2e} mean {mean:.2e}")
        assert mx < 2.5e-3 and srt[-2] < 1e-3 and mean < 1e-4, (k, mx, srt[-2], mean)
    grads = _named_grads(m)
    rows, (rel, cos) = og.grad_compare(grads, ref_grads)
    worst = max(rows.items(), key=lambda kv: kv[1][0])
    print(f"{name}: global rel {rel:.3e} cos {cos:.6f}; worst {worst[0]} rel {worst[1][0]:.3e}")
    assert rel < 2e-2 and cos > 0.9995, (rel, cos)
    for k, (rr, cc) in rows.items():
        assert np.isfinite(grads[k]).all(), k
        assert rr < 1.5e-1 and cc > 0.99, f"{k}: rel {rr:.3e} cos {cc:.5f}"


def test_training_step_is_deterministic_and_matches_oracle(ws, emb, dev):
    """Two identical steps give bit-identical gradients (fixed-order reductions, no float atomics);
    the gradients also agree with the numpy oracle's hand-derived backward on a batch that is not one
    of the goldens (odd ray count: padded sample rows)."""
    from oracle import nerf_oracle_grad as og
    n = 77
    rays = orc.make_rays(n, 41)
    rs = np.random.RandomState(7)
    target = rs.uniform(0, 1, (n, 3)).astype(np.float32)
    randoms = {"perturb_rand": rs.rand(n, 64).astype(np.float32), "u_rand": rs.rand(n, 64).astype(np.float32)}
    runs = []
    for _ in range(2):
        m = _build_trainable(ws, dev)
        out = nb.render_rays_loss(m, emb, torch.from_numpy(rays).to(dev), torch.from_numpy(target).to(dev), 64, False,
                                  1.0, 0.0, 64, 32768, True, randoms=to_dev(randoms, dev))
        out["loss"].backward()
        torch.cuda.synchronize()
        runs.append((float(out["loss"]), _named_grads(m)))
    assert runs[0][0] == runs[1][0]
    for k in runs[0][1]:
        np.testing.assert_array_equal(runs[0][1][k], runs[1][1][k], err_msg=k)
    loss, _, ref = og.render_rays_loss_grad(ws, rays, target, 64, False, 1.0, 0.0, 64, True, randoms)
    assert abs(runs[0][0] - loss) < 1e-3 * loss
    rows, (rel, cos) = og.grad_compare(runs[0][1], ref)
    assert rel < 5e-2 and cos > 0.998, (rel, cos)


def test_upstream_gradients_of_all_outputs(ws, emb, dev):
    """backward(d_rgb, d_depth, d_opacity) for both passes: a loss that uses every result tensor,
    fused backward vs plain torch autograd (autograd_impl='torch') on the same inputs."""
    n = 96
    rays = torch.from_numpy(orc.make_rays(n, 14)).to(dev)
    g = torch.Generator(device=dev).manual_seed(5)
    rnd = {"perturb_rand": torch.rand(n, 64, device=dev, generator=g), "u_rand": torch.rand(n, 64, device=dev, generator=g)}
    wts = {k: torch.randn(sh, device=dev, generator=g) for k, sh in
           (("rgb_coarse", (n, 3)), ("depth_coarse", (n,)), ("opacity_coarse", (n,)),
            ("rgb_fine", (n, 3)), ("depth_fine", (n,)), ("opacity_fine", (n,)))}
    grads = {}
    for impl in ("fused", "torch"):
        m = _build_trainable(ws, dev)
        out = nb.render_rays(m, emb, rays, 64, False, 1.0, 0.0, 64, 32768, False, randoms=rnd, autograd_impl=impl)
        loss = sum((out[k] * w).sum() for k, w in wts.items()) / n
        loss.backward()
        grads[impl] = [p.grad.detach().clone() for net in m for p in net.parameters()]
    num = sum(float(((a - b) ** 2).sum()) for a, b in zip(grads["fused"], grads["torch"]))
    den = sum(float((b ** 2).sum()) for b in grads["torch"])
    assert (num / den) ** 0.5 < 5e-2, (num / den) ** 0.5


def test_packed_weights_follow_data_copy_updates(ws, emb, dev):
    """ADVICE r1: optimisers that update through p.data.copy_ (the reference's RAdam / Ranger,
    utils/optimizers.py:88,163,242) do not bump Tensor._version; trainable networks are re-packed on
    every use, frozen ones after invalidate_packed()."""
    m = _build_trainable(ws, dev)
    rays = torch.from_numpy(orc.make_rays(64, 1)).to(dev)
    with torch.no_grad():
        a = nb.render_rays(m, emb, rays, 64, False, 0, 0, 64)["rgb_fine"].clone()
        v0 = m[1].rgb[0].bias._version
        m[1].rgb[0].bias.data.copy_(m[1].rgb[0].bias.data + 1.0)
        assert m[1].rgb[0].bias._version == v0                       # the blind spot
        b = nb.render_rays(m, emb, rays, 64, False, 0, 0, 64)["rgb_fine"].clone()
        assert float((a - b).abs().max()) > 1e-2
        for net in m:
            net.requires_grad_(False)
        c = nb.render_rays(m, emb, rays, 64, False, 0, 0, 64)["rgb_fine"].clone()
        assert torch.equal(b, c)
        m[1].rgb[0].bias.data.copy_(m[1].rgb[0].bias.data - 1.0)
        nb.invalidate_packed(m[1])
        d = nb.render_rays(m, emb, rays, 64, False, 0, 0, 64)["rgb_fine"]
        assert float((a - d).abs().max()) < 1e-6


def test_reference_style_module_through_render_rays(ws, emb, dev):
    """render_rays accepts a network built the way the reference builds its own NeRF (models/nerf.py:58-81:
    nn.Sequential(Linear, ReLU) attributes named xyz_encoding_i, ...), not only this package's class: the 24
    parameters are found by attribute name.  Same weights -> bit-identical result; float64 inputs are rejected."""
    from torch import nn

    class RefLike(nn.Module):
        def __init__(self):
            super().__init__()
            for i in range(8):
                n_in = 63 if i == 0 else (256 + 63 if i == 4 else 256)
                setattr(self, f"xyz_encoding_{i + 1}", nn.Sequential(nn.Linear(n_in, 256), nn.ReLU(True)))
            self.xyz_encoding_final = nn.Linear(256, 256)
            self.dir_encoding = nn.Sequential(nn.Linear(256 + 27, 128), nn.ReLU(True))
            self.sigma = nn.Linear(256, 1)
            self.rgb = nn.Sequential(nn.Linear(128, 3), nn.Sigmoid())

    ours, theirs = [], []
    for w in ws:
        sd = {k: torch.from_numpy(v) for k, v in w.items()}
        a, b = nb.NeRF(), RefLike()
        a.load_state_dict(sd)
        b.load_state_dict(sd)
        ours.append(a.to(dev).eval())
        theirs.append(b.to(dev).eval())
    rays = torch.from_numpy(orc.make_rays(100, 5)).to(dev)
    with torch.no_grad():
        x = nb.render_rays(ours, emb, rays, 64, False, 0, 0, 64, 32768, True)
        y = nb.render_rays(theirs, emb, rays, 64, False, 0, 0, 64, 32768, True)
    for k in x:
        assert torch.equal(x[k], y[k]), k
    with pytest.raises(ValueError):
        nb.searchsorted(torch.zeros(1, 3, device=dev, dtype=torch.float64), torch.zeros(1, 3, device=dev, dtype=torch.float64))


def test_fused_adam_matches_torch_adam(dev):
    """nerfb200_adam_step against torch.optim.Adam (the reference's optimiser, utils/__init__.py:16-18) on the
    48 parameter tensors of two NeRFs, 5 steps, with weight decay: same arithmetic, fp32 rounding only."""
    torch.manual_seed(3)
    a = [nb.NeRF().to(dev), nb.NeRF().to(dev)]
    b = [nb.NeRF().to(dev), nb.NeRF().to(dev)]
    for x, y in zip(a, b):
        y.load_state_dict(x.state_dict())
    pa = [p for m in a for p in m.parameters()]
    pb = [p for m in b for p in m.parameters()]
    oa = nb.FusedAdam(pa, lr=5e-4, eps=1e-8, weight_decay=1e-3)
    ob = torch.optim.Adam(pb, lr=5e-4, eps=1e-8, weight_decay=1e-3)
    g = torch.Generator(device=dev).manual_seed(1)
    for _ in range(5):
        for x, y in zip(pa, pb):
            gr = torch.randn(x.shape, device=dev, generator=g) * 1e-3
            x.grad = gr.clone()
            y.grad = gr.clone()
        oa.step()
        ob.step()
    for x, y in zip(pa, pb):
        assert torch.allclose(x, y, rtol=1e-5, atol=1e-7), float((x - y).abs().max())
    assert oa.state[pa[0]]["step"] == 5


def test_status_word_is_checked(dev):
    lib = _lib.load()
    assert lib.nerfb200_check_status() == 0


def test_fused_training_gradients_match_torch_autograd(ws, emb, dev):
    """FusedRenderFunction (fused forward with activation capture + hand-written sm_90a backward) against
    plain torch fp32 autograd through the same maths (the reference's graph, models/rendering.py +
    models/nerf.py), same pre-drawn randoms.  Per-parameter relative L2 error and cosine."""
    build = lambda: _build_trainable(ws, dev)
    n = 256
    rays = torch.from_numpy(orc.make_rays(n, 12)).to(dev)
    g = torch.Generator(device=dev).manual_seed(3)
    rnd = {"perturb_rand": torch.rand(n, 64, device=dev, generator=g), "u_rand": torch.rand(n, 64, device=dev, generator=g),
           "noise_coarse": torch.randn(n, 64, device=dev, generator=g), "noise_fine": torch.randn(n, 128, device=dev, generator=g)}
    tgt = torch.rand(n, 3, device=dev, generator=g)
    grads = {}
    outs = {}
    for impl in ("fused", "torch"):
        m = build()
        # noise_std = 0 (the README Blender recipe): with sigma noise the 1e10 far-plane delta turns
        # fp16-vs-fp32 sign flips of sigma+noise into O(1) per-ray differences (DESIGN.md section 5)
        out = nb.render_rays(m, emb, rays, 64, False, 1.0, 0.0, 64, 32768, True, randoms=rnd, autograd_impl=impl)
        loss = ((out["rgb_coarse"] - tgt) ** 2).mean() + ((out["rgb_fine"] - tgt) ** 2).mean()    # losses.py:9-14
        loss.backward()
        grads[impl] = [p.grad.detach().clone() for net in m for p in net.parameters()]
        outs[impl] = {k: v.detach() for k, v in out.items()}
    # forward values: fp16 tensor-core path vs torch fp32 at random (perturbed) depths; rays whose
    # far-plane sigma is ~0 flip alpha_last (DESIGN.md section 5 (ii)) and move by T_last, hence 5e-3 here
    # (reference parity proper is pinned by the golden tests above)
    for k in outs["torch"]:
        diff = (outs["fused"][k] - outs["torch"][k]).abs().flatten()
        if k.startswith("rgb"):
            assert float(diff.max()) < 5e-3, k
        else:   # depth / opacity move by T_last * far when alpha_last flips: check the bulk
            assert float(torch.quantile(diff, 0.98)) < 5e-3, k
    names = [f"{i}.{k}" for i in range(2) for k in orc.PARAM_KEYS]
    worst = 0.0
    for name, a, b in zip(names, grads["fused"], grads["torch"]):
        assert a.shape == b.shape and torch.isfinite(a).all(), name
        rel = float((a - b).norm() / (b.norm() + 1e-12))
        cos = float((a * b).sum() / (a.norm() * b.norm() + 1e-20))
        worst = max(worst, rel)
        assert rel < 5e-2 and cos > 0.998, f"{name}: rel {rel:.3e} cos {cos:.5f}"
    print(f"worst relative gradient error {worst:.3e}")


def test_sharded_render_over_nccl_equals_single_gpu():
    """SURVEY section 8e on real hardware: 2 ranks (one process per GPU, torchrun, NCCL), contiguous
    ray shards + ONE all-gather == the single-GPU render, bit-exactly (tools/nccl_check.py).
    Needs 2 GPUs on the box; skipped otherwise (the gloo twin runs on CPU in test_sharded_gloo.py)."""
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29731", "tools/nccl_check.py"],
                       cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.count("NCCL_CHECK_OK") == 2, r.stdout[-2000:] + r.stderr[-2000:]
