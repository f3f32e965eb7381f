"""skip="samples" on the device (nerf_pl_b200.culling.render_samples, csrc/sample_skip_kernels.cuh): with nothing to
skip it is render_rays bit for bit; on a partial grid its evaluated set is the float64 rule (tests/sample_skip_ref.py)
on the device's own points, its evaluated samples are the unskipped path's, skipped weights are 0, its fine depths are
the fused kernel's merge of its own weights; dead rays, degenerate rays, chunking and batch order; the trained scene."""
import numpy as np
import pytest
import torch

import bench
from nerf_pl_b200 import culling
from oracle import nerf_oracle as orc
from tests import cases
from tests import occupancy_ref as oc
from tests import render_tape as rt
from tests import sample_skip_ref as sk

pytestmark = pytest.mark.gpu
CUBE = ((-1.5, 1.5),) * 3


def _nb():
    import nerf_pl_b200 as nb
    return nb


def _emb():
    return [_nb().Embedding(3, 10), _nb().Embedding(3, 4)]


_M = {}


def _models(kind="random"):
    if kind not in _M:
        ws = cases.trained_weights() if kind == "trained" else [orc.make_weights(21), orc.make_weights(22)]
        ms = []
        for w in ws:
            m = _nb().NeRF()
            m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
            ms.append(m.cuda().eval())
        _M[kind] = ms
    return _M[kind]


def _grid(fill, ranges, N=33, seed=0):
    """A grid over `ranges`: every cell occupied (fill = 1.0) or a random fraction of them."""
    rng = np.random.default_rng(seed)
    sigma = np.where(rng.random((N, N, N)) < fill, 5.0, 0.0).astype(np.float32)
    return _nb().pack_occupancy(torch.from_numpy(sigma).cuda(), *ranges, 1.0, 0)


def _rays(kind, n, seed):
    if kind == "ndc":
        r = orc.make_rays(n, seed).copy()
        r[:, 6], r[:, 7] = 0.0, 1.0
        return torch.from_numpy(r).cuda()
    return torch.from_numpy(bench.blender_rays(n, seed)).cuda()


def _plain(models, rays, S, K, use_disp, white_back, test_time):
    with torch.no_grad():
        return _nb().render_rays(models, _emb(), rays, S, use_disp, 0, 0, K, 32768, white_back, test_time=test_time,
                                 match_reference_rng=False, extras=True)


def _same(a, b):
    """Bit for bit, NaN included."""
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _samples(models, rays, grid, S, K, use_disp, white_back, test_time, **kw):
    return culling.render_samples(models, rays, grid, S, use_disp, K, white_back, test_time, extras=True, **kw)


SHAPES = [(S, K) for S in (32, 64, 128) for K in range(0, 193 - S, 32)]     # every pair samples_shape_ok accepts


@pytest.mark.parametrize("S,K", SHAPES)
@pytest.mark.parametrize("kind", ["blender", "ndc"])
def test_nothing_to_skip_is_render_rays_bit_for_bit(S, K, kind):
    rays = _rays(kind, 700, 5)
    box = ((-1e4, 1e4),) * 3
    grid = _grid(1.0, box, N=3)
    for test_time, use_disp, white_back in ((True, False, True), (False, True, False), (False, False, True)):
        if kind == "blender" and use_disp:
            continue
        want = _plain(_models(), rays, S, K, use_disp, white_back, test_time)
        got = _samples(_models(), rays, grid, S, K, use_disp, white_back, test_time)
        assert got["live_samples"] == (700 * S, 700 * (S + K) if K else 0)
        for k, v in want.items():
            assert _same(got[k], v), (k, test_time, use_disp, white_back)
        culled = _nb().render_rays_culled(_models(), _emb(), rays, grid, S, use_disp, K, white_back, test_time,
                                          skip="samples", extras=True)
        for k, v in want.items():
            assert _same(culled[k], v), k


@pytest.mark.parametrize("test_time", [True, False])
@pytest.mark.parametrize("S,K", [(64, 128), (32, 64)])
def test_stages_on_a_partial_grid(S, K, test_time):
    rays = _rays("blender", 600, 7)
    ranges = ((-2.0, 2.0), (2.0, -2.0), (-1.5, 2.5))
    grid = _grid(0.05, ranges, N=17, seed=3)
    full = _grid(1.0, ((-1e4, 1e4),) * 3, N=3)
    got = _samples(_models(), rays, grid, S, K, False, True, test_time, per_sample=True)
    ref = _samples(_models(), rays, full, S, K, False, True, test_time, per_sample=True)
    words = grid.bits.cpu().numpy()
    rn = rays.cpu().numpy()
    zc = sk.z_base(rn, S)
    # the evaluated set is the float64 rule on the device's own points
    ev_c = sk.mask_bits(got["mask_coarse"].cpu().numpy(), S)
    assert np.array_equal(ev_c, sk.evaluated(rn, zc, words, grid.N, grid.ranges))
    zf = got["z_vals_fine"].cpu().numpy()
    ev_f = sk.mask_bits(got["mask_fine"].cpu().numpy(), S + K)
    assert np.array_equal(ev_f, sk.evaluated(rn, zf, words, grid.N, grid.ranges))
    assert 0 < ev_c.mean() < 0.9 and 0 < ev_f.mean()
    assert got["live_samples"] == (int(ev_c.sum()), int(ev_f.sum()))
    # evaluated coarse samples are the unskipped path's (same rays, same depths), skipped ones are 0 with weight 0
    sc, rc = got["samples_coarse"].cpu().numpy(), ref["samples_coarse"].cpu().numpy()
    assert np.array_equal(sc[ev_c], rc[ev_c]) and not sc[~ev_c].any()
    wc = got["weights_coarse"].cpu().numpy()
    assert not wc[~ev_c].any()
    sf = got["samples_fine"].cpu().numpy()
    assert not sf[~ev_f].any() and not got["weights_fine"].cpu().numpy()[~ev_f].any()
    # z_vals_fine: the fused kernel's resampling and merge of the path's own coarse weights
    want_z, _, _ = rt.z_fine(wc, zc, rt.fine_uniforms(rn.shape[0], K, 0.0))
    assert np.array_equal(zf, want_z)
    # compositing within render_tape's float64 bounds
    d = rn[:, 3:6]
    for S_, s_all, z_, w_, pre in ((S, sc, zc, wc, "coarse"), (S + K, sf, zf, got["weights_fine"].cpu().numpy(), "fine")):
        if pre == "coarse" and test_time:
            continue
        e = rt.composite_errors(s_all[..., 3], s_all[..., :3], z_, d, None, 0.0, True, w_,
                                got[f"rgb_{pre}"].cpu().numpy(), got[f"depth_{pre}"].cpu().numpy(),
                                got[f"opacity_{pre}"].cpu().numpy())
        assert not rt.composite_violations(e), (pre, e)


def test_evaluated_fine_samples_are_the_plain_kernels():
    """A sample's value depends only on its ray and depth: render the partial path's fine depths with nothing to skip
    (a fresh coarse pass is not involved: compare through the compacted MLP on the same rows)."""
    rays = _rays("blender", 300, 8)
    grid = _grid(0.05, CUBE, N=17, seed=4)
    full = _grid(1.0, ((-1e4, 1e4),) * 3, N=3)
    a = _samples(_models(), rays, grid, 64, 64, False, False, False, per_sample=True)
    b = _samples(_models(), rays, full, 64, 64, False, False, False, per_sample=True)
    ev = sk.mask_bits(a["mask_fine"].cpu().numpy(), 128)
    same = (a["z_vals_fine"] == b["z_vals_fine"]).cpu().numpy()   # depths both paths evaluated
    sel = ev & same
    assert sel.sum() > 100
    assert np.array_equal(a["samples_fine"].cpu().numpy()[sel], b["samples_fine"].cpu().numpy()[sel])


def test_dead_rays_all_skipped_rays_and_no_mlp_launch():
    nb = _nb()
    lib = nb._lib.load()
    rays = _rays("blender", 500, 9)
    grid = _grid(0.03, CUBE, N=33, seed=5)
    out = nb.render_rays_culled(_models(), _emb(), rays, grid, 64, False, 64, True, True, skip="samples")
    live_idx, _ = nb.cull_rays(rays, grid)
    assert out["live"] == live_idx.numel() and torch.equal(out["live_idx"], live_idx)
    dead = torch.ones(500, dtype=torch.bool, device="cuda")
    dead[live_idx] = False
    want = oc.vacuum_results(int(dead.sum()), ["opacity_coarse", "rgb_fine", "depth_fine", "opacity_fine"], True)
    for k, v in want.items():
        assert np.array_equal(out[k][dead].cpu().numpy(), v), k
    # a live ray with every sample skipped gets the vacuum value, and without evaluated samples no MLP runs
    flag = torch.zeros(500, dtype=torch.uint8, device="cuda")
    before = lib.nerfb200_launch_count()
    for m in _models():                                      # the weight-image packs render_samples itself makes
        nb.nerf.packed_weights(m)
    packs = lib.nerfb200_launch_count() - before
    before = lib.nerfb200_launch_count()
    res = culling.render_samples(_models(), rays, grid, 64, False, 64, True, False, live_flag=flag, extras=True)
    assert lib.nerfb200_launch_count() - before == 5 + packs   # classify, scan, coarse stage, scan, fine stage
    assert res["live_samples"] == (0, 0)
    want = oc.vacuum_results(500, ["rgb_coarse", "depth_coarse", "opacity_coarse", "rgb_fine", "depth_fine",
                                   "opacity_fine"], True)
    for k, v in want.items():
        assert np.array_equal(res[k].cpu().numpy(), v), k
    assert not res["weights_coarse"].any() and not res["weights_fine"].any()
    # no live ray at all: cull and scatter only
    empty = _grid(0.0, CUBE, N=9)
    before = lib.nerfb200_launch_count()
    out = nb.render_rays_culled(_models(), _emb(), rays, empty, 64, False, 64, True, skip="samples")
    assert lib.nerfb200_launch_count() - before == 3 and out["live"] == 0 and out["live_samples"] == (0, 0)


def test_degenerate_rays_equal_the_plain_render():
    rays = _rays("blender", 64, 10).cpu().numpy()
    bad = rays[:12].copy()
    bad[0, 0] = np.nan
    bad[1, 4] = np.inf
    bad[2, 7] = np.inf
    bad[3, 6] = np.nan
    bad[4, 6], bad[4, 7] = 6.0, 2.0                 # far <= near
    bad[5, 6] = bad[5, 7] = 4.0
    bad[6, 3:6] = 3e19                              # |d|^2 overflows
    bad[7, 3:6] = np.array([1e30, 0, 0], np.float32)  # 1e10 |d| overflows
    bad[8, 5] = -np.inf
    bad[9, 1] = np.inf
    allr = torch.from_numpy(np.concatenate([rays, bad])).cuda()
    grid = _grid(0.05, CUBE, N=17, seed=6)
    for S, K, test_time in ((64, 64, False), (64, 128, True)):
        want = _plain(_models(), allr, S, K, False, True, test_time)
        got = _samples(_models(), allr, grid, S, K, False, True, test_time)
        for k, v in want.items():
            a, b = got[k][64:74].cpu().numpy(), v[64:74].cpu().numpy()
            assert np.array_equal(a.view(np.int32), b.view(np.int32)), k


def test_independent_of_chunk_and_batch_position(monkeypatch):
    rays = _rays("blender", 900, 11)
    grid = _grid(0.05, CUBE, N=17, seed=7)
    base = _samples(_models(), rays, grid, 64, 128, False, True, False)
    monkeypatch.setattr(culling, "_SAMPLE_CHUNK", 257)
    chunked = _samples(_models(), rays, grid, 64, 128, False, True, False)
    perm = torch.randperm(900, generator=torch.Generator().manual_seed(0)).cuda()
    permuted = _samples(_models(), rays[perm].contiguous(), grid, 64, 128, False, True, False)
    for k, v in base.items():
        if k == "live_samples":
            assert chunked[k] == v and permuted[k] == v
            continue
        assert _same(chunked[k], v), k
        assert _same(permuted[k], v[perm]), k


# ---- the trained scene (tests/test_gpu_occupancy.py's grid: N = 128 over the box, sigma > 1, dilate 1) ----------
_GRID = []


def _trained_grid():
    if not _GRID:
        _GRID.append(_nb().occupancy_grid(_models("trained")[1], 128, *CUBE, 1.0, 1))
    return _GRID[0]


# Mean errors of "samples" against the plain render (max over the channels for rgb), pinned at about three times the
# largest value measured on an NVIDIA H100 80GB HBM3 at 700 W: view 61 (the worst of the views measured) gives
# |d rgb_fine| 3.2e-4, |d opacity_fine| 1.0e-2, |d depth_fine| 6.0e-2, view 62 1.3e-4, 7.4e-4 and 3.5e-3.
SAMPLES_MEAN_RGB = 1e-3
SAMPLES_MEAN_OPACITY = 3e-2
SAMPLES_MEAN_DEPTH = 2e-1


@pytest.mark.parametrize("seed", [61, 62])
def test_trained_scene(seed):
    nb = _nb()
    if not cases.have_trained():
        pytest.skip("no trained weights")
    rays = torch.from_numpy(bench.blender_rays(0, seed, W=160, H=160, pixels="all")).cuda()
    grid = _trained_grid()
    plain = _plain(_models("trained"), rays, 64, 128, False, True, True)
    out = nb.render_rays_culled(_models("trained"), _emb(), rays, grid, 64, False, 128, True, True, skip="samples")
    n = rays.shape[0]
    fc, ff = out["live_samples"][0] / (64 * n), out["live_samples"][1] / (192 * n)
    e_rgb = (out["rgb_fine"] - plain["rgb_fine"]).abs().amax(1)
    e_op = (out["opacity_fine"] - plain["opacity_fine"]).abs()
    e_d = (out["depth_fine"] - plain["depth_fine"]).abs()
    print(f"view {seed}: live rays {out['live'] / n:.3f}, evaluated samples coarse {fc:.3f} fine {ff:.3f}; "
          f"|d rgb| mean {float(e_rgb.mean()):.3e} max {float(e_rgb.max()):.3e}, |d opacity| mean "
          f"{float(e_op.mean()):.3e} max {float(e_op.max()):.3e}, |d depth| mean {float(e_d.mean()):.3e} max "
          f"{float(e_d.max()):.3e}")
    assert fc < 0.9 and ff < 0.9
    assert float(e_rgb.mean()) < SAMPLES_MEAN_RGB
    assert float(e_op.mean()) < SAMPLES_MEAN_OPACITY
    assert float(e_d.mean()) < SAMPLES_MEAN_DEPTH


def test_inference_entries_take_skip():
    nb = _nb()
    grid = _trained_grid() if cases.have_trained() else _grid(0.05, CUBE, N=17)
    models = _models("trained") if cases.have_trained() else _models()
    rays = torch.from_numpy(bench.blender_rays(0, 70, W=48, H=48, pixels="all")).cuda()
    a = nb.batched_inference(models, _emb(), rays, 64, 64, False, occupancy=grid, skip="samples")
    b = nb.render_rays_culled(models, _emb(), rays, grid, 64, False, 64, False, True, skip="samples")
    for k in ("opacity_coarse", "rgb_fine", "depth_fine", "opacity_fine"):
        assert torch.equal(a[k], b[k]), k
    assert a["live_samples"] == b["live_samples"]
    img = nb.render_image(models, _emb(), 48, 48, float(bench.IMG_W), np.eye(3, 4), 2.0, 6.0, 64, 64,
                          occupancy=grid, skip="samples")
    assert "live_samples" in img and img["rgb"].shape == (48, 48, 3)
