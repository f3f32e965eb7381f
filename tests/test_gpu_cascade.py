"""Cascaded occupancy grids on the device (levels=, DESIGN.md §10h) against their float64 restatement
(tests/cascade_ref.py) and against one-level grids (pytest -m gpu).

- L = 1: the package's calls equal raw one-level calls of the entries bit for bit.
- L > 1 without new tolerances: a cascade whose levels are all full behaves as a full one-level grid over the last
  level's box, and one whose outer levels are empty as the one-level grid over level 0.
- Against the restatement: per-sample classification, cull flags, no culled ray with an evaluated sample, and the
  density grid update bit for bit.
- CapturedTrainStep(occupancy=DensityGrid(levels=4), update_every=3) equals the eager loop bit for bit.
"""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import bench
import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib, culling
from oracle import nerf_oracle as orc
from tests import cascade_ref as cr
from tests import cases
from tests import occupancy_ref as oc
from tests import sample_skip_ref as ss

pytestmark = pytest.mark.gpu
BOX = ((-0.6, 0.6), (0.7, -0.5), (-0.4, 0.8))            # y reversed
R6 = tuple(v for r in BOX for v in r)
HYPER = dict(lr=5e-4, eps=1e-8)


def _emb():
    return [nb.Embedding(3, 10), nb.Embedding(3, 4)]


def _random_models(seed=0):
    ms = []
    for s in (21 + seed, 22 + seed):
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in orc.make_weights(s).items()})
        ms.append(m.cuda())
    return ms


_TRAINED = []


def _trained_models():
    if not _TRAINED:
        for w in cases.trained_weights():
            m = nb.NeRF()
            m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
            _TRAINED.append(m.cuda().eval())
    return _TRAINED


def _grid(words, N, L, box=BOX):
    bits = torch.from_numpy(np.ascontiguousarray(np.asarray(words, np.uint32)).view(np.int32)).cuda()
    return nb.OccupancyGrid(bits, N, *box, levels=L)


def _random_words(rng, N, L, p):
    M = N - 1
    return cr.pack(np.stack([(rng.random((M, M, M)) < p) & ~cr.inner_mask(N, k) for k in range(L)]))


def _rays(n, seed):
    return torch.from_numpy(bench.blender_rays(n, seed)).cuda()


def _eq(a, b):
    """Bit-for-bit equality of two result dicts on their common tensor keys."""
    for k in a:
        if torch.is_tensor(a[k]) and k in b:
            assert torch.equal(a[k].view(torch.int32) if a[k].dtype == torch.float32 else a[k],
                               b[k].view(torch.int32) if b[k].dtype == torch.float32 else b[k]), k


def _cull_flags_old(rays, g):
    dev, n = rays.device, rays.shape[0]
    ws = _lib.workspace(_lib.load().nerfb200_cull_workspace_bytes(n), dev)
    flag = torch.empty(n, dtype=torch.uint8, device=dev)
    live = ctypes.c_int64()
    _lib.call("nerfb200_cull_count", dev, rays.data_ptr(), n, g.bits.data_ptr(), g.N, (ctypes.c_double * 6)(*g.ranges),
              ws.data_ptr(), ws.numel(), flag.data_ptr(), ctypes.byref(live))
    return flag


# ------------------------------------------------------------------------------------------- L = 1 is today
def test_one_level_grids_call_the_entries_as_before():
    """With L = 1 the package passes the grid size as it always did (grid_n() == N) and its results equal raw calls
    of the entries bit for bit: culling, packing, popcount, the density update and points, both masked grids."""
    N = 33
    model = _trained_models()[1]
    sigma = nb.sigma_grid(model, N, *BOX)
    g = nb.pack_occupancy(sigma, *BOX, sigma_threshold=2.0, dilate=1)
    lib = _lib.load()
    ws = _lib.workspace(lib.nerfb200_occupancy_workspace_bytes(N), "cuda")
    old = torch.empty_like(g.bits)
    _lib.call("nerfb200_occupancy_pack", sigma.device, sigma.data_ptr(), N, 2.0, 1, ws.data_ptr(), ws.numel(),
              old.data_ptr())
    assert torch.equal(old, g.bits) and g.levels == 1 and g.grid_n() == N and "levels" not in g.state_dict()
    cnt = torch.empty(1, dtype=torch.int64, device="cuda")
    _lib.call("nerfb200_occupancy_popcount", g.device, g.bits.data_ptr(), N, cnt.data_ptr())
    assert int(cnt.item()) / (N - 1) ** 3 == g.occupied_fraction()
    rays = _rays(8192, 3)
    assert torch.equal(_cull_flags_old(rays, g), nb.cull_rays(rays, g, return_flag=True)[2])
    # masked grids through the one-level entries
    for entry, ch in (("nerfb200_sigma_grid_masked", 1), ("nerfb200_rgb_sigma_grid_masked", 4)):
        out = torch.empty((17, 17, 17) if ch == 1 else (17, 17, 17, 4), device="cuda")
        wsm = _lib.workspace(lib.nerfb200_masked_grid_workspace_bytes(4096), "cuda")
        ev = ctypes.c_int64()
        _lib.call(entry, g.device, nb.packed_weights(model).data_ptr(), 17, _lib.ranges_host(*BOX), g.bits.data_ptr(),
                  N, (ctypes.c_double * 6)(*g.ranges), 4096, wsm.data_ptr(), wsm.numel(), out.data_ptr(),
                  ctypes.byref(ev))
        fn = nb.sigma_grid if ch == 1 else nb.rgb_sigma_grid
        new, n_new = fn(model, 17, *BOX, 4096, occupancy=g, return_evaluated=True)
        assert torch.equal(out, new) and ev.value == n_new
    # density grid: the one-level entries on a second grid's tensors
    a = nb.DensityGrid(17, *BOX, sigma_threshold=1.0, decay=0.9, dilate=1, seed=5)
    b = nb.DensityGrid(17, *BOX, sigma_threshold=1.0, decay=0.9, dilate=1, seed=5)
    wsd = _lib.workspace(lib.nerfb200_density_workspace_bytes(17, b.chunk), "cuda")
    xyz = torch.empty((16 ** 3, 3), device="cuda")
    _lib.call("nerfb200_density_points", b.device, 17, (ctypes.c_double * 6)(*b.ranges), b.key.data_ptr(), 0,
              16 ** 3, xyz.data_ptr())
    assert torch.equal(xyz, a.points())
    for _ in range(3):
        a.update(model)
        _lib.call("nerfb200_density_update", b.device, nb.packed_weights(model).data_ptr(), 17,
                  (ctypes.c_double * 6)(*b.ranges), 1.0, b.decay, 1, b.chunk, b.key.data_ptr(), b._density.data_ptr(),
                  b.bits.data_ptr(), wsd.data_ptr(), wsd.numel())
    assert torch.equal(a._density, b._density) and torch.equal(a.bits, b.bits) and torch.equal(a.key, b.key)
    assert a.density.shape == (16, 16, 16) and "levels" not in a.state_dict()


# ------------------------------------------------------------------------------------------- equivalences
def _full_cascade(N, L):
    return cr.pack(np.stack([~cr.inner_mask(N, k) for k in range(L)]))


def _full_one(N):
    return oc.pack_bits(np.ones((N - 1,) * 3, bool))


def _consumers(g, models, rays, rgbs):
    """Every consumer's output through grid g: cull flags, skip='samples' renders with and without early stop,
    render_rays_loss (outputs and gradients) and both masked grids."""
    out = {"flag": nb.cull_rays(rays, g, return_flag=True)[2]}
    r = nb.render_rays_culled(models, _emb(), rays, g, 64, False, 64, False, False, skip="samples", extras=True)
    out.update({f"fine_{k}": v for k, v in r.items() if torch.is_tensor(v)})
    r = nb.render_rays_culled(models[:1], _emb(), rays, g, 64, False, 0, False, False, skip="samples", early_stop=1e-3)
    out.update({f"stop_{k}": v for k, v in r.items() if torch.is_tensor(v)})
    for m in models:
        m.zero_grad(set_to_none=True)
    res = nb.render_rays_loss(models, _emb(), rays, rgbs, 64, False, 0.0, 0.0, 64, 32768, False, occupancy=g)
    res["loss"].backward()
    out["loss"] = res["loss"].detach().clone()
    for i, m in enumerate(models):
        for j, p in enumerate(m.parameters()):
            out[f"grad{i}_{j}"] = p.grad.clone()
    out["sigma_grid"] = nb.sigma_grid(models[1], 33, (-3.0, 3.0), (-2.0, 3.0), (-2.0, 2.5), occupancy=g)
    out["rgb_sigma_grid"] = nb.rgb_sigma_grid(models[1], 17, (-3.0, 3.0), (-2.0, 3.0), (-2.0, 2.5), occupancy=g)
    return out


@pytest.mark.parametrize("N, L", [(17, 3), (10, 2)])
def test_a_full_cascade_is_a_full_grid_over_its_last_level(N, L):
    models = _trained_models()
    rays = _rays(4096, 11)
    rgbs = torch.rand(4096, 3, generator=torch.Generator().manual_seed(12)).cuda()
    last = cr.pairs(cr.level_ranges(R6, L - 1))
    a = _consumers(_grid(_full_cascade(N, L), N, L), models, rays, rgbs)
    b = _consumers(_grid(_full_one(N), N, 1, last), models, rays, rgbs)
    _eq(a, b)
    assert int(a["flag"].sum()) > 0


@pytest.mark.parametrize("N, L", [(17, 4), (13, 2)])
def test_a_cascade_with_empty_outer_levels_is_its_level_0(N, L):
    rng = np.random.default_rng(N)
    models = _trained_models()
    rays = _rays(4096, 13)
    rgbs = torch.rand(4096, 3, generator=torch.Generator().manual_seed(14)).cuda()
    w0 = _random_words(rng, N, 1, 0.3)
    words = np.concatenate([w0, np.zeros((L - 1) * cr.words_per_level(N), np.uint32)])
    _eq(_consumers(_grid(words, N, L), models, rays, rgbs), _consumers(_grid(w0, N, 1), models, rays, rgbs))


# ------------------------------------------------------------------------------------------- against the restatement
@pytest.mark.parametrize("seed, N, L", [(0, 9, 3), (1, 17, 4), (2, 12, 2), (3, 33, 8)])
def test_samples_cull_flags_and_the_superset_rule_against_float64(seed, N, L):
    """Per-sample masks of a skip='samples' render of every ray equal the restatement's; the cull flags equal its
    per-level walk except where a rounding could flip a decision; no culled ray has an evaluated sample."""
    rng = np.random.default_rng(seed)
    words = _random_words(rng, N, L, 0.05)
    g = _grid(words, N, L)
    models = _random_models(seed)
    rays = _rays(4096, 20 + seed)
    res = culling.render_samples(models, rays, g, 64, False, 64, False, False, per_sample=True, extras=True)
    r = rays.cpu().numpy()
    zc = ss.z_base(r, 64)
    want_c = cr.evaluated(r, zc, words, N, L, R6)
    want_f = cr.evaluated(r, res["z_vals_fine"].cpu().numpy(), words, N, L, R6)
    got_c = ss.mask_bits(res["mask_coarse"].cpu().numpy(), 64)
    got_f = ss.mask_bits(res["mask_fine"].cpu().numpy(), 128)
    assert np.array_equal(got_c, want_c) and np.array_equal(got_f, want_f)
    flag = nb.cull_rays(rays, g, return_flag=True)[2].cpu().numpy().astype(bool)
    want = cr.ray_live(r, words, N, L, R6)
    occ = cr.unpack(words, N, L)
    margin = np.min([oc.ray_live(r, occ[k], cr.pairs(cr.level_ranges(R6, k)))[1] for k in range(L)], 0)
    bad = (flag != want) & (margin > 1e-9)
    assert not bad.any(), np.nonzero(bad)[0]
    assert not (got_c.any(1) | got_f.any(1))[~flag].any()   # a culled ray has no evaluated sample
    print(f"N = {N}, L = {L}: {flag.sum()} of {len(flag)} rays live, {got_c.sum()} coarse samples evaluated")


def _state(dg):
    torch.cuda.synchronize()
    return {"density": dg._density.cpu().numpy().copy(), "bits": dg.bits.cpu().numpy().view(np.uint32).copy(),
            "key": int(dg.key.item())}


def _assert_state_eq(a, b, what=""):
    assert a["key"] == b["key"] and np.array_equal(a["bits"], b["bits"]), what
    assert np.array_equal(np.asarray(a["density"], np.float32).view(np.uint32),
                          np.asarray(b["density"], np.float32).view(np.uint32)), what


@pytest.mark.parametrize("N, L, seeds", [(17, 2, (0, 99)), (17, 4, (12345, -7)), (129, 2, (2024,)), (129, 4, (5,))])
def test_density_update_equals_the_restatement(N, L, seeds):
    """Points, density and bits of updates bit for bit; a fresh grid skips nothing but the inner cells."""
    model = _trained_models()[1]
    for seed in seeds:
        dg = nb.DensityGrid(N, *BOX, sigma_threshold=2.0, decay=0.85, dilate=1, seed=seed, levels=L)
        _assert_state_eq(_state(dg), cr.initial(N, L, seed), "initial")
        assert dg.density.shape == (L, N - 1, N - 1, N - 1) and dg.state_dict()["levels"] == L
        for k in range(L):
            got = dg.points(level=k).cpu().numpy()
            assert np.array_equal(got.view(np.uint32), cr.points(seed, N, L, R6, k).view(np.uint32)), (seed, k)
        st = cr.initial(N, L, seed)
        for u in range(2 if N > 17 else 3):
            dg.update(model)
            st = cr.update(st, lambda p: nb.query_sigma(model, torch.from_numpy(p).cuda()).cpu().numpy(), N, L, R6,
                           2.0, 0.85, 1)
            _assert_state_eq(_state(dg), st, (seed, u))
        frac = dg.grid.occupied_fraction()
        assert 0.0 < frac < 1.0 and frac * dg.grid.n_cells() == int(np.unpackbits(st["bits"].view(np.uint8)).sum())


def _chunk_case(chunk, N=17, L=3):
    model = _trained_models()[1]
    dg = nb.DensityGrid(N, *BOX, sigma_threshold=2.0, decay=0.8, dilate=1, seed=77, chunk=chunk, levels=L)
    for _ in range(3):
        dg.update(model)
    return _state(dg)


def test_density_results_do_not_depend_on_the_chunk():
    full = _chunk_case(1 << 21)
    for chunk in (1, 97, 3584, 4096, 4097):            # 16^3 = 4096 cells, 3584 non-inner cells per level >= 1
        _assert_state_eq(_chunk_case(chunk), full, chunk)


_CTAS_CASE = """
import sys, numpy as np
sys.path.insert(0, {root!r})
from tests import test_gpu_cascade as t
s = t._chunk_case(1 << 21, N=65, L=4)
np.savez({out!r}, density=s["density"], bits=s["bits"], key=np.int64(s["key"]))
"""


def test_density_results_do_not_depend_on_the_cta_count(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path / "one_cta.npz")
    env = dict(os.environ, NERFB200_MAX_CTAS="1")
    proc = subprocess.run([sys.executable, "-c", _CTAS_CASE.format(root=root, out=out)], env=env, cwd=root,
                          capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stderr[-3000:]
    one = np.load(out)
    _assert_state_eq({"density": one["density"], "bits": one["bits"], "key": int(one["key"])},
                     _chunk_case(1 << 21, N=65, L=4), "one CTA")


def test_occupancy_grid_builds_each_level_from_its_own_lattice():
    """nb.occupancy_cascade(levels=3) equals the restatement applied to nb.sigma_grid over each level's box; the
    state_dict round trip keeps the cascade."""
    model = _trained_models()[1]
    N, L = 17, 3
    g = nb.occupancy_cascade(model, N, *BOX, sigma_threshold=5.0, levels=L, dilate=1)
    sig = np.stack([nb.sigma_grid(model, N, *cr.pairs(cr.level_ranges(R6, k))).cpu().numpy() for k in range(L)])
    assert np.array_equal(g.bits.cpu().numpy().view(np.uint32), cr.pack_sigma(sig, 5.0, 1))
    dense = g.to_dense().cpu().numpy()
    assert dense.shape == (L, N - 1, N - 1, N - 1) and np.array_equal(dense, cr.unpack(cr.pack_sigma(sig, 5.0, 1), N, L))
    h = nb.OccupancyGrid.from_state_dict(g.state_dict())
    assert h.levels == L and torch.equal(h.bits, g.bits)


# ------------------------------------------------------------------------------------------- capture
def _eager_step(models, opt, rays, rgbs, randoms, grid):
    opt.zero_grad(set_to_none=True)
    out = nb.render_rays_loss(models, _emb(), rays, rgbs, 64, False, 1.0, 0.0, 64, 32768, True, randoms=randoms,
                              occupancy=grid)
    out["loss"].backward()
    opt.step()
    return out["loss"].detach().clone(), out["live_samples"]


def _dgrid(net):
    probe = nb.DensityGrid(17, *BOX, seed=123, levels=4)
    thr = float(torch.cat([nb.query_sigma(net, probe.points(level=k)) for k in range(4)]).median())
    return nb.DensityGrid(17, *BOX, sigma_threshold=thr, decay=0.8, dilate=0, seed=123, levels=4)


def test_captured_step_maintains_a_cascade_as_the_eager_loop_does():
    """24 replays with an update every 3 (epochs of 10 batches); in-kernel randoms."""
    B, per_epoch, steps, R = 1024, 10, 24, 3
    n = per_epoch * B + 100
    batches = nb.DeviceRayBatches(torch.from_numpy(bench.blender_rays(n, 60)),
                                  torch.rand(n, 3, generator=torch.Generator().manual_seed(61)), batch_size=B, seed=62)
    models = _random_models()
    opt = nb.FusedAdam([p for m in models for p in m.parameters()], capturable=True, **HYPER)
    dg = _dgrid(models[-1])
    step = nb.CapturedTrainStep(models, batches, opt, 64, False, 1.0, 0.0, 64, True, randoms={"seed": 7000},
                                occupancy=dg, update_every=R)
    _assert_state_eq(_state(dg), cr.initial(17, 4, 123), "the warm-up leaves no trace")
    ref_models = _random_models()
    ref_opt = nb.FusedAdam([p for m in ref_models for p in m.parameters()], capturable=True, **HYPER)
    ref_dg = _dgrid(ref_models[-1])
    recorded = []
    for k in range(steps):
        loss, _ = step.step()
        recorded.append((step.batch_indices.clone(), loss.clone(), step.live_samples.clone()))
    lives = set()
    for k, (ix, loss, live) in enumerate(recorded):
        if k % R == 0:
            ref_dg.update(ref_models[-1])
        ref_loss, ref_live = _eager_step(ref_models, ref_opt, batches.rays[ix], batches.rgbs[ix], {"seed": 7000 + k},
                                         ref_dg.grid)
        assert torch.equal(loss, ref_loss), k
        assert tuple(live.tolist()) == ref_live, k
        lives.add(ref_live)
    assert len(lives) > 1
    _assert_state_eq(_state(dg), _state(ref_dg), "grid")
    for p, q in zip(step.params, [p for m in ref_models for p in m.parameters()]):
        assert torch.equal(p, q)
