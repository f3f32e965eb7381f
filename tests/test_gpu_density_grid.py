"""The density grid (nb.DensityGrid, csrc/density_kernels.cuh) against its float64 restatement (tests/density_ref.py),
and CapturedTrainStep(occupancy=DensityGrid, update_every=R) against an eager loop (pytest -m gpu).

- The points of an update equal the host replica bit for bit; an update's density equals step 4 applied to
  nb.query_sigma at the replica's points, and its bits equal the float64 rule on the device's own density.
- NaN sigma, chunk sizes, NERFB200_MAX_CTAS=1, capture, allocation, state_dict resume.
- The captured training loop with the grid maintained inside it equals the eager loop bit for bit.
- On the trained test network, renders with the maintained grid stay within a pinned bar of the plain render.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import bench
import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib
from oracle import nerf_oracle as orc
from tests import cases
from tests import density_ref as dr

pytestmark = pytest.mark.gpu
BOX = ((-1.5, 1.5),) * 3
UNEQUAL = ((-1.5, 1.5), (1.4, -1.2), (-0.5, 2.25))           # y reversed
REVERSED = ((1.5, -1.5), (2.0, -1.0), (0.5, -2.5))
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


def _sigma_fn(model):
    return lambda p: nb.query_sigma(model, torch.from_numpy(p).cuda()).cpu().numpy()


def _state(dg):
    torch.cuda.synchronize()
    return {"density": dg._density.cpu().numpy().copy(), "bits": dg.bits.cpu().numpy().view(np.uint32).copy(),
            "key": int(dg.key.item())}


def _assert_state(dg, want, what=""):
    got = _state(dg)
    assert got["key"] == want["key"], what
    assert np.array_equal(got["density"].view(np.uint32), np.asarray(want["density"], np.float32).view(np.uint32)), what
    assert np.array_equal(got["bits"], want["bits"]), what


def _status_ok():
    torch.cuda.synchronize()
    return _lib.load().nerfb200_check_status() == 0


# ------------------------------------------------------------------------------------------- points
@pytest.mark.parametrize("N, ranges, seeds", [(2, BOX, (0, 7, -5)), (17, UNEQUAL, (0, 12345, -(1 << 62) - 3)),
                                              (17, REVERSED, (99,)), (128, UNEQUAL, (2024,))])
def test_points_equal_the_host_replica(N, ranges, seeds):
    for seed in seeds:
        dg = nb.DensityGrid(N, *ranges, seed=seed)
        for key in (seed, seed + 1, seed + 1000):
            dg.key.fill_(key)
            got = dg.points().cpu().numpy()
            want = dr.points(key, N, ranges)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (N, seed, key)
        C = (N - 1) ** 3
        part = dg.points(C // 3, C - C // 3).cpu().numpy()
        assert np.array_equal(part, dr.points(seed + 1000, N, ranges, C // 3, C - C // 3))


# ------------------------------------------------------------------------------------------- one update
def _known_state(dg, seed):
    """Density with values on both sides of the threshold and exactly at it, some cells 0."""
    rng = np.random.default_rng(seed)
    C = (dg.N - 1) ** 3
    d = rng.uniform(0.0, 2.0 * dg.sigma_threshold + 1.0, C).astype(np.float32)
    d[rng.random(C) < 0.3] = 0.0
    d[rng.random(C) < 0.05] = np.float32(dg.sigma_threshold)
    dg._density.copy_(torch.from_numpy(d))
    return d


@pytest.mark.parametrize("dilate", [0, 1, 2])
@pytest.mark.parametrize("which", ["random", "trained"])
def test_update_equals_the_rule(which, dilate):
    model = _random_models()[1] if which == "random" else _trained_models()[1]
    N, thr, decay = 33, 1.0, 0.9
    dg = nb.DensityGrid(N, *UNEQUAL, sigma_threshold=thr, decay=decay, dilate=dilate, seed=31 + dilate)
    d0 = _known_state(dg, dilate)
    key = int(dg.key.item())
    dg.update(model)
    st = _state(dg)
    sigma = _sigma_fn(model)(dr.points(key, N, UNEQUAL))
    want = dr.decay_max(d0, sigma, decay)
    assert np.array_equal(st["density"].view(np.uint32), want.view(np.uint32))
    assert np.array_equal(st["bits"], dr.bits(st["density"], N, thr, dilate)) and st["key"] == key + 1
    occ = dr.occupied(st["density"], N, thr, 0).mean()
    print(f"{which} network, dilate {dilate}: {occ:.3f} of the cells above the threshold before dilation")
    assert 0.0 < occ < 1.0
    assert torch.equal(dg.grid.to_dense().cpu(), torch.from_numpy(dr.occupied(st["density"], N, thr, dilate)))
    assert dg.density.shape == (N - 1,) * 3 and dg.density[3, 5, 7] == dg._density[(7 * (N - 1) + 5) * (N - 1) + 3]


def test_five_updates_follow_the_replica():
    model = _trained_models()[1]
    N = 17
    dg = nb.DensityGrid(N, *BOX, sigma_threshold=5.0, decay=0.7, dilate=1, seed=5)
    ref = dr.initial(N, 5)
    _assert_state(dg, ref, "initial")
    for k in range(5):
        dg.update(model)
        ref = dr.update(ref, _sigma_fn(model), N, BOX, 5.0, 0.7, 1)
        _assert_state(dg, ref, k)
    dg.reset()
    _assert_state(dg, dr.initial(N, 5), "reset")


def test_nan_parameter_decays_the_density():
    model = _random_models()[1]
    N = 9
    dg = nb.DensityGrid(N, *BOX, sigma_threshold=1.0, decay=0.5, dilate=0, seed=1)
    d0 = _known_state(dg, 3)
    with torch.no_grad():
        model.sigma.weight[0, 0] = float("nan")
        model.sigma.bias[0] = float("nan")
    assert torch.isnan(nb.query_sigma(model, dg.points())).all()
    dg.update(model)
    st = _state(dg)
    assert np.array_equal(st["density"], (np.float32(0.5) * d0).astype(np.float32)) and np.isfinite(st["density"]).all()
    assert np.array_equal(st["bits"], dr.bits(st["density"], N, 1.0, 0))
    assert _status_ok()


# ------------------------------------------------------------------------------------------- launch shape
def _chunk_case(chunk, N=9):
    model = _trained_models()[1]
    dg = nb.DensityGrid(N, *UNEQUAL, sigma_threshold=2.0, decay=0.8, dilate=1, seed=77, chunk=chunk)
    for _ in range(3):
        dg.update(model)
    return _state(dg)


def test_results_do_not_depend_on_the_chunk():
    full = _chunk_case(1 << 21)
    for chunk in (1, 97, 511, 512, 513):              # 512 cells
        _assert_state_eq(_chunk_case(chunk), full, chunk)


def _assert_state_eq(a, b, what):
    assert a["key"] == b["key"] and np.array_equal(a["bits"], b["bits"]), what
    assert np.array_equal(a["density"].view(np.uint32), b["density"].view(np.uint32)), what


_CTAS_CASE = """
import sys, numpy as np
sys.path.insert(0, {root!r})
from tests import test_gpu_density_grid as t
s = t._chunk_case(1 << 21, N=65)
np.savez({out!r}, density=s["density"], bits=s["bits"], key=np.int64(s["key"]))
"""


def test_results_do_not_depend_on_the_cta_count(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path / "one_cta.npz")
    env = dict(os.environ, NERFB200_MAX_CTAS="1")
    proc = subprocess.run([sys.executable, "-c", _CTAS_CASE.format(root=root, out=out)], env=env, cwd=root,
                          capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stderr[-3000:]
    one = np.load(out)
    full = _chunk_case(1 << 21, N=65)
    _assert_state_eq({"density": one["density"], "bits": one["bits"], "key": int(one["key"])}, full, "one CTA")


# ------------------------------------------------------------------------------------------- capture, memory, resume
def test_captured_updates_equal_eager_updates_and_allocate_nothing():
    model = _trained_models()[1]
    N = 65
    eager = nb.DensityGrid(N, *BOX, sigma_threshold=1.0, decay=0.9, dilate=1, seed=11, chunk=100000)
    capt = nb.DensityGrid(N, *BOX, sigma_threshold=1.0, decay=0.9, dilate=1, seed=11, chunk=100000)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        capt.update(model)                            # first call: workspace, packed image
    torch.cuda.current_stream().wait_stream(side)
    capt.reset()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        capt.update(model)
    capt.reset()                                      # the capture ran nothing
    for k in range(4):
        graph.replay()
        eager.update(model)
        _assert_state_eq(_state(capt), _state(eager), k)
    torch.cuda.synchronize()
    base, peak = torch.cuda.memory_allocated(), torch.cuda.max_memory_allocated()
    for _ in range(200):
        eager.update(model)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == base and torch.cuda.max_memory_allocated() == peak
    assert int(eager.key.item()) == 11 + 204 and _status_ok()


def test_state_dict_resume_gives_the_same_next_update(tmp_path):
    model = _trained_models()[1]
    a = nb.DensityGrid(33, *UNEQUAL, sigma_threshold=1.5, decay=0.85, dilate=2, seed=3)
    for _ in range(3):
        a.update(model)
    path = tmp_path / "grid.pt"
    torch.save(a.state_dict(), path)
    b = nb.DensityGrid.from_state_dict(torch.load(path), "cuda")
    c = nb.DensityGrid(33, *UNEQUAL, sigma_threshold=1.5, decay=0.85, dilate=2, seed=0).load_state_dict(a.state_dict())
    _assert_state_eq(_state(b), _state(a), "loaded")
    for g in (a, b, c):
        g.update(model)
    _assert_state_eq(_state(b), _state(a), "resumed")
    _assert_state_eq(_state(c), _state(a), "loaded in place")
    with pytest.raises(ValueError, match="load_state_dict"):
        nb.DensityGrid(33, *UNEQUAL, sigma_threshold=1.5, decay=0.8, dilate=2).load_state_dict(a.state_dict())


# ------------------------------------------------------------------------------------------- CapturedTrainStep
def _eager_step(models, opt, rays, rgbs, cfg, randoms, grid):
    opt.zero_grad(set_to_none=True)
    out = nb.render_rays_loss(models, _emb(), rays, rgbs, 64, False, 1.0, cfg["noise"], cfg["K"], 32768,
                              cfg["white"], randoms=randoms, occupancy=grid)
    out["loss"].backward()
    opt.step()
    return out["loss"].detach().clone(), out["live_samples"]


def _dgrid(net=None):
    """With ``net``: the threshold is the median sigma of ``net`` at the first update's points, so that about half
    the cells are occupied and the grid both skips samples and changes under training."""
    thr = 2.0
    if net is not None:
        thr = float(nb.query_sigma(net, nb.DensityGrid(33, *BOX, seed=123).points()).median())
    return nb.DensityGrid(33, *BOX, sigma_threshold=thr, decay=0.8, dilate=0, seed=123)


@pytest.mark.parametrize("mode, K", [("torch", 64), ("kernel", 64), ("kernel", 0)])
def test_captured_step_maintains_the_grid_as_the_eager_loop_does(mode, K):
    """50 replays with an update every R = 3 (epochs of 20 batches: two reshuffles), lr changed before replay 30;
    the eager loop updates its own grid from the last trained model every 3 steps and is fed the replays' batches
    and randoms."""
    B, per_epoch, steps, R = 1024, 20, 50, 3
    n = per_epoch * B + 100
    cfg = dict(K=K, noise=1.0 if mode == "torch" else 0.0, white=mode == "kernel")
    batches = nb.DeviceRayBatches(torch.from_numpy(bench.blender_rays(n, 60)),
                                  torch.rand(n, 3, generator=torch.Generator().manual_seed(61)), batch_size=B, seed=62)
    models = _random_models()
    nets = models[:2 if K else 1]
    opt = nb.FusedAdam([p for m in nets for p in m.parameters()], capturable=True, **HYPER)
    dg = _dgrid(nets[-1])
    randoms = {"seed": 7000} if mode == "kernel" else None
    step = nb.CapturedTrainStep(models, batches, opt, 64, False, 1.0, cfg["noise"], K, cfg["white"], randoms=randoms,
                                occupancy=dg, update_every=R)
    assert step.density_grid is dg and step.launches_per_update > 0
    _assert_state(dg, dr.initial(33, 123), "the warm-up leaves no trace")
    assert step.launches_per_update == 5               # points, sigma, decay and pack (dilate 0), one chunk
    ref_models = _random_models()
    ref_nets = ref_models[:2 if K else 1]
    ref_opt = nb.FusedAdam([p for m in ref_nets for p in m.parameters()], capturable=True, **HYPER)
    ref_dg = _dgrid(ref_nets[-1])
    assert ref_dg.sigma_threshold == dg.sigma_threshold
    recorded = []
    for k in range(steps):
        if k == 30:
            opt.param_groups[0]["lr"] = 2e-4
        loss, _ = step.step()
        rnd = {key: v.clone() for key, v in step.randoms.items()}
        if mode == "kernel":
            rnd["seed"] = 7000 + k
        recorded.append((step.batch_indices.clone(), rnd, loss.clone(), step.live_samples.clone()))
    assert step.epoch == 2 and _status_ok()
    lib = _lib.load()
    lives = set()
    for k, (ix, rnd, loss, live) in enumerate(recorded):
        if k == 30:
            ref_opt.param_groups[0]["lr"] = 2e-4
        if k % R == 0:
            n0 = lib.nerfb200_launch_count()
            ref_dg.update(ref_nets[-1])
            if k == 0:
                assert lib.nerfb200_launch_count() - n0 == step.launches_per_update
        n0 = lib.nerfb200_launch_count()
        ref_loss, ref_live = _eager_step(ref_models, ref_opt, batches.rays[ix], batches.rgbs[ix], cfg, rnd, ref_dg.grid)
        if k == 0:
            assert lib.nerfb200_launch_count() - n0 == step.launches_per_step
        assert torch.equal(loss, ref_loss), k
        assert tuple(live.tolist()) == ref_live and 0 < ref_live[0] < B * 64, (k, live, ref_live)
        lives.add(ref_live)
    print(f"{mode}, K = {K}: evaluated (coarse, fine) samples per step {sorted(lives)[:3]} ... {sorted(lives)[-1]}")
    assert len(lives) > 1                              # the grid changes under the loop
    _assert_state_eq(_state(dg), _state(ref_dg), "grid")
    for p, q in zip(step.params, [p for m in ref_nets for p in m.parameters()]):
        assert torch.equal(p, q)
        for key in ("exp_avg", "exp_avg_sq", "step"):
            assert torch.equal(opt.state[p][key], ref_opt.state[q][key]), key


def test_captured_step_argument_errors():
    n = 2048
    batches = nb.DeviceRayBatches(torch.from_numpy(bench.blender_rays(n, 80)), torch.rand(n, 3), batch_size=1024,
                                  seed=82)
    models = _random_models()
    opt = nb.FusedAdam([p for m in models for p in m.parameters()], capturable=True, **HYPER)
    grid = nb.occupancy_grid(models[1], 17, *BOX, 1.0, 1)
    for occ in (None, grid):
        with pytest.raises(ValueError, match="update_every needs occupancy=DensityGrid"):
            nb.CapturedTrainStep(models, batches, opt, occupancy=occ, update_every=4)
    for bad in (None, 0, -1, 2.5):
        with pytest.raises(ValueError, match="needs update_every"):
            nb.CapturedTrainStep(models, batches, opt, occupancy=_dgrid(), update_every=bad)
    step = nb.CapturedTrainStep(models, batches, opt, occupancy=_dgrid(), update_every=2, randoms="kernel")
    with pytest.raises(ValueError, match="maintains its DensityGrid"):
        step.set_occupancy(grid)
    step.step()
    assert _status_ok()
    plain = nb.CapturedTrainStep(models, batches, opt)
    assert plain.update_graph is None and plain.launches_per_update == 0 and plain.density_grid is None


# ------------------------------------------------------------------------------------------- usefulness
# Mean over pixels of max-channel |rgb_fine(skip="samples" with the maintained grid) - rgb_fine(plain)| on the three
# test views (200 x 200, 64 + 128 samples) after 8 updates of a 128-point grid over the tests' box (sigma > 1,
# decay 0.95, dilate 1) from the trained fine network.  Measured on an NVIDIA H100 80GB HBM3: 4.1e-4, 2.5e-4 and
# 2.8e-4 with 23 % of the cells occupied (DESIGN.md §10d); pinned at about three times the largest.
MAINTAINED_MEAN_RGB = 1.2e-3


@pytest.mark.parametrize("seed", [61, 62, 63])
def test_maintained_grid_renders_the_trained_scene(seed):
    models = _trained_models()
    dg = nb.DensityGrid(128, *BOX, sigma_threshold=1.0, decay=0.95, dilate=1, seed=4)
    for _ in range(8):
        dg.update(models[1])
    rays = torch.from_numpy(bench.blender_rays(0, seed, W=200, H=200, pixels="all")).cuda()
    with torch.no_grad():
        plain = nb.render_rays(models, _emb(), rays, 64, False, 0, 0, 128, 32768, True, test_time=True,
                               match_reference_rng=False)
    res = nb.render_rays_culled(models, _emb(), rays, dg.grid, 64, False, 128, True, test_time=True, skip="samples")
    err = (res["rgb_fine"] - plain["rgb_fine"]).abs().amax(1)
    frac = dg.grid.occupied_fraction()
    n = rays.shape[0]
    print(f"view {seed}: {frac:.4f} of the cells occupied, {res['live']} of {n} rays live, evaluated fine samples "
          f"{res['live_samples'][1] / (n * 192):.3f}; max-channel |rgb_fine - plain| mean {float(err.mean()):.3e} "
          f"max {float(err.max()):.3e}")
    assert 0.005 < frac < 0.5 and res["live"] < n
    assert float(err.mean()) < MAINTAINED_MEAN_RGB
