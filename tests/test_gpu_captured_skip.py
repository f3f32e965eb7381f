"""The training step with empty samples skipped, captured as one CUDA graph (pytest -m gpu): the device-planned path
of nerfb200_train_samples_forward_dev / _backward_dev and CapturedTrainStep(occupancy=grid).

- Replays equal an eager loop of render_rays_loss(occupancy=) with capturable FusedAdam bit for bit, across
  reshuffles, an lr change and a set_occupancy, and run as many library kernels as the eager step.
- Row counts on both sides of the wgrad planner's clamps and of the chain's probe limit, built from hand-made grids:
  a replay after one with more rows equals an eager step on a fresh workspace; an empty pass gives exact zeros.
- NERFB200_MAX_CTAS=1, memory over 200 replays, non-finite rays (status 103), argument errors.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib
from nerf_pl_b200.train_skip import SkipTrainWorkspace, render_rays_train_skip
from oracle import nerf_oracle as orc

pytestmark = pytest.mark.gpu
HYPER = dict(lr=5e-4, eps=1e-8)
BOX = ((-1.5, 1.5),) * 3


def _emb():
    return [nb.Embedding(3, 10), nb.Embedding(3, 4)]


def _models(seed=0):
    ms = []
    for s in (21 + seed, 22 + seed):
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in orc.make_weights(s).items()})
        ms.append(m.cuda())
    return ms


def _grid(fill, N=17, seed=0, ranges=BOX):
    rng = np.random.default_rng(seed)
    sigma = np.where(rng.random((N, N, N)) < fill, 5.0, 0.0).astype(np.float32)
    return nb.pack_occupancy(torch.from_numpy(sigma).cuda(), *ranges, 1.0, 0)


def _blender(n, seed):
    import bench
    return torch.from_numpy(bench.blender_rays(n, seed))


def _status_ok():
    torch.cuda.synchronize()
    return _lib.load().nerfb200_check_status() == 0


def _eager_step(models, opt, rays, rgbs, cfg, randoms, grid):
    opt.zero_grad(set_to_none=True)
    out = nb.render_rays_loss(models, _emb(), rays, rgbs, cfg["S"], False, 1.0, cfg["noise"], cfg["K"], 32768,
                              cfg["white"], randoms=randoms, occupancy=grid)
    out["loss"].backward()
    opt.step()
    return out["loss"].detach().clone(), out["live_samples"]


# ------------------------------------------------------------------------------------------- captured == eager
@pytest.mark.parametrize("mode", ["torch", "kernel"])
def test_captured_skip_step_equals_eager_loop(mode):
    """50 replays (epochs of 20 batches: two reshuffles), set_occupancy with another grid before replay 25, lr
    changed before replay 30; the eager loop is fed the replays' batches, randoms and grids."""
    B, per_epoch, steps = 1024, 20, 50
    n = per_epoch * B + 100
    cfg = dict(S=64, K=64, noise=1.0 if mode == "torch" else 0.0, white=mode == "kernel")
    batches = nb.DeviceRayBatches(_blender(n, 60), torch.rand(n, 3, generator=torch.Generator().manual_seed(61)),
                                  batch_size=B, seed=62)
    grids = [_grid(0.3, seed=1), _grid(0.5, seed=2)]
    models = _models()
    opt = nb.FusedAdam([p for m in models for p in m.parameters()], capturable=True, **HYPER)
    randoms = {"seed": 7000} if mode == "kernel" else None
    step = nb.CapturedTrainStep(models, batches, opt, 64, False, 1.0, cfg["noise"], 64, cfg["white"],
                                randoms=randoms, occupancy=grids[0])
    ref_models = _models()
    ref_opt = nb.FusedAdam([p for m in ref_models for p in m.parameters()], capturable=True, **HYPER)
    for a, b in zip(models, ref_models):
        for p, q in zip(a.parameters(), b.parameters()):
            assert torch.equal(p, q)
    recorded = []
    for k in range(steps):
        if k == 25:
            step.set_occupancy(grids[1])
        if k == 30:
            opt.param_groups[0]["lr"] = 2e-4
        loss, _ = step.step()
        rnd = {key: v.clone() for key, v in step.randoms.items()}
        if mode == "kernel":
            rnd["seed"] = 7000 + k
        recorded.append((step.batch_indices.clone(), rnd, loss.clone(), step.live_samples.clone()))
    assert step.epoch == 2 and _status_ok()
    lib = _lib.load()
    for k, (ix, rnd, loss, live) in enumerate(recorded):
        if k == 30:
            ref_opt.param_groups[0]["lr"] = 2e-4
        n0 = lib.nerfb200_launch_count()
        ref_loss, ref_live = _eager_step(ref_models, ref_opt, batches.rays[ix], batches.rgbs[ix], cfg, rnd,
                                         grids[k >= 25])
        if k == 0:
            assert lib.nerfb200_launch_count() - n0 == step.launches_per_step
        assert torch.equal(loss, ref_loss), k
        assert tuple(live.tolist()) == ref_live and 0 < ref_live[0] < B * 64, (k, live, ref_live)
    for p, q in zip(step.params, [p for m in ref_models for p in m.parameters()]):
        assert torch.equal(p, q)
        for key in ("exp_avg", "exp_avg_sq", "step"):
            assert torch.equal(opt.state[p][key], ref_opt.state[q][key]), key


# ------------------------------------------------------------------------------------------- row-count sweep
def _box_grid(x0, x1):
    """One occupied cell: x in [x0, x1], y and z in [-1, 1] (space outside the grid counts as empty)."""
    bits = torch.ones(1, dtype=torch.int32, device="cuda")
    return nb.OccupancyGrid(bits, 2, (x0, x1), (-1.0, 1.0), (-1.0, 1.0))


def _counted_rays(per_ray):
    """Rays along +x with perturb = 0: ray j's coarse samples are at x = 100.5 - c_j + i (i = 0..63), so exactly
    c_j of them lie in the cell x in [0, 100] of _box_grid(0, 100)."""
    n = len(per_ray)
    r = torch.zeros(n, 8)
    r[:, 0] = 100.5 - torch.tensor(per_ray, dtype=torch.float32)
    r[:, 3] = 1.0
    r[:, 7] = 63.0
    return r.cuda()


def _split(total, n, S=64):
    c = [S] * (total // S) + ([total % S] if total % S else [])
    return c + [0] * (n - len(c))


class _Captured:
    """render_rays_train_skip(live_samples=) and its backward captured on static rays, grid bits and workspace."""

    def __init__(self, models, rays, S, K, grid, ws):
        self.models, self.S, self.K = models, S, K
        n = rays.shape[0]
        self.rays = rays.clone()
        self.rgbs = torch.rand(n, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
        self.grid = nb.OccupancyGrid(grid.bits.clone(), grid.N, grid.ranges[0:2], grid.ranges[2:4],
                                     grid.ranges[4:6])
        self.ws = ws
        self.live = torch.zeros(2, dtype=torch.int64, device="cuda")
        self.params = [p for m in models[:2 if K else 1] for p in m.parameters()]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            self._body()
        torch.cuda.current_stream().wait_stream(side)
        for p in self.params:
            p.grad = None
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.loss = self._body()
        self.grads = [p.grad for p in self.params]

    def _body(self):
        res = render_rays_train_skip(self.models, self.rays, self.S, False, 0.0, 0.0, self.K, False, None, None, None,
                                     None, self.rgbs, self.grid, workspace=self.ws, live_samples=self.live)
        res["loss"].backward()
        return res["loss"].detach()

    def run(self, rays, grid):
        self.rays.copy_(rays)
        self.grid.bits.copy_(grid.bits)
        self.graph.replay()
        torch.cuda.synchronize()
        return self.loss.clone(), tuple(self.live.tolist()), [g.clone() for g in self.grads]


def _eager_fresh(models, rays, rgbs, S, K, grid):
    SkipTrainWorkspace.clear()                  # a freshly zeroed workspace
    for m in models:
        m.zero_grad(set_to_none=True)
    res = render_rays_train_skip(models, rays, S, False, 0.0, 0.0, K, False, None, None, None, None, rgbs, grid)
    res["loss"].backward()
    live = res["live_samples"]
    grads = []
    for m in models[:2 if K else 1]:
        for p in m.parameters():
            grads.append(p.grad.clone() if p.grad is not None else None)
    return res["loss"].detach().clone(), live, grads


def _check_sweep(cases, S, K):
    """Replays in the order given (each with fewer rows than the one before), one graph per grid geometry, all on
    one workspace; each equals an eager step on a fresh workspace."""
    models = _models()
    n = cases[0][0].shape[0]
    ws = SkipTrainWorkspace(torch.device("cuda:0"), n, S, K)
    graphs = {}
    seen = []
    for rays, grid in cases:
        key = (grid.N, tuple(grid.ranges))
        if key not in graphs:
            graphs[key] = _Captured(models, rays, S, K, grid, ws)
        step = graphs[key]
        loss, live, grads = step.run(rays, grid)
        ref_loss, ref_live, ref_grads = _eager_fresh(models, rays, step.rgbs, S, K, grid)
        assert live == ref_live, (live, ref_live)
        assert torch.equal(loss, ref_loss), live
        nets = 2 if K else 1
        for i, (g, r) in enumerate(zip(grads, ref_grads)):
            if live[i // 24] == 0:
                assert r is None or not torch.any(r), live       # eager: nothing launched, the zeros Python wrote
                assert not torch.any(g), (live, i)               # captured: exact zeros from the device path
            else:
                assert torch.equal(g, r), (live, i)
        assert i == 24 * nets - 1
        seen.append(live)
    assert _status_ok()
    return seen


def test_row_count_sweep_coarse():
    """S = 64, K = 0, 512 rays (carved 32,768 rows = 256 tiles, above the 132-tile probe): the carved maximum, then
    131, 132 and 133 tiles, 129, 128, 127, 1 and 0 rows, each replay after one with more rows."""
    n, S = 512, 64
    grid = _box_grid(0.0, 100.0)
    totals = [n * S, 133 * 128, 132 * 128, 131 * 128, 129, 128, 127, 1, 0]
    seen = _check_sweep([(_counted_rays(_split(t, n)), grid) for t in totals], S, 0)
    assert [s[0] for s in seen] == totals and all(s[1] == 0 for s in seen)


def test_row_count_sweep_empty_passes():
    """S = 64, K = 128: coarse and fine rows from the counted rays, then a coarse pass with no evaluated sample
    whose fine pass has some (the first resampled depth, 0.5, lies in a cell between two coarse samples), then both
    passes empty."""
    n, S, K = 64, 64, 128
    box = _box_grid(0.0, 100.0)
    gap = _box_grid(100.3, 100.7)              # coarse x = 100 + i never in it; the fine sample at z = 0.5 is
    origin = torch.zeros(n, 8, device="cuda")
    origin[:, 0], origin[:, 3], origin[:, 7] = 100.0, 1.0, 63.0
    cases = [(_counted_rays([64] * n), box), (_counted_rays(_split(129, n)), box), (origin, gap),
             (_counted_rays([0] * n), box)]
    seen = _check_sweep(cases, S, K)
    assert seen[0][0] == n * S and seen[1][0] == 129
    assert seen[2][0] == 0 and seen[2][1] > 0, seen
    assert seen[3] == (0, 0), seen


def test_row_count_sweep_piece_clamp():
    """8,192 rays at 64 + 128 samples on a full grid (1.57M fine rows: the wgrad planner lengthens each CTA's pieces
    to stay within its piece table, the max_pieces clamp; 0.52M coarse rows, below it), then on a partial grid of the
    same geometry (fewer rows)."""
    n, S, K = 8192, 64, 128
    rays = _blender(n, 70).cuda()
    wide = ((-8.0, 8.0),) * 3                   # holds every sample of these rays
    cases = [(rays, _grid(1.0, N=17, seed=4, ranges=wide)), (rays, _grid(0.3, N=17, seed=4, ranges=wide))]
    seen = _check_sweep(cases, S, K)
    assert seen[0] == (n * S, n * (S + K)) and seen[1][1] < seen[0][1]


# ------------------------------------------------------------------------------------------- one CTA
_CTAS_CASE = """
import sys, numpy as np, torch
sys.path.insert(0, {root!r})
from tests import test_gpu_captured_skip as t
np.savez({out!r}, **t._ctas_case())
"""


def _ctas_case():
    """Eager and captured results and gradients of a partial-grid step with noise and in-kernel randoms."""
    n, S, K = 900, 64, 128
    out = {}
    for name in ("eager", "captured"):
        models = _models()
        rays = _blender(n, 17).cuda()
        rgbs = torch.rand(n, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
        g = torch.Generator(device="cuda").manual_seed(6)
        nc, nf = torch.randn(n, S, device="cuda", generator=g), torch.randn(n, S + K, device="cuda", generator=g)
        grid = _grid(0.3, seed=5)
        live = None if name == "eager" else torch.zeros(2, dtype=torch.int64, device="cuda")
        ws = None if name == "eager" else SkipTrainWorkspace(torch.device("cuda:0"), n, S, K)

        def body():
            res = render_rays_train_skip(models, rays, S, False, 1.0, 1.0, K, True, None, nc, None, nf, rgbs, grid,
                                         rng_seed=4242, extras=True, workspace=ws, live_samples=live)
            res["loss"].backward()
            return res
        if name == "captured":
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                body()
            torch.cuda.current_stream().wait_stream(side)
            for m in models:
                m.zero_grad(set_to_none=True)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                res = body()
            graph.replay()
            torch.cuda.synchronize()
        else:
            res = body()
        out.update({f"{name}.{k}": np.atleast_1d(v.detach().cpu().numpy()) for k, v in res.items()
                    if torch.is_tensor(v)})
        out.update({f"{name}.grad{i}.{k}": p.grad.cpu().numpy() for i, m in enumerate(models)
                    for k, p in m.named_parameters()})
    return out


def test_results_do_not_depend_on_the_cta_count(tmp_path):
    """NERFB200_MAX_CTAS=1 (read once per process, hence the subprocess): eager and captured results, per-row
    gradients and the 48 gradients are bit for bit those of the full grid."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path / "one_cta.npz")
    env = dict(os.environ, NERFB200_MAX_CTAS="1")
    proc = subprocess.run([sys.executable, "-c", _CTAS_CASE.format(root=root, out=out)], env=env, cwd=root,
                          capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stderr[-3000:]
    one = np.load(out)
    full = _ctas_case()
    assert set(one.files) == set(full)
    for k, v in full.items():
        assert v.dtype == one[k].dtype and np.array_equal(v.view(np.uint8), one[k].view(np.uint8)), k
    for k in full:                              # the captured step is the eager one
        if k.startswith("eager.") and k != "eager.live_samples":
            c = "captured." + k[len("eager."):]
            assert np.array_equal(full[k].view(np.uint8), full[c].view(np.uint8)), k


# ------------------------------------------------------------------------------------------- memory, 103, errors
def _step_on(n, grid=None):
    batches = nb.DeviceRayBatches(_blender(n, 80), torch.rand(n, 3, generator=torch.Generator().manual_seed(81)),
                                  batch_size=n, seed=82)
    models = _models()
    opt = nb.FusedAdam([p for m in models for p in m.parameters()], capturable=True, **HYPER)
    return nb.CapturedTrainStep(models, batches, opt, 64, False, 1.0, 1.0, 64, False, randoms={"seed": 1},
                                occupancy=grid if grid is not None else _grid(0.3))


def test_replays_over_four_grids_allocate_nothing():
    grids = [_grid(f, seed=i) for i, f in enumerate((0.05, 0.3, 0.7, 1.0))]
    step = _step_on(1024, grid=grids[0])
    counts = set()
    for k in range(200):
        step.set_occupancy(grids[k % 4])
        step.step()
        counts.add(tuple(step.live_samples.tolist()))
        if k == 3:                    # the next four replays are one cycle of the grids: their peak is the steady one
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
        if k == 7:
            torch.cuda.synchronize()
            base, peak = torch.cuda.memory_allocated(), torch.cuda.max_memory_allocated()
    torch.cuda.synchronize()
    assert len(counts) >= 4 and _status_ok()
    assert torch.cuda.memory_allocated() == base
    assert torch.cuda.max_memory_allocated() == peak


def test_non_finite_rays_report_status_103():
    """A ray with a non-finite direction (evaluated at every sample) in a replay's batch: its per-sample gradients
    are not finite, which the next library call reports."""
    step = _step_on(1024)
    step.step()
    assert _status_ok()
    step.batches.rays[5, 3:6] = float("nan")       # the one batch of this data set holds ray 5 on every replay
    step.step()
    torch.cuda.synchronize()
    with pytest.raises(_lib.NerfB200Error, match="status 103"):
        nb.render_rays_loss(step.models, _emb(), step.batches.rays[:64], step.batches.rgbs[:64], 64, False, 1.0, 0.0,
                            64, 32768, False, occupancy=_grid(1.0))
    assert _status_ok()


def test_set_occupancy_errors():
    step = _step_on(1024)
    with pytest.raises(ValueError, match="captured N"):
        step.set_occupancy(_grid(0.3, N=9))
    with pytest.raises(ValueError, match="captured N"):
        step.set_occupancy(_grid(0.3, ranges=((-2.0, 2.0),) * 3))
    g = _grid(0.3)
    with pytest.raises(ValueError, match="captured N"):
        step.set_occupancy(nb.OccupancyGrid(g.bits, g.N, g.ranges[0:2], g.ranges[2:4], g.ranges[4:6], dilate=1))
    cpu_grid = object.__new__(nb.OccupancyGrid)
    cpu_grid.bits = torch.zeros(1, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="occupancy grid is on"):
        step.set_occupancy(cpu_grid)
    with pytest.raises(ValueError, match="OccupancyGrid"):
        step.set_occupancy(object())
    step.set_occupancy(_grid(0.7, seed=9))           # same N, ranges and dilate
    step.step()
    assert _status_ok()
    plain = nb.CapturedTrainStep(step.models, step.batches, step.optimizer, 64, False, 1.0, 1.0, 64, False)
    assert plain.live_samples is None
    with pytest.raises(ValueError, match="without occupancy"):
        plain.set_occupancy(_grid(0.3))
