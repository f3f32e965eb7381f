"""Training from the device as one CUDA graph (pytest -m gpu).

A. FusedAdam(capturable=True) (nerfb200_adam_step_dev): m and v bit-identical to FusedAdam, p within the adam_ref
   bars; lr schedules; parameters without a gradient; checkpoints with torch.optim.Adam(capturable=True) and with
   non-capturable FusedAdam.
B. In-kernel random numbers keyed from device memory: the same renders and gradients as the host seed, and graph
   replays that advance the word consume seeds s, s + 1, ... (checked against tests/philox.py).
C. CapturedTrainStep: 50 replays crossing epoch boundaries equal an eager loop fed the same batches and random
   inputs, bit for bit, with an lr change and eager renders / training steps of the same shape between replays.
"""
import io

import numpy as np
import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib
from oracle import nerf_oracle as orc
from tests import adam_ref, cases, philox
from tests.test_gpu_train_loop import AdamCheck, _grads_for, _params

pytestmark = pytest.mark.gpu

HYPER = dict(lr=5e-4, eps=1e-8)
SHAPES = [(0,), (1,), (255,), (1025,), (300_007,), (256, 63), (3,)]


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def emb():
    return [nb.Embedding(3, 10), nb.Embedding(3, 4)]


def _models(dev, ws=None):
    out = []
    for w in (ws or cases.weights()):
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in w.items()})
        out.append(m.to(dev))
    return out


def _status_ok():
    torch.cuda.synchronize()
    return _lib.load().nerfb200_check_status() == 0


# ------------------------------------------------------------------------------------------- A. capturable Adam
@pytest.mark.parametrize("wd", [0.0, 1e-3])
def test_capturable_adam_vs_fused_adam_and_float64(wd, dev):
    """300 steps.  Before every step the non-capturable optimiser is given the capturable one's parameters, so each
    step compares one update: m and v bit for bit, p against adam_ref (and the count of p elements that differ from
    the host-formed bias corrections' update is reported).  One launch per step for all tensors."""
    ps = _params(SHAPES, 30, dev)
    qs = [p.clone() for p in ps]
    oc = nb.FusedAdam(ps, weight_decay=wd, capturable=True, **HYPER)
    oh = nb.FusedAdam(qs, weight_decay=wd, **HYPER)
    chk = AdamCheck()
    lib = _lib.load()
    differ, total = 0, 0
    for t in range(1, 301):
        for p, q, g in zip(ps, qs, _grads_for(ps, t, 30, dev)):
            p.grad, q.grad = g, g.clone()
            q.data.copy_(p.data)
        n0 = lib.nerfb200_launch_count()
        chk.step(oc, "capturable")
        assert lib.nerfb200_launch_count() - n0 == 1
        oh.step()
        for p, q in zip(ps, qs):
            for k in ("exp_avg", "exp_avg_sq"):
                assert torch.equal(oc.state[p][k], oh.state[q][k]), (t, k)
            differ += int((p != q).sum())
            total += p.numel()
    assert all(oc.state[p]["step"].is_cuda and int(oc.state[p]["step"]) == 300 for p in ps)
    print(f"\n[capturable Adam wd={wd}] p elements differing from the host-formed update: {differ} of {total}")
    chk.report(f"capturable wd={wd}")
    assert not chk.bad(), chk.bad()


def test_capturable_adam_lr_schedule_and_missing_gradients(dev):
    """A cosine schedule changes group['lr'] between steps; some parameters have no gradient in some steps and keep
    their own step count; every step against adam_ref (per-tensor bias corrections in one launch)."""
    ps = _params([(1000,), (5000,), (3,), (256, 63)], 31, dev)
    opt = nb.FusedAdam(ps, weight_decay=1e-4, capturable=True, **HYPER)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=20, eta_min=1e-6)
    chk = AdamCheck()
    lrs = set()
    for t in range(20):
        gs = _grads_for(ps, t, 31, dev)
        for i, (p, g) in enumerate(zip(ps, gs)):
            p.grad = None if (i % 2 and t in (3, 4, 9)) else g
        lrs.add(opt.param_groups[0]["lr"])
        chk.step(opt, "schedule")
        sched.step()
    assert len(lrs) > 10
    assert [int(opt.state[p]["step"]) for p in ps] == [20, 17, 20, 17]
    chk.report("capturable, schedule + missing gradients")
    assert not chk.bad(), chk.bad()


def _roundtrip(obj):
    buf = io.BytesIO()
    torch.save(obj, buf)
    buf.seek(0)
    return torch.load(buf, weights_only=False)


def _run(opt, ps, t0, t1, seed, dev):
    for t in range(t0, t1):
        for p, g in zip(ps, _grads_for(ps, t, seed, dev)):
            p.grad = g
        opt.step()


def test_capturable_checkpoints(dev):
    """Capturable FusedAdam -> torch.optim.Adam(capturable=True) -> capturable FusedAdam, and capturable <->
    non-capturable FusedAdam: moments carried bit for bit, steps on the device (capturable) or the host, and the
    continued runs of both FusedAdam forms agree: m and v bit for bit, p within a few ulps."""
    seed, k = 32, 6
    shapes = [(256, 63), (256,), (1025,), (3,)]
    a = _params(shapes, seed, dev)
    oa = nb.FusedAdam(a, capturable=True, **HYPER)
    _run(oa, a, 0, k, seed, dev)
    b = [p.clone() for p in a]
    ot = torch.optim.Adam(b, capturable=True, **HYPER)
    ot.load_state_dict(_roundtrip(oa.state_dict()))
    for p, q in zip(a, b):
        for key in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(oa.state[p][key], ot.state[q][key])
        assert ot.state[q]["step"].is_cuda and int(ot.state[q]["step"]) == k
    _run(ot, b, k, k + 2, seed, dev)
    c = [p.clone() for p in b]
    oc = nb.FusedAdam(c, capturable=True, **HYPER)
    oc.load_state_dict(_roundtrip(ot.state_dict()))
    assert oc.param_groups[0]["capturable"] is True
    for p, q in zip(b, c):
        assert oc.state[q]["step"].is_cuda and int(oc.state[q]["step"]) == k + 2
        assert torch.equal(ot.state[p]["exp_avg_sq"], oc.state[q]["exp_avg_sq"])
    _run(oc, c, k + 2, k + 4, seed, dev)
    # capturable -> non-capturable and back, continued side by side
    d = [p.clone() for p in c]
    od = nb.FusedAdam(d, **HYPER)
    od.load_state_dict(_roundtrip(oc.state_dict()))
    assert all(not od.state[p]["step"].is_cuda for p in d)
    e = [p.clone() for p in d]
    oe = nb.FusedAdam(e, capturable=True, **HYPER)
    oe.load_state_dict(_roundtrip(od.state_dict()))
    assert all(oe.state[p]["step"].is_cuda for p in e)
    _run(od, d, k + 4, k + 9, seed, dev)
    _run(oe, e, k + 4, k + 9, seed, dev)
    for p, q in zip(d, e):
        assert int(od.state[p]["step"]) == int(oe.state[q]["step"]) == k + 9
        for key in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(od.state[p][key], oe.state[q][key])
        ulps = ((p - q).abs() / adam_ref.ulp32(p).to(torch.float32)).max()
        assert float(ulps) <= 8, float(ulps)


def test_capture_needs_capturable_adam(dev):
    models = _models(dev)
    rays, rgbs = torch.from_numpy(orc.make_rays(2048, 1)), torch.rand(2048, 3)
    batches = nb.DeviceRayBatches(rays, rgbs, seed=1)
    opt = nb.FusedAdam([p for m in models for p in m.parameters()], **HYPER)
    with pytest.raises(ValueError, match="capturable"):
        nb.CapturedTrainStep(models, batches, opt)


# ------------------------------------------------------------------------------------------- B. device-keyed RNG
SEED = 0xDEADBEEF12345678            # above 2^63: the int64 word holds the same 64 bits


def _seed_word(s, dev):
    return torch.tensor(s - (1 << 64) if s >= 1 << 63 else s, dtype=torch.int64, device=dev)


@pytest.mark.parametrize("noise", [0.0, 1.0])
def test_device_seed_equals_host_seed(noise, dev, emb):
    """render_rays_loss with {'seed': word on the device} == {'seed': s}: outputs, loss and all 48 gradients bit for
    bit (the Gaussian noise, when on, is the same tensor in both)."""
    n = 1024
    rays = torch.from_numpy(orc.make_rays(n, 40)).to(dev)
    tgt = torch.rand(n, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(41))
    g = torch.Generator(device=dev).manual_seed(42)
    rnd = {"noise_coarse": torch.randn(n, 64, device=dev, generator=g),
           "noise_fine": torch.randn(n, 128, device=dev, generator=g)} if noise else {}
    res = []
    for seed in (SEED, _seed_word(SEED, dev)):
        models = _models(dev)
        out = nb.render_rays_loss(models, emb, rays, tgt, 64, False, 1.0, noise, 64, 32768, True,
                                  randoms=dict(rnd, seed=seed))
        out["loss"].backward()
        res.append(({k: v.detach() for k, v in out.items()}, [p.grad for m in models for p in m.parameters()]))
    assert _status_ok()
    for k in res[0][0]:
        assert torch.equal(res[0][0][k], res[1][0][k]), k
    for x, y in zip(res[0][1], res[1][1]):
        assert torch.equal(x, y)


def test_graph_replays_advance_the_seed(dev, emb):
    """A captured inference render keyed by a device word that the graph increments: replay k renders exactly as
    the tensor inputs tests/philox.py generates for seed s + k."""
    n, S, K = 512, 64, 64
    rays = torch.from_numpy(orc.make_rays(n, 43)).to(dev)
    models = _models(dev)
    for m in models:
        m.requires_grad_(False)
    word = _seed_word(SEED, dev)
    args = (S, False, 1.0, 0.0, K, 32768, True)
    with torch.no_grad():
        nb.render_rays(models, emb, rays, *args, randoms={"seed": word})        # first-call set-up
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = nb.render_rays(models, emb, rays, *args, randoms={"seed": word})
            word.add_(1)
        for k in range(5):
            graph.replay()
            got = {key: v.clone() for key, v in out.items()}
            s = (SEED + k) & 0xFFFFFFFFFFFFFFFF
            rnd = {key: torch.from_numpy(v).to(dev) for key, v in philox.randoms(s, n, S, K).items()}
            ref = nb.render_rays(models, emb, rays, *args, randoms=rnd)
            for key in ref:
                assert torch.equal(got[key], ref[key]), (k, key)
    assert int(word) == int(_seed_word((SEED + 5) & 0xFFFFFFFFFFFFFFFF, dev))
    assert _status_ok()


def test_host_kernel_seed_is_refused_under_capture(dev, emb):
    models = _models(dev)
    rays = torch.from_numpy(orc.make_rays(64, 44)).to(dev)
    tgt = torch.rand(64, 3, device=dev)
    nb.render_rays_loss(models, emb, rays, tgt, randoms="kernel")
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(ValueError, match="replay one seed"):
        with torch.cuda.graph(graph):
            nb.render_rays_loss(models, emb, rays, tgt, randoms="kernel")


# ------------------------------------------------------------------------------------------- C. captured step
def _eager_step(models, emb, opt, rays, rgbs, cfg, randoms):
    opt.zero_grad(set_to_none=True)
    out = nb.render_rays_loss(models, emb, rays, rgbs, cfg["S"], False, 1.0, cfg["noise"], cfg["K"], 32768,
                              cfg["white"], randoms=randoms)
    out["loss"].backward()
    opt.step()
    return out["loss"].detach().clone()


@pytest.mark.parametrize("mode", ["torch", "kernel"])
def test_captured_step_equals_eager_loop(mode, dev, emb):
    """50 replays (epochs of 20 full batches: two reshuffles) against an eager loop with capturable FusedAdam fed
    the replays' batches and random inputs: every loss, the parameters and the Adam state bit for bit.  The lr is
    changed after replay 30 (for both); after replay 10 an eager inference render and an eager training step of the
    same shape on other models run in between.  The replays' batches form per-epoch permutations, and a replay runs
    as many library kernels as an eager step."""
    B, per_epoch, steps = 1024, 20, 50
    n = per_epoch * B + 300
    noise = 1.0 if mode == "torch" else 0.0
    cfg = dict(S=64, K=64, noise=noise, white=mode == "kernel")
    rays = torch.from_numpy(orc.make_rays(n, 50))
    rgbs = torch.rand(n, 3, generator=torch.Generator().manual_seed(51))
    batches = nb.DeviceRayBatches(rays, rgbs, batch_size=B, seed=52)
    models = _models(dev)
    opt = nb.FusedAdam([p for m in models for p in m.parameters()], capturable=True, **HYPER)
    randoms = {"seed": 9000} if mode == "kernel" else None
    step = nb.CapturedTrainStep(models, batches, opt, 64, False, 1.0, noise, 64, cfg["white"], randoms=randoms)
    assert step.per_epoch == per_epoch
    ref_models = _models(dev)
    ref_opt = nb.FusedAdam([p for m in ref_models for p in m.parameters()], capturable=True, **HYPER)
    for a, b in zip(models, ref_models):                   # construction left the models as they were
        for p, q in zip(a.parameters(), b.parameters()):
            assert torch.equal(p, q)
    others = _models(dev, cases.trained_weights() if cases.have_trained() else None)
    other_opt = nb.FusedAdam([p for m in others for p in m.parameters()], **HYPER)
    lib = _lib.load()
    recorded = []
    for k in range(steps):
        if k == 30:
            opt.param_groups[0]["lr"] = 2e-4
        loss, _ = step.step()
        rnd = {key: v.clone() for key, v in step.randoms.items()}
        if mode == "kernel":
            rnd["seed"] = 9000 + k
        recorded.append((step.batch_indices.clone(), rnd, loss.clone()))
        if k == 10:
            with torch.no_grad():
                nb.render_rays(others, emb, batches.rays[:B], 64, False, 1.0, 0.0, 64, 32768, True,
                               randoms={"seed": 1})
            _eager_step(others, emb, other_opt, batches.rays[B:2 * B], batches.rgbs[B:2 * B], cfg, {"seed": 2})
    assert step.epoch == 2 and _status_ok()
    idx = torch.stack([r[0] for r in recorded]).cpu()
    for e in range(3):
        ep = idx[e * per_epoch:(e + 1) * per_epoch].reshape(-1)
        assert ep.unique().numel() == ep.numel()
    assert not torch.equal(idx[:per_epoch], idx[per_epoch:2 * per_epoch])
    for k, (ix, rnd, loss) in enumerate(recorded):
        if k == 30:
            ref_opt.param_groups[0]["lr"] = 2e-4
        n0 = lib.nerfb200_launch_count()
        ref_loss = _eager_step(ref_models, emb, ref_opt, batches.rays[ix], batches.rgbs[ix], cfg, rnd)
        if k == 0:
            assert lib.nerfb200_launch_count() - n0 == step.launches_per_step
        assert torch.equal(loss, ref_loss), k
    for p, q in zip(step.params, [p for m in ref_models for p in m.parameters()]):
        assert torch.equal(p, q)
        for key in ("exp_avg", "exp_avg_sq", "step"):
            assert torch.equal(opt.state[p][key], ref_opt.state[q][key]), key
    assert int(opt.state[step.params[0]]["step"]) == steps
    assert _status_ok()


def test_replay_between_an_eager_forward_and_its_backward(dev, emb):
    """An eager training forward of the graph's shape, then a replay, then the eager backward: the eager gradients
    equal those of the same forward + backward with no replay in between, bit for bit.  (A replay overwrites its
    training workspace; the graph's is its own, so the eager call's pending workspace is untouched.)"""
    B = 1024
    rays = torch.from_numpy(orc.make_rays(4 * B, 60))
    rgbs = torch.rand(4 * B, 3, generator=torch.Generator().manual_seed(61))
    batches = nb.DeviceRayBatches(rays, rgbs, batch_size=B, seed=62)
    models = _models(dev)
    opt = nb.FusedAdam([p for m in models for p in m.parameters()], capturable=True, **HYPER)
    step = nb.CapturedTrainStep(models, batches, opt, 64, False, 1.0, 0.0, 64, True, randoms={"seed": 5})
    r, c = batches.rays[2 * B:3 * B], batches.rgbs[2 * B:3 * B]
    grads = []
    for replay in (True, False):
        others = _models(dev, cases.trained_weights() if cases.have_trained() else None)
        out = nb.render_rays_loss(others, emb, r, c, 64, False, 1.0, 0.0, 64, 32768, True, randoms={"seed": 6})
        if replay:
            step.step()
            step.step()
        out["loss"].backward()
        grads.append([p.grad.clone() for m in others for p in m.parameters()])
    assert _status_ok()
    for x, y in zip(*grads):
        assert torch.equal(x, y)


def test_parameters_outside_the_models_are_left_alone(dev, emb):
    """N_importance = 0 with an optimizer that also holds the fine model, whose parameters carry stale gradients:
    neither the warm-up nor the replays update them, and the coarse model trains."""
    B = 1024
    rays = torch.from_numpy(orc.make_rays(3 * B, 63))
    rgbs = torch.rand(3 * B, 3, generator=torch.Generator().manual_seed(64))
    batches = nb.DeviceRayBatches(rays, rgbs, batch_size=B, seed=65)
    models = _models(dev)
    opt = nb.FusedAdam([p for m in models for p in m.parameters()], capturable=True, **HYPER)
    for p in models[1].parameters():
        p.grad = torch.ones_like(p)
    fine0 = [p.detach().clone() for p in models[1].parameters()]
    coarse0 = [p.detach().clone() for p in models[0].parameters()]
    step = nb.CapturedTrainStep(models, batches, opt, 64, False, 1.0, 0.0, 0, True)
    for _ in range(3):
        step.step()
    assert _status_ok()
    for p, q in zip(models[1].parameters(), fine0):
        assert torch.equal(p, q) and len(opt.state.get(p, {})) == 0
    assert not all(torch.equal(p, q) for p, q in zip(models[0].parameters(), coarse0))
