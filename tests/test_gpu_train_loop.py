"""What carries over from one training step to the next (pytest -m gpu).

A. FusedAdam against float64 Adam (tests/adam_ref.py), one step at a time: the reference is fed the kernel's own
   fp32 p, m, v of the previous step, so every step is held to the kernel's own rounding.
B. FusedAdam's state: checkpoints (also from and to torch.optim.Adam), rollback into the same instance, steps in
   which some parameters have no gradient.  Bit for bit against uninterrupted runs.
C. The pooled training workspaces keep nothing from one step to the next: a probe step on a workspace that has
   served a sequence of different steps equals, bit for bit, the same step on a fresh workspace.
D. A render's workspace is released when its graph is freed without a backward.
E. A short training run (fused render + loss, fused backward, FusedAdam) checked at every step.

Measured values (H100 80GB HBM3) stand next to each bar.
"""
import copy
import io
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib
from nerf_pl_b200.training import NerfTrainWorkspace, TrainWorkspace
from oracle import nerf_oracle as orc
from oracle import nerf_oracle_grad as og
from tests import adam_ref, cases
from tests.test_gpu_train_stages import stage_report

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def emb():
    return [nb.Embedding(3, 10), nb.Embedding(3, 4)]


def _models(ws, dev):
    out = []
    for w in ws:
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in w.items()})
        out.append(m.to(dev))
    return out


def _status_ok():
    torch.cuda.synchronize()
    return _lib.load().nerfb200_check_status() == 0


# ------------------------------------------------------------------------------------------- A. FusedAdam vs float64
def _flat(ts, like=None):
    if not ts:
        return torch.zeros(0, dtype=torch.float32, device=like)
    return torch.cat([t.detach().reshape(-1) for t in ts])


def _state(opt, ps, key):
    return _flat([opt.state[p][key] if len(opt.state[p]) else torch.zeros_like(p) for p in ps])


def _step_of(opt, p):
    st = opt.state[p]
    return int(st["step"]) if len(st) else 0


class AdamCheck:
    """``step(opt)`` runs ``opt.step()`` and compares every stepped parameter with adam_ref, fed the fp32 p, m, v
    the optimiser held before the step; keeps the worst error per quantity."""

    def __init__(self):
        self.worst = {"m": 0.0, "v": 0.0, "p": 0.0}
        self.where = {}

    def step(self, opt, tag=""):
        snaps = []
        for group in opt.param_groups:
            by_t = {}
            for p in group["params"]:
                if p.grad is not None:
                    by_t.setdefault(_step_of(opt, p) + 1, []).append(p)
            hyper = (group["lr"], *group["betas"], group["eps"], group["weight_decay"])
            for t, ps in by_t.items():
                snaps.append((t, hyper, ps, (_flat(ps), _flat([p.grad for p in ps]), _state(opt, ps, "exp_avg"),
                                             _state(opt, ps, "exp_avg_sq"))))
        opt.step()
        for t, hyper, ps, before in snaps:
            after = (_flat(ps), _state(opt, ps, "exp_avg"), _state(opt, ps, "exp_avg_sq"))
            e = adam_ref.errors(before, after, t, *hyper)
            for k, v in e.items():
                if v > self.worst[k]:
                    self.worst[k] = v
                    self.where[k] = f"{tag} step {t}"
        return self

    def report(self, name):
        print(f"\n[{name}] worst Adam error (ulps): " +
              " ".join(f"{k} {v:.3g} ({self.where.get(k, '-')})" for k, v in self.worst.items()))

    def bad(self):
        return {k: v for k, v in self.worst.items() if not v <= adam_ref.BARS[k]}


def _grads_for(ps, t, seed, dev):
    """Seeded gradients of step t: N(0, 1) times a per-tensor scale from 1e-1 to 1e-6 (so that eps matters for some)."""
    g = torch.Generator(device=dev).manual_seed(seed * 100003 + t)
    return [torch.randn(p.shape, device=dev, generator=g) * 10.0 ** -(1 + i % 6) for i, p in enumerate(ps)]


def _set_grads(ps, t, seed, dev):
    for p, g in zip(ps, _grads_for(ps, t, seed, dev)):
        p.grad = g


def _params(shapes, seed, dev, scale=0.05):
    g = torch.Generator(device=dev).manual_seed(seed)
    return [torch.randn(s, device=dev, generator=g) * scale for s in shapes]


SHAPES = [(0,), (1,), (255,), (1023,), (1024,), (1025,), (300_007,), (256, 63), (3,)]


@pytest.mark.parametrize("wd", [0.0, 1e-3])
def test_adam_shapes_vs_float64(wd, dev):
    """numel 0 / 1 / 255 / 1023 / 1024 / 1025 / ~300k: steps 1-20 compared every step, then 300 steps of the small
    tensors, then the step count jumped to 1e5 (bias corrections -> 1)."""
    ps = _params(SHAPES, 1, dev)
    opt = nb.FusedAdam(ps, lr=5e-4, eps=1e-8, weight_decay=wd)
    chk = AdamCheck()
    for t in range(1, 21):
        _set_grads(ps, t, 1, dev)
        chk.step(opt, "dense")
    small = [p for p in ps if p.numel() <= 1025]
    opt2 = nb.FusedAdam(small, lr=1e-3, eps=1e-8, weight_decay=wd)
    for t in range(1, 301):
        _set_grads(small, t, 2, dev)
        chk.step(opt2, "long")
    for p in ps:
        opt.state[p]["step"] = torch.tensor(1e5)
    for t in range(3):
        _set_grads(ps, 100 + t, 1, dev)
        chk.step(opt, "t=1e5")
    assert all(int(opt.state[p]["step"]) == 100003 for p in ps)
    chk.report(f"shapes wd={wd}")
    assert not chk.bad(), chk.bad()


def test_adam_zero_parameters_expose_the_update(dev):
    """Parameters at exactly 0 with weight_decay 0: p' = -update, so p is held to the update's own rounding.  p is
    set back to 0 before every step (the reference takes the kernel's state, so this is a valid state).  An fp32
    bias correction 1 - b2^t is ~50 ulps of the update wrong at t = 2, 3."""
    ps = [torch.zeros(s, device=dev) for s in [(4099,), (256, 256), (1,)]]
    opt = nb.FusedAdam(ps, lr=5e-4, eps=1e-8)
    chk = AdamCheck()
    for t in range(1, 21):
        _set_grads(ps, t, 3, dev)
        for p in ps:
            p.zero_()
        chk.step(opt, "zero")
    chk.report("zero parameters")
    assert not chk.bad(), f"{chk.bad()} at {chk.where}"


def test_adam_many_tensors_and_groups_vs_float64(dev):
    """One group of 70 tensors (two launches), the 48 tensors of two NeRFs in a second group with other lr / betas /
    eps / weight decay, and non-contiguous gradients for some tensors."""
    many = _params([(1 + 97 * i,) for i in range(70)], 4, dev)
    torch.manual_seed(4)
    nets = [nb.NeRF().to(dev), nb.NeRF().to(dev)]
    nerf = [p.data for m in nets for p in m.parameters()]
    opt = nb.FusedAdam([{"params": many},
                        {"params": nerf, "lr": 2e-3, "betas": (0.8, 0.99), "eps": 1e-6, "weight_decay": 1e-2}],
                       lr=5e-4, eps=1e-8)
    chk = AdamCheck()
    for t in range(1, 21):
        _set_grads(many + nerf, t, 4, dev)
        for p in nerf:
            if p.dim() == 2 and min(p.shape) > 1:    # the same values through a transposed (non-contiguous) view
                p.grad = p.grad.t().contiguous().t()
                assert not p.grad.is_contiguous()
        chk.step(opt, "groups")
    chk.report("70 tensors + 48 NeRF tensors, two groups")
    assert not chk.bad(), chk.bad()


def test_adam_learning_rate_schedules_vs_float64(dev):
    """group['lr'] changed between steps by torch's schedulers (the reference's steplr / cosine, and a linear
    warm-up as GradualWarmupScheduler does it)."""
    chk = AdamCheck()
    sched = {
        "multistep": lambda o: torch.optim.lr_scheduler.MultiStepLR(o, milestones=[5, 10], gamma=0.5),
        "cosine": lambda o: torch.optim.lr_scheduler.CosineAnnealingLR(o, T_max=20, eta_min=1e-6),
        "warmup": lambda o: torch.optim.lr_scheduler.LambdaLR(o, lambda e: min(1.0, (e + 1) / 8)),
    }
    for i, (name, make) in enumerate(sched.items()):
        ps = _params([(1000,), (5000,), (3,)], 10 + i, dev)
        opt = nb.FusedAdam(ps, lr=5e-4, eps=1e-8, weight_decay=1e-4)
        s = make(opt)
        lrs = set()
        for t in range(1, 21):
            _set_grads(ps, t, 10 + i, dev)
            lrs.add(opt.param_groups[0]["lr"])
            chk.step(opt, name)
            s.step()
        assert len(lrs) > 2, name
    chk.report("lr schedules")
    assert not chk.bad(), chk.bad()


# ------------------------------------------------------------------------------------------- B. FusedAdam state
B_SHAPES = [(256, 63), (256,), (3, 128), (3,), (1025,), (1,), (70_000,)]
B_HYPER = dict(lr=5e-4, eps=1e-8, weight_decay=1e-3)


def _run(opt, ps, t0, t1, seed, dev):
    for t in range(t0, t1):
        _set_grads(ps, t, seed, dev)
        opt.step()


def _roundtrip(obj):
    buf = io.BytesIO()
    torch.save(obj, buf)
    buf.seek(0)
    return torch.load(buf, weights_only=False)


def _assert_same(a, b, what):
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), f"{what}: tensor {i} differs, max {float((x - y).abs().max()):.3g}"


def _moments(opt, ps):
    return [opt.state[p][k] for p in ps for k in ("exp_avg", "exp_avg_sq")]


def test_checkpoint_resume_is_bit_exact(dev):
    """state_dict after k steps, loaded (through torch.save / torch.load) into a fresh FusedAdam over a copy of the
    parameters, continued j steps == k + j uninterrupted steps, bit for bit."""
    k, j, seed = 7, 6, 20
    base = _params(B_SHAPES, seed, dev)
    full = [p.clone() for p in base]
    of = nb.FusedAdam(full, **B_HYPER)
    _run(of, full, 0, k + j, seed, dev)
    a = [p.clone() for p in base]
    oa = nb.FusedAdam(a, **B_HYPER)
    _run(oa, a, 0, k, seed, dev)
    ck = _roundtrip(oa.state_dict())
    b = [p.clone() for p in a]
    ob = nb.FusedAdam(b, **B_HYPER)
    ob.load_state_dict(ck)
    _run(ob, b, k, k + j, seed, dev)
    _assert_same(b, full, "parameters")
    _assert_same(_moments(ob, b), _moments(of, full), "moments")
    assert all(torch.is_tensor(ob.state[p]["step"]) and int(ob.state[p]["step"]) == k + j for p in b)


def test_checkpoint_rollback_into_the_same_instance(dev):
    """The step-k checkpoint loaded into the instance that has gone on to step k + j, then continued: the loaded
    moments and step count are used (not those of the tensors the instance held before the load), bit for bit.
    Once from an in-memory deep copy, once through torch.save / torch.load (new state tensors)."""
    k, j, seed = 5, 4, 21
    base = _params(B_SHAPES, seed, dev)
    full = [p.clone() for p in base]
    of = nb.FusedAdam(full, **B_HYPER)
    _run(of, full, 0, k + j, seed, dev)
    a = [p.clone() for p in base]
    oa = nb.FusedAdam(a, **B_HYPER)
    _run(oa, a, 0, k, seed, dev)
    pk = [p.clone() for p in a]
    ck_mem = copy.deepcopy(oa.state_dict())
    buf = io.BytesIO()
    torch.save(oa.state_dict(), buf)
    for how, ck in (("deepcopy", lambda: ck_mem), ("torch.load", lambda: torch.load(io.BytesIO(buf.getvalue())))):
        _run(oa, a, k, k + j, seed + 1, dev)             # go on with other gradients
        for p, q in zip(a, pk):
            p.copy_(q)
        oa.load_state_dict(ck())
        _run(oa, a, k, k + j, seed, dev)
        _assert_same(a, full, f"parameters after rollback ({how})")
        _assert_same(_moments(oa, a), _moments(of, full), f"moments after rollback ({how})")
        assert all(int(oa.state[p]["step"]) == k + j for p in a)


def test_torch_adam_checkpoint_resumes_in_fused_adam(dev):
    """A torch.optim.Adam checkpoint (tensor step) resumed by FusedAdam gives the trajectory of FusedAdam continuing
    from identical state with a number step (the form FusedAdam's own checkpoints had before); and a FusedAdam
    checkpoint loads into torch.optim.Adam and steps there."""
    k, j, seed = 6, 5, 22
    base = _params(B_SHAPES, seed, dev)
    a = [p.clone() for p in base]
    ot = torch.optim.Adam(a, **B_HYPER)
    _run(ot, a, 0, k, seed, dev)
    ck = _roundtrip(ot.state_dict())
    assert all(torch.is_tensor(s["step"]) for s in ck["state"].values())
    ck_int = _roundtrip(ck)
    for s in ck_int["state"].values():
        s["step"] = int(s["step"])
    runs = []
    for c in (ck, ck_int):
        b = [p.clone() for p in a]
        ob = nb.FusedAdam(b, **B_HYPER)
        ob.load_state_dict(c)
        _run(ob, b, k, k + j, seed, dev)
        runs.append((b, ob))
    _assert_same(runs[0][0], runs[1][0], "parameters")
    _assert_same(_moments(runs[0][1], runs[0][0]), _moments(runs[1][1], runs[1][0]), "moments")
    assert all(int(runs[0][1].state[p]["step"]) == k + j for p in runs[0][0])
    # the other direction: FusedAdam's checkpoint into torch.optim.Adam
    b, ob = runs[0]
    c = [p.clone() for p in b]
    ot2 = torch.optim.Adam(c, **B_HYPER)
    ot2.load_state_dict(_roundtrip(ob.state_dict()))
    _assert_same(_moments(ot2, c), _moments(ob, b), "moments loaded into torch.optim.Adam")
    _run(ot2, c, k + j, k + j + 2, seed, dev)
    assert all(int(ot2.state[p]["step"]) == k + j + 2 for p in c)


def test_parameters_without_gradient_keep_their_own_step(dev):
    """Steps in which some parameters have grad None: those are skipped and keep their step count; later steps use
    per-parameter bias corrections (as torch.optim.Adam does).  Bit for bit against two FusedAdams that each own one
    of the two sets and step only when their set has gradients; every step also against adam_ref."""
    seed = 23
    base = _params(B_SHAPES, seed, dev)
    a = [p.clone() for p in base]
    oa = nb.FusedAdam(a, **B_HYPER)
    odd = set(range(1, len(a), 2))
    split = [[p.clone() for i, p in enumerate(base) if (i in odd) == s] for s in (False, True)]
    os_ = [nb.FusedAdam(ps, **B_HYPER) for ps in split]
    chk = AdamCheck()
    for t in range(12):
        skip_odd = t in (2, 3, 7)
        skip_even = t in (5,)
        gs = _grads_for(a, t, seed, dev)
        for i, (p, g) in enumerate(zip(a, gs)):
            p.grad = None if (i in odd and skip_odd) or (i not in odd and skip_even) else g.clone()
        chk.step(oa, "partial")
        for s, (ps, o) in enumerate(zip(split, os_)):
            if (skip_odd if s else skip_even):
                continue
            for p, g in zip(ps, [g for i, g in enumerate(gs) if (i in odd) == bool(s)]):
                p.grad = g.clone()
            o.step()
    steps = [_step_of(oa, p) for p in a]
    assert steps == [12 - 3 if i in odd else 12 - 1 for i in range(len(a))], steps
    ev = [p for i, p in enumerate(a) if i not in odd]
    od = [p for i, p in enumerate(a) if i in odd]
    _assert_same(ev, split[0], "parameters (even)")
    _assert_same(od, split[1], "parameters (odd)")
    chk.report("grad None steps")
    assert not chk.bad(), chk.bad()


# ------------------------------------------------------------------------------------------- C. workspace reuse
def _render_step(kind, models, emb, n, S, K, seed, dev):
    """One training step of ``kind`` on fresh copies of the weights.  Returns (workspace, outputs, grads)."""
    rs = np.random.RandomState(seed)
    rays = torch.from_numpy(orc.make_rays(n, seed)).to(dev)
    noise = 1.0 if kind == "noise" else 0.0
    rnd = {"perturb_rand": rs.rand(n, S)}
    if K:
        rnd["u_rand"] = rs.rand(n, K)
    if noise:
        rnd["noise_coarse"] = rs.randn(n, S)
        if K:
            rnd["noise_fine"] = rs.randn(n, S + K)
    rnd = {k: torch.from_numpy(v.astype(np.float32)).to(dev) for k, v in rnd.items()}
    if kind == "seed":
        rnd = {"seed": 3000 + seed}
    args = (S, False, 1.0, noise, K, 32768, True)
    target = torch.from_numpy(rs.uniform(0, 1, (n, 3)).astype(np.float32)).to(dev)
    if kind == "tiny":                 # residuals ~1e-4: the target is the rendered colour of the finest pass
        with torch.no_grad():
            inf = nb.render_rays(models, emb, rays, *args, randoms=rnd)
        target = inf["rgb_fine" if K else "rgb_coarse"] + torch.from_numpy(
            rs.uniform(-1e-4, 1e-4, (n, 3)).astype(np.float32)).to(dev)
    if kind == "all6":
        out = nb.render_rays(models, emb, rays, *args, randoms=rnd)
        g = torch.Generator(device=dev).manual_seed(seed)
        loss = sum((v * torch.randn(v.shape, device=dev, generator=g)).sum() for v in out.values()) / n
        res = {k: v.detach() for k, v in out.items()}
    else:
        out = nb.render_rays_loss(models, emb, rays, target, *args[:5], 32768, True, randoms=rnd)
        loss = out["loss"]
        res = {k: v.detach() for k, v in out.items() if k != "loss"}
        res["loss"] = loss.detach()
    ws = out["rgb_coarse"].grad_fn.keep[-1]
    loss.backward()
    assert _status_ok(), kind
    grads = [p.grad.clone() for m in models[:2 if K else 1] for p in m.parameters()]
    return ws, res, grads


SEQUENCE = ("large", "tiny", "noise", "seed", "all6", "large")


@pytest.mark.parametrize("n,S,K", [(64, 64, 64), (64, 64, 0), (1024, 64, 64)])
def test_reused_render_workspace_has_no_memory(n, S, K, dev, emb):
    """A probe step (residuals ~1e-4) on a workspace that has served a sequence of other steps (large residuals,
    sigma noise, in-kernel uniforms, upstream gradients on all outputs, then large residuals again) equals the
    same step on a fresh workspace: outputs, loss and every .grad element, bit for bit; status 0 after each."""
    ws_np = cases.weights()
    TrainWorkspace.clear()
    used = None
    for i, kind in enumerate(SEQUENCE):
        ws, _, _ = _render_step(kind, _models(ws_np, dev), emb, n, S, K, 400 + i, dev)
        assert used is None or ws is used, "the sequence did not reuse one workspace"
        used = ws
    ws_a, out_a, g_a = _render_step("tiny", _models(ws_np, dev), emb, n, S, K, 499, dev)
    assert ws_a is used
    held = dict(TrainWorkspace._pool)           # keep the used workspace alive: the fresh one is new memory
    TrainWorkspace.clear()
    ws_b, out_b, g_b = _render_step("tiny", _models(ws_np, dev), emb, n, S, K, 499, dev)
    assert ws_b is not used
    del held
    for k in out_a:
        assert torch.equal(out_a[k], out_b[k]), k
    _assert_same(g_a, g_b, "gradients on a reused vs a fresh workspace")


def test_reused_nerf_workspace_has_no_memory(dev):
    """The same for nerf_forward_train (NeRF.forward with autograd_impl='fused') and its NerfTrainWorkspace pool:
    upstream gradients ~0.3, ~1e-4, skewed, sigma only, ~0.3; then a ~1e-4 probe, reused vs fresh."""
    n = 5000
    w = cases.weights()[0]
    rs = np.random.RandomState(600)
    x = torch.from_numpy(np.concatenate([orc.embed(rs.uniform(-1.5, 1.5, (n, 3)).astype(np.float32), 10),
                                         orc.embed(rs.randn(n, 3).astype(np.float32), 4)], 1).astype(np.float32)).to(dev)

    def step(kind, seed):
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        m = m.to(dev)
        m.autograd_impl = "fused"
        r = np.random.RandomState(seed)
        g = (r.randn(n, 4) * 0.3).astype(np.float32)
        if kind == "tiny":
            g *= 1e-4 / 0.3
        elif kind == "skewed":
            g[:256] *= 1e-4 / 0.3
        elif kind == "sigma":
            g[:, :3] = 0
        out = m(x)
        ws = out.grad_fn.lease.ws
        out.backward(torch.from_numpy(g).to(dev))
        assert _status_ok(), kind
        return ws, out.detach(), [p.grad.clone() for p in m.parameters()]

    NerfTrainWorkspace.clear()
    used = None
    for i, kind in enumerate(("large", "tiny", "skewed", "sigma", "large")):
        ws, _, _ = step(kind, 610 + i)
        assert used is None or ws is used
        used = ws
    ws_a, out_a, g_a = step("tiny", 620)
    assert ws_a is used
    held = dict(NerfTrainWorkspace._pool)
    NerfTrainWorkspace.clear()
    ws_b, out_b, g_b = step("tiny", 620)
    assert ws_b is not used
    del held
    assert torch.equal(out_a, out_b)
    _assert_same(g_a, g_b, "gradients on a reused vs a fresh workspace")


# ------------------------------------------------------------------------------------------- D. workspace lifetime
def _render_pool(dev):
    return [ws for key, wss in TrainWorkspace._pool.items() if key[0] == dev.index for ws in wss]


def test_render_workspace_pool_stays_bounded(dev, emb):
    """Renders under grad mode whose outputs are dropped without a backward (a skipped batch, a metric) leave one
    idle workspace, not one per call; renders with a pending backward each hold their own; a second backward of
    the same graph is a clear RuntimeError."""
    TrainWorkspace.clear()
    try:
        models = _models(cases.weights(), dev)
        rays = torch.from_numpy(orc.make_rays(64, 700)).to(dev)
        tgt = torch.rand(64, 3, device=dev)
        args = (64, False, 1.0, 0.0, 64, 32768, True)
        out = nb.render_rays(models, emb, rays, *args, randoms={"seed": 1})
        float(out["rgb_fine"].mean())
        del out
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated(dev)
        for i in range(40):
            if i % 2:
                out = nb.render_rays(models, emb, rays, *args, randoms={"seed": i})
            else:
                out = nb.render_rays_loss(models, emb, rays, tgt, *args[:5], 32768, True, randoms={"seed": i})
            float(out["rgb_fine"].mean())          # used for a metric only
            del out
        pool = _render_pool(dev)
        assert len(pool) == 1 and not pool[0].busy, f"{len(pool)} workspaces after 40 dropped renders"
        torch.cuda.synchronize()
        assert torch.cuda.memory_allocated(dev) <= base
        outs = [nb.render_rays_loss(models, emb, rays, tgt, *args[:5], 32768, True, randoms={"seed": 50 + i})
                for i in range(3)]
        assert sum(ws.busy for ws in _render_pool(dev)) == 3
        sum(o["loss"] for o in outs).backward()
        assert not any(ws.busy for ws in _render_pool(dev))
        del outs
        out = nb.render_rays_loss(models, emb, rays, tgt, *args[:5], 32768, True, randoms={"seed": 60})
        out["loss"].backward(retain_graph=True)
        with pytest.raises(RuntimeError, match="already run"):
            out["loss"].backward()
        del out
        assert len(_render_pool(dev)) == 3 and not any(ws.busy for ws in _render_pool(dev))
        assert _status_ok()
    finally:
        TrainWorkspace.clear()


# ------------------------------------------------------------------------------------------- E. a short training run
E_STEPS = 40
E_CHECK = (0, E_STEPS // 2, E_STEPS - 1)        # steps with the full stage report
# Bars of E against autograd_impl='torch' and the torch loop; measured worst on an H100 80GB HBM3 (700 W) in
# brackets.  Whole gradient: relative L2 / cosine over all 48 tensors; per tensor: the worst tensor of any step.
# From the random start the bars of test_training_step_gradients_vs_reference_golden hold.  With trained weights
# (sharp density) the fp16 forward flips the ReLU masks of more pre-activations, each an O(1) error in that
# element's gradient; on its own masks the kernel stays as close to float64 as from the random start (the stage
# reports, which also held at steps 10, 31 and 38, the three steps above 1e-2), so there the whole-gradient bar is
# wider and the per-tensor bars carry the check.  The loss curves of
# the two loops share only their start: the trajectories diverge, so no bar applies to the weights.
E_BARS = {
    "random": {"grad_rel": 5e-3, "grad_cos": 0.9999,             # [4.9e-4, 1.000000]
               "grad_rel_tensor": 8e-2, "grad_cos_tensor": 0.997,  # [5.4e-3, 0.999986]
               "loss_rel": 1e-3},                                  # [1.1e-4]
    "trained": {"grad_rel": 5e-2, "grad_cos": 0.999,             # [2.8e-2 at step 10, else <= 1.3e-2; 0.99960]
                "grad_rel_tensor": 0.15, "grad_cos_tensor": 0.99,  # [0.078, 0.996999: coarse layer 2, step 31]
                "loss_rel": 5e-2},                                 # [1.7e-2]
}


def _np_weights(models):
    return [{k: v.detach().cpu().numpy() for k, v in m.state_dict().items()} for m in models]


def _named_grads(models):
    return {f"{tag}.{k}": p.grad.detach().cpu().numpy() for tag, m in zip(("coarse", "fine"), models)
            for k, p in m.named_parameters()}


@pytest.mark.parametrize("start", ["random", "trained"])
def test_short_training_run(start, dev, emb):
    """40 steps of render_rays_loss -> backward -> FusedAdam.step on 1024 rays at 64 + 64, with seeded pre-drawn
    randoms that differ per step.  Targets: the trained fine network's render at perturbed depths (start 'random'),
    or that render through a gamma of 1.5 (start 'trained'), so that the loss falls and the residuals, and with them
    the per-layer gradient scales, shrink over the run.  Every step: the Adam update against adam_ref, status 0,
    the packed image current, the gradient against autograd_impl='torch' at the loop's weights and randoms.  Steps
    0, 20, 39: the full stage report of test_gpu_train_stages.py.  End: the loss curve against a parallel loop with
    autograd_impl='torch' + torch.optim.Adam from the same start.  Their trajectories diverge (ReLU-mask flips
    of the fp16 forward differ per step), so only the losses are compared, not the weights."""
    n, S, K = 1024, 64, 64
    rays_np = orc.make_rays(n, 130)
    rays = torch.from_numpy(rays_np).to(dev)
    trained_np = cases.trained_weights()
    with torch.no_grad():
        target = nb.render_rays(_models(trained_np, dev), emb, rays, S, False, 1.0, 0.0, K, 32768, True,
                                randoms={"seed": 131})["rgb_fine"]
    if start == "trained":
        target = target.clamp(0, 1) ** 1.5
    start_np = trained_np if start == "trained" else cases.weights()
    models = _models(start_np, dev)
    models_t = _models(start_np, dev)
    params = [p for m in models for p in m.parameters()]
    opt = nb.FusedAdam(params, lr=5e-4, eps=1e-8)
    opt_t = torch.optim.Adam([p for m in models_t for p in m.parameters()], lr=5e-4, eps=1e-8)
    chk = AdamCheck()
    args = (S, False, 1.0, 0.0, K, 32768, True)
    bars = E_BARS[start]
    losses, losses_t, grad_rows, bad = [], [], [], []
    tensor_worst = [0.0, "", 1.0, ""]
    secs = {}

    def lap(name, t0=[None]):
        torch.cuda.synchronize()
        now = time.perf_counter()
        if name is not None:
            secs[name] = secs.get(name, 0.0) + now - t0[0]
        t0[0] = now

    pool = ThreadPoolExecutor(len(E_CHECK))     # the float64 stage reports run on the host beside the loop
    reports = []
    lap(None)
    for step in range(E_STEPS):
        g = torch.Generator(device=dev).manual_seed(140 + step)
        rnd = {"perturb_rand": torch.rand(n, S, device=dev, generator=g), "u_rand": torch.rand(n, K, device=dev, generator=g)}
        # packed image current: the loop's modules render like fresh modules with the same weights
        with torch.no_grad():
            a = nb.render_rays(models, emb, rays, S, False, 0.0, 0.0, K, 32768, True)
            b = nb.render_rays(_models(_np_weights(models), dev), emb, rays, S, False, 0.0, 0.0, K, 32768, True)
        if not all(torch.equal(a[k], b[k]) for k in a):
            bad.append(f"step {step}: the loop's render differs from fresh modules with its weights")
        lap("packed image")
        # the gradient reference: autograd_impl='torch' at the loop's current weights and this step's randoms
        ref_models = _models(_np_weights(models), dev)
        out_r = nb.render_rays(ref_models, emb, rays, *args, randoms=rnd, autograd_impl="torch")
        (((out_r["rgb_coarse"] - target) ** 2).mean() + ((out_r["rgb_fine"] - target) ** 2).mean()).backward()
        lap("torch gradient")
        # the fused step
        opt.zero_grad(set_to_none=True)
        out = nb.render_rays_loss(models, emb, rays, target, *args[:5], 32768, True, randoms=rnd)
        ws = out["rgb_coarse"].grad_fn.keep[-1]
        out["loss"].backward()
        if not _status_ok():
            bad.append(f"step {step}: status after the backward")
        losses.append(float(out["loss"]))
        lap("fused step")
        rows, (rel, cos) = og.grad_compare(_named_grads(models), _named_grads(ref_models))
        grad_rows.append((rel, cos))
        for k, (r, c) in rows.items():
            if r > tensor_worst[0]:
                tensor_worst[:2] = r, f"{k} step {step}"
            if c < tensor_worst[2]:
                tensor_worst[2:] = c, f"{k} step {step}"
        lap("gradient compare")
        if step in E_CHECK:
            with torch.no_grad():
                inf = nb.render_rays(models, emb, rays, *args, randoms=rnd, extras=True)
            rgb = {p: out[f"rgb_{p}"].detach().cpu().numpy().astype(np.float64) for p in ("coarse", "fine")}
            tnp = target.cpu().numpy().astype(np.float64)
            run = dict(c=dict(use_disp=False, perturb=1.0, noise_std=0.0, white_back=True), n=n, S=S, K=K,
                       rays=rays_np, randoms={k: v.cpu().numpy() for k, v in rnd.items()},
                       raw=ws.buf.cpu().numpy(),
                       grads=[{k: p.grad.detach().cpu().numpy() for k, p in m.named_parameters()} for m in models],
                       seeds=[((2.0 * (rgb[p] - tnp) / (3 * n)).astype(np.float32), None, None)
                              for p in ("coarse", "fine")],
                       noise=[None, None], ws=_np_weights(models), z_fine=inf["z_vals_fine"].cpu().numpy(),
                       seed=150 + step)
            reports.append((step, pool.submit(stage_report, run)))
            del run
            lap("stage report inputs")
        chk.step(opt, f"run {start}")
        if not _status_ok():
            bad.append(f"step {step}: status after the Adam step")
        lap("Adam + check")
        # the parallel torch loop
        opt_t.zero_grad(set_to_none=True)
        out_t = nb.render_rays(models_t, emb, rays, *args, randoms=rnd, autograd_impl="torch")
        loss_t = ((out_t["rgb_coarse"] - target) ** 2).mean() + ((out_t["rgb_fine"] - target) ** 2).mean()
        loss_t.backward()
        opt_t.step()
        losses_t.append(float(loss_t))
        lap("torch loop")
    for step, rep in reports:
        lines, sbad = rep.result()
        print(f"\n[{start} step {step}] stage report")
        print("\n".join(lines))
        bad += [f"step {step}: {b}" for b in sbad]
    pool.shutdown()
    lap("stage reports (rest)")
    chk.report(f"training run, {start} start")
    print(f"[{start}] gradient vs autograd_impl='torch', whole (rel L2, cos) per step: " +
          " ".join(f"({r:.2e},{c:.6f})" for r, c in grad_rows))
    print(f"[{start}] worst per tensor: rel {tensor_worst[0]:.3g} ({tensor_worst[1]}) cos {tensor_worst[2]:.6f} "
          f"({tensor_worst[3]})")
    print(f"[{start}] seconds: " + " ".join(f"{k} {v:.1f}" for k, v in secs.items()))
    rel_loss = [abs(x - y) / y for x, y in zip(losses, losses_t)]
    print(f"[{start}] loss fused: " + " ".join(f"{x:.5g}" for x in losses))
    print(f"[{start}] loss torch: " + " ".join(f"{x:.5g}" for x in losses_t))
    print(f"[{start}] worst relative loss difference {max(rel_loss):.3g}")
    worst_rel = max(r for r, _ in grad_rows)
    worst_cos = min(c for _, c in grad_rows)
    print(f"[{start}] worst whole gradient: rel {worst_rel:.3g} cos {worst_cos:.6f}")
    if not (worst_rel < bars["grad_rel"] and worst_cos > bars["grad_cos"]):
        bad.append(f"whole-gradient error rel {worst_rel:.3g} cos {worst_cos:.6f}")
    if not (tensor_worst[0] < bars["grad_rel_tensor"] and tensor_worst[2] > bars["grad_cos_tensor"]):
        bad.append(f"per-tensor gradient error rel {tensor_worst[0]:.3g} cos {tensor_worst[2]:.6f}")
    if not max(rel_loss) < bars["loss_rel"]:
        bad.append(f"loss curves differ by {max(rel_loss):.3g} relative")
    if not np.mean(losses[-5:]) < 0.9 * np.mean(losses[:5]):
        bad.append(f"the loss did not fall: {np.mean(losses[:5]):.4g} -> {np.mean(losses[-5:]):.4g}")
    bad += [f"Adam {k} {v:.3g} ulps" for k, v in chk.bad().items()]
    assert not bad, "\n".join(bad)
