"""render_rays(..., occupancy=grid) on the device: with a gradient graph every output is differentiable and its
forward is render_rays_loss(..., occupancy=)'s; without one it is culling.render_samples over every ray, equal to the
graph path's forward for the same randoms and, unperturbed, to render_rays_culled(skip="samples").  The general seed
of the sparse compositing backward is held to the float64 restatement (tests/train_skip_seed_ref.py) and the 48
gradients to DESIGN.md section 2's bars."""
from collections import defaultdict

import numpy as np
import pytest
import torch

from tests import sample_skip_ref as sk
from tests import test_gpu_train_skip as ts
from tests import train_skip_ref as tr
from tests import train_skip_seed_ref as seed_ref

pytestmark = pytest.mark.gpu
KEYS = ts.KEYS


def _nb():
    import nerf_pl_b200 as nb
    return nb


def _grads(models, K):
    return {f"{i}.{k}": (p.grad if p.grad is not None else torch.zeros_like(p)).detach().cpu().numpy().astype(np.float64)
            for i, m in enumerate(models[:2 if K else 1]) for k, p in m.named_parameters()}


def _weights(n, K, seed):
    """Random per-ray weights of a loss on every output."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = {}
    for k in KEYS[:6 if K else 3]:
        w[k] = torch.randn((n, 3) if k.startswith("rgb") else (n,), device="cuda", generator=g)
        if k.startswith("depth"):
            w[k] = w[k] * 0.1
    return w


def _wloss(res, w):
    return sum((res[k] * w[k]).sum() for k in w)


def _render(models, rays, S, K, use_disp, perturb, noise, white_back, randoms, grid=None, **kw):
    return _nb().render_rays(models, ts._emb(), rays, S, use_disp, perturb, noise, K, 32768, white_back,
                             randoms=randoms, occupancy=grid, **kw)


def _kernel_randoms(n, S, K, seed):
    return {"seed": 1234, **{k: v for k, v in ts._randoms(n, S, K, seed).items() if k.startswith("noise")}}


@pytest.mark.parametrize("S,K", [(32, 0), (64, 0), (128, 0), (64, 64), (128, 64), (64, 128), (32, 128)])
@pytest.mark.parametrize("kind,use_disp,noise,white_back", [("blender", False, 1.0, True), ("blender", True, 0.0, False),
                                                           ("ndc", False, 1.0, False), ("ndc", False, 0.0, True)])
@pytest.mark.parametrize("rng", ["tensor", "kernel"])
def test_full_grid_is_plain_render_rays(S, K, kind, use_disp, noise, white_back, rng):
    n = 700
    rays = ts._rays(kind, n, 3)
    randoms = ts._randoms(n, S, K, 5) if rng == "tensor" else _kernel_randoms(n, S, K, 5)
    models = ts._models()
    grid = ts._grid(1.0, ts.FULL, N=3)
    w = _weights(n, K, 9)
    out = []
    for occ in (None, grid):
        for m in models:
            m.zero_grad(set_to_none=True)
        res = _render(models, rays, S, K, use_disp, 1.0, noise, white_back, randoms, occ)
        assert sorted(res) == sorted(KEYS[:6 if K else 3])
        assert all(v.requires_grad for v in res.values())
        _wloss(res, w).backward()
        out.append((res, _grads(models, K)))
    (want, gw), (got, gg) = out
    for k in want:
        assert ts._same(got[k].detach(), want[k].detach()), k
    tot, worst = ts._grad_bars(gg, gw)
    print(f"\nS={S} K={K} {kind}: whole-gradient rel L2 {tot:.2e}, worst tensor {worst:.2e}")
    assert _nb()._lib.load().nerfb200_check_status() == 0


def _autograd_reference(models, rays, got, S, K, noise_std, white_back, randoms, w, copies=(0, 0)):
    """The 24 or 48 gradients of sum_k <w_k, out_k> as an autograd composition: the evaluated rows through
    NeRF.forward, float64 torch compositing with skipped samples at sigma = 0 (exact zeros for a network with no
    evaluated row).  `copies` plants ts._last_row_counted in the coarse / fine pass."""
    nb = _nb()
    n = rays.shape[0]
    loss = 0.0
    for ps, (model, Sp) in enumerate(((models[0], S), (models[1], S + K))[:2 if K else 1]):
        name = "coarse" if ps == 0 else "fine"
        z = got["z_vals_" + name]
        ev = torch.from_numpy(sk.mask_bits(got["mask_" + name].cpu().numpy(), Sp)).cuda()
        xyz = (rays[:, None, 0:3] + rays[:, None, 3:6] * z[:, :, None])[ev]
        d = rays[:, None, 3:6].expand(n, Sp, 3)[ev]
        x = torch.cat([nb.Embedding(3, 10)(xyz), nb.Embedding(3, 4)(d)], -1)
        out = ts._last_row_counted(model(x), copies[ps]) if x.shape[0] else x.new_zeros(0, 4)
        s_ev = out[:, 3].double()
        if noise_std > 0:
            s_ev = s_ev + randoms["noise_" + name][ev].double() * noise_std
        sig = torch.zeros(n, Sp, dtype=torch.float64, device="cuda").index_put((ev,), s_ev)
        rgb = torch.zeros(n, Sp, 3, dtype=torch.float64, device="cuda").index_put((ev,), out[:, :3].double())
        c, dep, op = tr.composite_torch(z.double(), sig, rgb, rays[:, 3:6].double(), white_back)
        loss = loss + (c * w["rgb_" + name]).sum() + (dep * w["depth_" + name]).sum() + (op * w["opacity_" + name]).sum()
    for m in models:
        m.zero_grad(set_to_none=True)
    if loss.requires_grad:
        loss.backward()
    return _grads(models, K)


def _partial(n, S, K, noise, white_back, w, seed=8):
    """One step of sum_k <w_k, out_k> on a partial grid through render_rays_train_skip(target=None, extras=True)."""
    rays = ts._rays("blender", n, 7)
    grid = ts._grid(0.3, ((-2.0, 2.0), (2.0, -2.0), (-1.5, 2.5)), N=9, seed=3)
    randoms = ts._randoms(n, S, K, seed)
    models = ts._models()
    from nerf_pl_b200.train_skip import render_rays_train_skip
    for m in models:
        m.zero_grad(set_to_none=True)
    got = render_rays_train_skip(models, rays, S, False, 1.0, noise, K, white_back, randoms["perturb_rand"],
                                 randoms["noise_coarse"] if noise else None, randoms["u_rand"],
                                 randoms["noise_fine"] if noise else None, None, grid, extras=True)
    assert "loss" not in got
    _wloss(got, w).backward()
    return rays, randoms, models, got


@pytest.mark.parametrize("S,K,noise,white_back", [(64, 128, 1.0, True), (32, 64, 0.0, False), (64, 64, 1.0, False)])
def test_partial_grid_general_seed(S, K, noise, white_back):
    n = 1000
    w = _weights(n, K, 11)
    rays, randoms, models, got = _partial(n, S, K, noise, white_back, w)
    gg = _grads(models, K)
    rn = rays.cpu().numpy()
    wn = {k: v.cpu().numpy() for k, v in w.items()}
    for ps, (name, Sp) in enumerate((("coarse", S), ("fine", S + K))):
        ev = sk.mask_bits(got["mask_" + name].cpu().numpy(), Sp)
        assert 0.05 < ev.mean() < 0.95
        smp = got["samples_" + name].cpu().numpy()
        rows = int(ev.sum())
        ds = got["dsigma_" + name][:rows].cpu().numpy()
        dp = got["dprergb_" + name][:rows].cpu().numpy()
        noise_t = randoms["noise_" + name].cpu().numpy() if noise else None
        other = "fine" if ps == 0 else "coarse"

        def ref(seeds=name, g_depth=True, g_opacity=True, wb=white_back):
            return seed_ref.backward(got["z_vals_" + name].cpu().numpy(), smp[..., 3], smp[..., :3], ev, rn[:, 3:6],
                                     noise_t, noise, wb, wn["rgb_" + seeds],
                                     wn["depth_" + seeds] if g_depth else None,
                                     wn["opacity_" + seeds] if g_opacity else None)

        ds_ref, dp_ref = ref()
        errs = tr.backward_errors(ds, dp, ev, ds_ref, dp_ref)
        print(f"\n{name}: per-row d sigma error {errs[0]:.2e}, d rgb_pre {errs[1]:.2e} (bar {tr.BWD_BAR})")
        assert max(errs) <= tr.BWD_BAR, (name, errs)
        planted = {"depth seed dropped": dict(g_depth=False), "opacity seed dropped": dict(g_opacity=False),
                   "white_back ignored": dict(wb=not white_back), "passes swapped": dict(seeds=other)}
        for what, kw in planted.items():
            bds, bdp = ref(**kw)
            bad = tr.backward_errors(bds[ev].astype(np.float32), bdp[ev].astype(np.float32), ev, ds_ref, dp_ref)
            assert max(bad) > tr.BWD_BAR, (name, what, bad)
    tot, worst = ts._grad_bars(gg, _autograd_reference(models, rays, got, S, K, noise, white_back, randoms, w))
    print(f"\npartial grid S={S} K={K}: whole-gradient rel L2 {tot:.2e}, worst tensor {worst:.2e}")


@pytest.mark.parametrize("only", ["depth_fine", "opacity_fine", "rgb_coarse", "depth_coarse"])
def test_one_seed_at_a_time(only):
    """One output seeded: the other network's 24 gradients are exact zeros, the seeded network's are finite and
    not all zero."""
    n, S, K = 800, 64, 64
    rays = ts._rays("blender", n, 5)
    grid = ts._grid(0.3, ((-1.5, 1.5),) * 3, N=17, seed=1)
    models = ts._models()
    for m in models:
        m.zero_grad(set_to_none=True)
    res = _render(models, rays, S, K, False, 1.0, 1.0, True, ts._randoms(n, S, K, 2), grid)
    w = torch.randn(res[only].shape, device="cuda")
    (res[only] * w).sum().backward()
    seeded = models[1] if only.endswith("fine") else models[0]
    other = models[0] if only.endswith("fine") else models[1]
    assert all(torch.equal(p.grad, torch.zeros_like(p.grad)) for p in other.parameters()), only
    assert all(torch.isfinite(p.grad).all() for p in seeded.parameters())
    assert any(p.grad.any() for p in seeded.parameters())
    assert _nb()._lib.load().nerfb200_check_status() == 0


@pytest.mark.parametrize("S,K,rng", [(64, 128, "tensor"), (64, 64, "kernel"), (128, 0, "tensor")])
def test_against_the_fused_loss(S, K, rng):
    """render_rays(occupancy=) + the reference's MSELoss (losses.py: coarse + fine) against render_rays_loss(occupancy=):
    the same outputs bit for bit, gradients within the bars."""
    n = 900
    rays = ts._rays("blender", n, 4)
    rgbs = torch.rand(n, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    grid = ts._grid(0.3, ((-1.5, 1.5),) * 3, N=17, seed=4)
    randoms = ts._randoms(n, S, K, 6) if rng == "tensor" else _kernel_randoms(n, S, K, 6)
    models = ts._models()
    want, gw = ts._step(models, rays, rgbs, S, K, False, 1.0, True, randoms, grid)
    for m in models:
        m.zero_grad(set_to_none=True)
    got = _render(models, rays, S, K, False, 1.0, 1.0, True, randoms, grid)
    mse = torch.nn.MSELoss(reduction="mean")
    loss = mse(got["rgb_coarse"], rgbs)
    if K:
        loss = loss + mse(got["rgb_fine"], rgbs)
    loss.backward()
    for k in got:
        assert ts._same(got[k].detach(), want[k].detach()), k
    assert abs(float(loss.detach()) - float(want["loss"].detach())) <= 1e-6 * abs(float(want["loss"].detach()))
    tot, worst = ts._grad_bars(_grads(models, K), gw)
    print(f"\nuser MSE vs fused S={S} K={K}: whole-gradient rel L2 {tot:.2e}, worst tensor {worst:.2e}")


@pytest.mark.parametrize("test_time", [False, True])
@pytest.mark.parametrize("extras", [False, True])
def test_no_graph_unperturbed_is_render_rays_culled(test_time, extras):
    n, S, K = 1500, 64, 128
    rays = ts._rays("blender", n, 6)
    grid = ts._grid(0.3, ((-1.5, 1.5),) * 3, N=17, seed=6)
    models = ts._models()
    with torch.no_grad():
        got = _render(models, rays, S, K, False, 0.0, 0.0, True, None, grid, test_time=test_time, extras=extras)
        want = _nb().render_rays_culled(models, ts._emb(), rays, grid, S, False, K, True, test_time, skip="samples",
                                        extras=extras)
    keys = ts.KEYS if not test_time else ("opacity_coarse",) + ts.KEYS[3:]
    extra_keys = ("weights_coarse", "weights_fine", "z_vals_fine") if extras else ()
    assert sorted(got) == sorted(keys + extra_keys)
    for k in got:
        assert ts._same(got[k], want[k]), k


@pytest.mark.parametrize("rng", ["tensor", "kernel"])
@pytest.mark.parametrize("S,K", [(64, 128), (32, 0)])
def test_no_graph_is_the_graph_forward(monkeypatch, rng, S, K):
    """perturb = noise = 1: the no-graph render, in chunks of 257 rays, gives the graph path's forward bit for bit."""
    from nerf_pl_b200 import culling
    n = 1300
    rays = ts._rays("blender", n, 8)
    grid = ts._grid(0.3, ((-1.5, 1.5),) * 3, N=17, seed=7)
    randoms = ts._randoms(n, S, K, 9) if rng == "tensor" else _kernel_randoms(n, S, K, 9)
    models = ts._models()
    graph = _render(models, rays, S, K, False, 1.0, 1.0, True, randoms, grid)
    assert all(v.requires_grad for v in graph.values())
    monkeypatch.setattr(culling, "_SAMPLE_CHUNK", 257)
    with torch.no_grad():
        plain = _render(models, rays, S, K, False, 1.0, 1.0, True, randoms, grid)
    assert sorted(plain) == sorted(graph)
    for k in graph:
        assert ts._same(plain[k], graph[k].detach()), k
    # the perturbation is live: an unperturbed render differs
    with torch.no_grad():
        flat = _render(models, rays, S, K, False, 0.0, 0.0, True, None, grid)
    assert not ts._same(flat["opacity_coarse"], plain["opacity_coarse"])


def _system_forward(models, rays, grid, S, K, chunk):
    """The reference's NeRFSystem.forward (train.py): render_rays per chunk, then torch.cat of every key."""
    B = rays.shape[0]
    results = defaultdict(list)
    for i in range(0, B, chunk):
        rendered = _nb().render_rays(models, ts._emb(), rays[i:i + chunk], S, False, 0.0, 0.0, K, chunk, False, False,
                                     occupancy=grid)
        for k, v in rendered.items():
            results[k] += [v]
    return {k: torch.cat(v, 0) for k, v in results.items()}


def test_the_references_chunked_forward():
    n, S, K, chunk = 700, 64, 64, 256
    rays = ts._rays("blender", n, 10)
    grid = ts._grid(0.3, ((-1.5, 1.5),) * 3, N=17, seed=8)
    models = ts._models()
    w = _weights(n, K, 12)
    out = []
    for c in (chunk, n):
        for m in models:
            m.zero_grad(set_to_none=True)
        res = _system_forward(models, rays, grid, S, K, c)
        assert sorted(res) == sorted(KEYS)
        _wloss(res, w).backward()
        out.append((res, _grads(models, K)))
    (got, gg), (want, gw) = out
    for k in want:       # unperturbed: a ray's values do not depend on its chunk
        assert ts._same(got[k].detach(), want[k].detach()), k
    ts._grad_bars(gg, gw)
    with torch.no_grad():
        res = _system_forward(models, rays, grid, S, K, chunk)
    assert sorted(res) == sorted(KEYS)
    for k in res:
        assert ts._same(res[k], want[k].detach()), k


def test_capture():
    """Forward + an L1 loss + backward captured in one CUDA graph: replays give the eager outputs and gradients bit for
    bit."""
    n, S, K = 1024, 64, 64
    rays = ts._rays("blender", n, 13)
    rgbs = torch.rand(n, 3, device="cuda")
    grid = ts._grid(0.3, ((-1.5, 1.5),) * 3, N=17, seed=9)
    randoms = ts._randoms(n, S, K, 10)
    models = ts._models()
    params = [p for m in models for p in m.parameters()]

    def step():
        res = _render(models, rays, S, K, False, 1.0, 1.0, False, randoms, grid)
        loss = (res["rgb_coarse"] - rgbs).abs().mean() + (res["rgb_fine"] - rgbs).abs().mean()
        return [res[k] for k in KEYS] + [loss] + list(torch.autograd.grad(loss, params))

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            eager = [t.detach().clone() for t in step()]
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        static = step()
    for _ in range(3):
        for t in static:
            t.detach().zero_()
        g.replay()
        torch.cuda.synchronize()
        for a, b in zip(static, eager):
            assert ts._same(a.detach(), b)
    assert _nb()._lib.load().nerfb200_check_status() == 0
