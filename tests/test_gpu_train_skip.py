"""render_rays_loss(..., occupancy=grid) on the device (nerf_pl_b200/train_skip.py, csrc/train_skip_kernels.cuh): with
nothing to skip its results are the plain training step's bit for bit and its gradients meet DESIGN.md section 2's bars
against it; on a partial grid its evaluated set is the float64 rule (tests/sample_skip_ref.py) on its own perturbed
depths, skipped samples have weight 0, compositing is the float64 restatement (tests/train_skip_ref.py) and the 48
gradients match an autograd composition of NeRF on the same rows; vacuum and degenerate rays, batch order, and a
workspace that never grows."""
import numpy as np
import pytest
import torch

import bench
from oracle import nerf_oracle as orc
from tests import sample_skip_ref as sk
from tests import train_skip_ref as tr

pytestmark = pytest.mark.gpu
FULL = ((-1e4, 1e4),) * 3


def _nb():
    import nerf_pl_b200 as nb
    return nb


def _emb():
    return [_nb().Embedding(3, 10), _nb().Embedding(3, 4)]


def _models(seed=0):
    ms = []
    for s in (21 + seed, 22 + seed):
        m = _nb().NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in orc.make_weights(s).items()})
        ms.append(m.cuda())
    return ms


def _grid(fill, ranges, N=33, seed=0):
    rng = np.random.default_rng(seed)
    sigma = np.where(rng.random((N, N, N)) < fill, 5.0, 0.0).astype(np.float32)
    return _nb().pack_occupancy(torch.from_numpy(sigma).cuda(), *ranges, 1.0, 0)


def _rays(kind, n, seed):
    if kind == "ndc":
        r = orc.make_rays(n, seed).copy()
        r[:, 6], r[:, 7] = 0.0, 1.0
        return torch.from_numpy(r).cuda()
    return torch.from_numpy(bench.blender_rays(n, seed)).cuda()


def _randoms(n, S, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = dict(perturb_rand=torch.rand(n, S, device="cuda", generator=g),
             noise_coarse=torch.randn(n, S, device="cuda", generator=g))
    if K:
        r.update(u_rand=torch.rand(n, K, device="cuda", generator=g),
                 noise_fine=torch.randn(n, S + K, device="cuda", generator=g))
    return r


def _step(models, rays, rgbs, S, K, use_disp, noise, white_back, randoms, occupancy=None):
    for m in models:
        m.zero_grad(set_to_none=True)
    res = _nb().render_rays_loss(models, _emb(), rays, rgbs, S, use_disp, 1.0, noise, K, 32768, white_back,
                                 randoms=randoms, occupancy=occupancy)
    res["loss"].backward()
    grads = {f"{i}.{k}": p.grad.detach().cpu().numpy().astype(np.float64)
             for i, m in enumerate(models[:2 if K else 1]) for k, p in m.named_parameters()}
    return res, grads


def _same(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _grad_bars(got, ref):
    """DESIGN section 2's end-to-end bars: per tensor relative L2 < 8e-2, cosine > 0.997; whole gradient < 5e-3."""
    num = den = 0.0
    worst = 0.0
    for k, r in ref.items():
        a = got[k]
        num += float(((a - r) ** 2).sum())
        den += float((r ** 2).sum())
        rel = np.linalg.norm(a - r) / max(np.linalg.norm(r), 1e-30)
        cos = float((a * r).sum() / max(np.linalg.norm(a) * np.linalg.norm(r), 1e-30))
        assert rel < 8e-2 and cos > 0.997, f"{k}: rel {rel:.3e} cos {cos:.5f}"
        worst = max(worst, rel)
    tot = (num / den) ** 0.5
    assert tot < 5e-3, tot
    return tot, worst


KEYS = ("rgb_coarse", "depth_coarse", "opacity_coarse", "rgb_fine", "depth_fine", "opacity_fine")
# every (N_samples, N_importance) pair the C ABI accepts (capi.cu samples_shape_ok)
PAIRS = [(S, K) for S in (32, 64, 128) for K in range(0, 193 - S, 32)]


@pytest.mark.parametrize("S,K", PAIRS)
@pytest.mark.parametrize("kind,use_disp,noise,white_back", [("blender", False, 1.0, True), ("blender", True, 0.0, False),
                                                           ("ndc", False, 1.0, False), ("ndc", False, 0.0, True)])
@pytest.mark.parametrize("rng", ["tensor", "kernel"])
def test_nothing_to_skip_is_the_plain_step(S, K, kind, use_disp, noise, white_back, rng):
    n = 700
    rays = _rays(kind, n, 3)
    rgbs = torch.rand(n, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    randoms = _randoms(n, S, K, 5) if rng == "tensor" else {"seed": 1234, **{k: v for k, v in _randoms(n, S, K, 5).items()
                                                                           if k.startswith("noise")}}
    models = _models()
    grid = _grid(1.0, FULL, N=3)
    want, gw = _step(models, rays, rgbs, S, K, use_disp, noise, white_back, randoms)
    assert _nb()._lib.load().nerfb200_check_status() == 0
    got, gg = _step(models, rays, rgbs, S, K, use_disp, noise, white_back, randoms, grid)
    assert got["live_samples"] == (n * S, n * (S + K) if K else 0)
    for k in KEYS:
        if k in want:
            assert _same(got[k].detach(), want[k].detach()), k
    # the loss terms: the same squared errors summed in another order
    for k in ("loss", "mse_coarse", "mse_fine", "psnr"):
        a, b = float(got[k].detach()), float(want[k].detach())
        assert abs(a - b) <= 1e-6 * abs(b), (k, a, b)
    tot, worst = _grad_bars(gg, gw)
    print(f"\nS={S} K={K} {kind}: whole-gradient rel L2 {tot:.2e}, worst tensor {worst:.2e}")


@pytest.mark.parametrize("rng", ["tensor", "kernel"])
def test_fine_depths_are_the_plain_steps(rng):
    n, S, K = 500, 64, 128
    rays = _rays("blender", n, 9)
    rgbs = torch.rand(n, 3, device="cuda")
    randoms = _randoms(n, S, K, 2)
    models = _models()
    seed = 987654321 if rng == "kernel" else None
    with torch.no_grad():
        plain = _nb().render_rays(models, _emb(), rays, S, False, 1.0, 0.0, K, 32768, False,
                                  randoms=randoms if seed is None else {"seed": seed}, extras=True)
    from nerf_pl_b200.train_skip import render_rays_train_skip
    pr, ur = (randoms["perturb_rand"], randoms["u_rand"]) if seed is None else (None, None)
    got = render_rays_train_skip(models, rays, S, False, 1.0, 0.0, K, False, pr, None, ur, None, rgbs,
                                 _grid(1.0, FULL, N=3), rng_seed=seed, extras=True)
    assert _same(got["z_vals_fine"], plain["z_vals_fine"])
    assert _same(got["weights_coarse"], plain["weights_coarse"]) and _same(got["weights_fine"], plain["weights_fine"])


def _last_row_counted(out, copies):
    """out with the gradient of its last row counted 1 + copies times (the value unchanged): the planted defect of a
    backward that lets the padding rows of the last MLP tile, copies of the last row, into the weight gradients."""
    if not copies or not out.shape[0]:
        return out
    return torch.cat([out[:-1], out[-1:] * (1 + copies) - out[-1:].detach() * copies])


def _autograd_reference(models, rays, rgbs, got, S, K, noise_std, white_back, randoms, copies=(0, 0)):
    """The 24 or 48 gradients of the same step as an autograd composition: the evaluated rows through NeRF.forward
    (autograd_impl="fused"), float64 torch compositing with skipped samples at sigma = 0 (exact zeros for a network
    with no evaluated row).  `copies` plants _last_row_counted in the coarse / fine pass."""
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
        out = _last_row_counted(model(x), copies[ps]) if x.shape[0] else x.new_zeros(0, 4)
        sig = torch.zeros(n, Sp, dtype=torch.float64, device="cuda")
        rgb = torch.zeros(n, Sp, 3, dtype=torch.float64, device="cuda")
        noise = randoms.get("noise_" + name)
        s_ev = out[:, 3].double()
        if noise is not None and noise_std > 0:
            s_ev = s_ev + noise[ev].double() * noise_std
        sig = sig.index_put((ev,), s_ev)
        rgb = rgb.index_put((ev,), out[:, :3].double())
        c, _, _ = tr.composite_torch(z.double(), sig, rgb, rays[:, 3:6].double(), white_back)
        loss = loss + ((c - rgbs.double()) ** 2).mean()
    for m in models:
        m.zero_grad(set_to_none=True)
    if torch.is_tensor(loss) and loss.requires_grad:
        loss.backward()
    return {f"{i}.{k}": (p.grad if p.grad is not None else torch.zeros_like(p)).detach().cpu().numpy().astype(np.float64)
            for i, m in enumerate(models[:2 if K else 1]) for k, p in m.named_parameters()}


@pytest.mark.parametrize("S,K,noise,white_back", [(64, 128, 1.0, True), (32, 64, 0.0, False)])
def test_partial_grid(S, K, noise, white_back):
    n = 1000
    rays = _rays("blender", n, 7)
    rgbs = torch.rand(n, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    ranges = ((-2.0, 2.0), (2.0, -2.0), (-1.5, 2.5))
    grid = _grid(0.3, ranges, N=9, seed=3)
    randoms = _randoms(n, S, K, 8)
    models = _models()
    from nerf_pl_b200.train_skip import render_rays_train_skip
    for m in models:
        m.zero_grad(set_to_none=True)
    got = render_rays_train_skip(models, rays, S, False, 1.0, noise, K, white_back, randoms["perturb_rand"],
                                 randoms["noise_coarse"] if noise else None, randoms["u_rand"],
                                 randoms["noise_fine"] if noise else None, rgbs, grid, extras=True)
    got["loss"].backward()
    gg = {f"{i}.{k}": p.grad.detach().cpu().numpy().astype(np.float64)
          for i, m in enumerate(models) for k, p in m.named_parameters()}
    words, rn = grid.bits.cpu().numpy(), rays.cpu().numpy()
    # the evaluated sets are the float64 rule on the device's own perturbed / merged depths
    zc, zf = got["z_vals_coarse"].cpu().numpy(), got["z_vals_fine"].cpu().numpy()
    ev_c = sk.mask_bits(got["mask_coarse"].cpu().numpy(), S)
    ev_f = sk.mask_bits(got["mask_fine"].cpu().numpy(), S + K)
    assert np.array_equal(ev_c, sk.evaluated(rn, zc, words, grid.N, grid.ranges))
    assert np.array_equal(ev_f, sk.evaluated(rn, zf, words, grid.N, grid.ranges))
    assert 0.05 < ev_c.mean() < 0.95 and got["live_samples"] == (int(ev_c.sum()), int(ev_f.sum()))
    # skipped samples: no network value, weight exactly 0; compositing meets the float64 restatement
    for name, ev, Sp in (("coarse", ev_c, S), ("fine", ev_f, S + K)):
        smp = got["samples_" + name].cpu().numpy()
        w = got["weights_" + name].cpu().numpy()
        assert not smp[~ev].any() and not w[~ev].any()
        noise_t = randoms["noise_" + name].cpu().numpy() if noise else None
        ref = tr.forward(got["z_vals_" + name].cpu().numpy(), smp, ev, rn, noise_t, noise, white_back)
        tr.assert_close(ref, {k: got[k + "_" + name].detach().cpu().numpy() for k in ("rgb", "depth", "opacity")},
                        w, ref_weights=True)
    # per-row d sigma / d rgb_pre of the sparse compositing backward against float64 on the device's own depths,
    # network values, noise and results; each comparison rejects a backward with one planted defect
    for name, ev, Sp in (("coarse", ev_c, S), ("fine", ev_f, S + K)):
        smp = got["samples_" + name].cpu().numpy()
        rows = int(ev.sum())
        ds = got["dsigma_" + name][:rows].cpu().numpy()
        dp = got["dprergb_" + name][:rows].cpu().numpy()
        noise_t = randoms["noise_" + name].cpu().numpy() if noise else None

        def ref_bwd(ev_=ev, noise_std=noise, wb=white_back):
            return tr.backward(got["z_vals_" + name].cpu().numpy(), smp[..., 3], smp[..., :3], ev_, rn[:, 3:6],
                               noise_t, noise_std, wb, got["rgb_" + name].detach().cpu().numpy(), rgbs.cpu().numpy(), n)

        ds_ref, dp_ref = ref_bwd()
        errs = tr.backward_errors(ds, dp, ev, ds_ref, dp_ref)
        print(f"\n{name}: per-row d sigma error {errs[0]:.2e}, d rgb_pre {errs[1]:.2e} (bar {tr.BWD_BAR})")
        assert max(errs) <= tr.BWD_BAR, (name, errs)
        planted = {"white_back ignored": dict(wb=not white_back)}
        if noise:       # without noise a skipped sample composited at sigma 0 is indistinguishable from a skipped one
            planted.update({"noise dropped": dict(noise_std=0.0), "skipped samples composited": dict(ev_=np.ones_like(ev))})
        for what, kw in planted.items():
            bds, bdp = ref_bwd(**kw)
            bad = tr.backward_errors(bds[ev].astype(np.float32), bdp[ev].astype(np.float32), ev, ds_ref, dp_ref)
            assert max(bad) > tr.BWD_BAR, (name, what, bad)
        if noise:       # noise added to skipped samples is rejected by the forward check
            bad_noise = tr.forward(got["z_vals_" + name].cpu().numpy(), smp, np.ones_like(ev), rn, noise_t, noise,
                                   white_back)
            with pytest.raises(AssertionError):
                tr.assert_close(bad_noise, {k: got[k + "_" + name].detach().cpu().numpy()
                                            for k in ("rgb", "depth", "opacity")},
                                got["weights_" + name].cpu().numpy(), ref_weights=True)
    ref = _autograd_reference(models, rays, rgbs, got, S, K, noise, white_back, randoms)
    tot, worst = _grad_bars(gg, ref)
    print(f"\npartial grid S={S} K={K}: whole-gradient rel L2 {tot:.2e}, worst tensor {worst:.2e}")


def test_vacuum_rays():
    """With an empty grid every sample is skipped: the vacuum value and no gradient."""
    n, S, K = 256, 64, 64
    rays = _rays("blender", n, 11)
    rgbs = torch.rand(n, 3, device="cuda")
    models = _models()
    from nerf_pl_b200.train_skip import render_rays_train_skip
    empty = _grid(0.0, ((-1.5, 1.5),) * 3, N=9)
    for white_back in (False, True):
        got = render_rays_train_skip(models, rays, S, False, 0.0, 0.0, K, white_back, None, None, None, None, rgbs,
                                     empty, extras=True)
        assert got["live_samples"] == (0, 0)
        assert not got["opacity_fine"].any() and not got["depth_fine"].any()
        assert torch.all(got["rgb_fine"] == (1.0 if white_back else 0.0))
        for m in models:
            m.zero_grad(set_to_none=True)
        got["loss"].backward()
        assert all(not p.grad.any() for m in models for p in m.parameters())


COLS = ("ox", "oy", "oz", "dx", "dy", "dz", "near", "far")


def _degenerate_catalogue():
    """test_gpu_degenerate_rays.py's ray families: (name, ray (8,), finite depths and directions)."""
    F32 = np.float32
    base = orc.make_rays(1, 11)[0]
    out = []
    for c in range(8):
        for v in (np.nan, np.inf, -np.inf):
            r = base.copy()
            r[c] = v
            out.append((f"{COLS[c]}={v}", r, False))
    deg = {
        "d=0": (lambda r: r.__setitem__(slice(3, 6), 0.0), True),
        "|d|=1e-30": (lambda r: r.__setitem__(slice(3, 6), r[3:6] * F32(1e-30)), True),
        "d_subnormal": (lambda r: r.__setitem__(slice(3, 6), r[3:6] * F32(1e-39)), True),
        "|d|=1e20": (lambda r: r.__setitem__(slice(3, 6), r[3:6] * F32(1e20)), False),
        "ndc": (lambda r: r.__setitem__(slice(0, 8), orc.make_rays(1, 12, "ndc")[0]), True),
        "near<0": (lambda r: r.__setitem__(6, -1.5), True),
        "far=1e10": (lambda r: r.__setitem__(7, 1e10), False),
        "far=3e38": (lambda r: r.__setitem__(7, 3e38), False),          # fp32 mid-points overflow: delta |d| not finite
        "far<=near": (lambda r: r.__setitem__(7, r[6]), True),
    }
    for name, (f, finite) in deg.items():
        r = base.copy()
        f(r)
        out.append((name, r.astype(F32), finite))
    return out


@pytest.mark.parametrize("perturb,noise", [(0.0, 0.0), (1.0, 1.0)])
def test_degenerate_rays(perturb, noise):
    """Every family of the degenerate-ray catalogue mixed into ordinary rays on a partial grid: the evaluated sets are
    the float64 rule on the device's own depths (a ray with a non-finite value, far <= near, or a pass with a
    non-finite delta |d| is evaluated at every sample), and the backward runs on them: a batch with a non-finite
    family reports status 103, a batch of the families with finite depths returns finite gradients."""
    nb = _nb()
    S, K = 64, 64
    cat = _degenerate_catalogue()
    grid = _grid(0.3, ((-1.5, 1.5),) * 3, N=17, seed=2)
    from nerf_pl_b200.train_skip import render_rays_train_skip
    for subset in ("all", "finite"):
        fams = [c for c in cat if subset == "all" or c[2]]
        n = 700
        rn = orc.make_rays(n, 21)
        where = {}
        for j, (name, r, _) in enumerate(fams):
            for p in (10 + 17 * j, 11 + 17 * j):
                rn[p] = r
                where[p] = name
        rays = torch.from_numpy(rn).cuda()
        rgbs = torch.rand(n, 3, device="cuda")
        rnd = _randoms(n, S, K, 4)
        models = _models()
        for m in models:
            m.zero_grad(set_to_none=True)
        got = render_rays_train_skip(models, rays, S, False, perturb, noise, K, False,
                                     rnd["perturb_rand"] if perturb else None, rnd["noise_coarse"] if noise else None,
                                     rnd["u_rand"] if perturb else None, rnd["noise_fine"] if noise else None, rgbs,
                                     grid, extras=True)
        words = grid.bits.cpu().numpy()
        for name, Sp in (("coarse", S), ("fine", S + K)):
            ev = sk.mask_bits(got["mask_" + name].cpu().numpy(), Sp)
            z = got["z_vals_" + name].cpu().numpy()
            want = sk.evaluated(rn, z, words, grid.N, grid.ranges)
            assert np.array_equal(ev, want), (name, [where.get(int(r)) for r in np.nonzero((ev != want).any(1))[0]])
            plain = sk.plain_pass(rn, z)
            assert ev[plain].all() and plain[[p for p, nm in where.items() if "=" in nm and nm[:2] in
                                              ("ox", "oy", "oz", "dx", "dy", "dz", "ne", "fa") and
                                              not nm.startswith(("far=1", "far=3"))]].all(), name
        torch.cuda.synchronize()
        assert nb._lib.load().nerfb200_check_status() == 0          # the forward reports nothing
        got["loss"].backward()
        torch.cuda.synchronize()
        st = nb._lib.load().nerfb200_check_status()
        if subset == "all":
            assert st != 0                                            # status 103: a non-finite per-sample gradient
        else:
            assert st == 0
            assert all(torch.isfinite(p.grad).all() for m in models for p in m.parameters())


def test_batch_order():
    n, S, K = 800, 64, 64
    rays = _rays("blender", n, 12)
    rgbs = torch.rand(n, 3, device="cuda")
    grid = _grid(0.3, ((-1.5, 1.5),) * 3, N=17, seed=1)
    randoms = _randoms(n, S, K, 3)
    perm = torch.randperm(n, device="cuda")
    models = _models()
    a, ga = _step(models, rays, rgbs, S, K, False, 1.0, False, randoms, grid)
    b, gb = _step(models, rays[perm], rgbs[perm], S, K, False, 1.0, False,
                  {k: v[perm].contiguous() for k, v in randoms.items()}, grid)
    for k in KEYS[:6]:
        assert _same(b[k].detach(), a[k].detach()[perm]), k
    assert a["live_samples"] == b["live_samples"]
    for k in ga:      # the wgrad sums the same rows in another order
        assert np.linalg.norm(gb[k] - ga[k]) <= 1e-4 * np.linalg.norm(ga[k]) + 1e-12, k


def test_changing_row_counts_allocate_nothing():
    """Steps whose evaluated sample counts change share one workspace, sized once: after the first steps, no step
    allocates more than its own small result and gradient tensors, and the memory in use does not grow."""
    n, S, K = 1024, 64, 64
    rays = _rays("blender", n, 13)
    rgbs = torch.rand(n, 3, device="cuda")
    models = _models()
    grids = [_grid(f, ((-1.5, 1.5),) * 3, N=17, seed=i) for i, f in enumerate((0.05, 0.3, 0.7, 1.0))]
    counts = set()
    for step in range(200):
        for m in models:
            m.zero_grad(set_to_none=False)
        res = _nb().render_rays_loss(models, _emb(), rays, rgbs, S, False, 1.0, 1.0, K, 32768, False,
                                     randoms="kernel", occupancy=grids[step % 4])
        res["loss"].backward()
        counts.add(res["live_samples"])
        del res
        if step == 3:                 # the next four steps are one cycle of the grids: their peak is the steady one
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
        if step == 7:
            torch.cuda.synchronize()
            pool = _nb().train_skip.SkipTrainWorkspace._pool[(0, n, S, K)]
            buf = pool[0].buf.data_ptr()
            base, peak = torch.cuda.memory_allocated(), torch.cuda.max_memory_allocated()
    torch.cuda.synchronize()
    assert len(counts) > 4
    assert len(pool) == 1 and pool[0].buf.data_ptr() == buf
    assert torch.cuda.memory_allocated() == base
    assert torch.cuda.max_memory_allocated() == peak


def test_argument_errors():
    nb = _nb()
    models = _models()
    rays = _rays("blender", 64, 1)
    rgbs = torch.rand(64, 3, device="cuda")
    grid = _grid(1.0, FULL, N=3)
    with pytest.raises(ValueError, match="N_samples"):
        nb.render_rays_loss(models, _emb(), rays, rgbs, 48, N_importance=64, occupancy=grid)
    with pytest.raises(ValueError, match="OccupancyGrid"):
        nb.render_rays_loss(models, _emb(), rays, rgbs, 64, N_importance=64, occupancy=object())
    with pytest.raises(ValueError, match="randoms must be"):
        nb.render_rays_loss(models, _emb(), rays, rgbs, 64, N_importance=64, randoms="philox", occupancy=grid)
    cpu_grid = object.__new__(nb.OccupancyGrid)
    cpu_grid.bits = torch.zeros(1, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="occupancy grid is on"):
        nb.render_rays_loss(models, _emb(), rays, rgbs, 64, N_importance=64, occupancy=cpu_grid)


_CTAS_CASE = """
import sys, numpy as np, torch
sys.path.insert(0, {root!r})
from tests import test_gpu_train_skip as t
np.savez({out!r}, **t._ctas_case())
"""


def _ctas_case():
    """Results, per-row gradients and the 48 gradients of one partial-grid step with noise and in-kernel randoms."""
    n, S, K = 900, 64, 128
    rays = _rays("blender", n, 17)
    rgbs = torch.rand(n, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    noise = _randoms(n, S, K, 6)
    models = _models()
    from nerf_pl_b200.train_skip import render_rays_train_skip
    got = render_rays_train_skip(models, rays, S, False, 1.0, 1.0, K, True, None, noise["noise_coarse"], None,
                                 noise["noise_fine"], rgbs, _grid(0.3, ((-1.5, 1.5),) * 3, N=17, seed=5),
                                 rng_seed=4242, extras=True)
    got["loss"].backward()
    out = {k: np.atleast_1d(v.detach().cpu().numpy()) for k, v in got.items() if torch.is_tensor(v)}
    out.update({f"grad{i}.{k}": p.grad.cpu().numpy() for i, m in enumerate(models) for k, p in m.named_parameters()})
    return out


def test_results_do_not_depend_on_the_cta_count(tmp_path):
    """NERFB200_MAX_CTAS=1 (read once per process, hence the subprocess) caps every grid-stride launch at one block:
    results, per-row gradients and the 48 gradients are bit for bit those of the full grid."""
    import os
    import subprocess
    import sys
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
