"""Training a direct NeRF.forward call on the sm_90a kernels (``model.autograd_impl = "fused"``,
``nerf_pl_b200.nerf_forward_train``; pytest -m gpu).

The forward is one save-mode launch of the MLP kernel; the backward is the render path's backward kernels seeded
from the upstream (B, 4) gradient.  Stage by stage this file holds them, on the device's own stored values, to the
bars of tests/train_tape.py (the workspace keeps the render path's per-pass buffer order; one pass, one sample per
row, followed by the fp16 direction rows).  In this path the direction slice of dir_encoding is an fp16
tensor-core operand (fp16 weights, fp16 inputs) where the render path adds a per-ray fp32 direction term, so the
direction-layer and direction-gradient references are the MLP-mode variants written here.
"""
import numpy as np
import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib
from nerf_pl_b200.training import NerfTrainWorkspace
from oracle import nerf_oracle as orc
from tests import cases
from tests import train_tape as tt

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _model(w, dev, impl="fused"):
    m = nb.NeRF()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
    m = m.to(dev)
    m.autograd_impl = impl
    return m


def _x(n, seed):
    """(n, 90) embedded xyz + embedded direction, as render_rays' callers build them."""
    rs = np.random.RandomState(seed)
    xyz = rs.uniform(-1.5, 1.5, (n, 3)).astype(np.float32)
    d = rs.randn(n, 3).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return np.concatenate([orc.embed(xyz, 10), orc.embed(d, 4)], 1).astype(np.float32)


def _layout(n):
    """Offsets of the NeRF.forward workspace (csrc/capi.cu make_mlp_train_layout): the render path's per-pass buffers
    for one pass of n one-sample rays, then the tiled (n_pad, 64) direction rows."""
    P = tt.layout(n, 1, 0)[0]
    P["xdir"] = P["dpre"] + (P["n_pad"] * 512 * 8 + 1023) // 1024 * 1024
    return P


def _xdir(raw, P):
    return tt.untile(raw[P["xdir"]:P["xdir"] + P["n_pad"] * 128], P["n_pad"], 64)[:P["n"]]


def _workspace(out):
    return out.grad_fn.lease.ws


# ------------------------------------------------------------------------------------------------ 1. forward
@pytest.mark.parametrize("B", [1, 127, 128, 129, 4099, 196608])
def test_forward_equals_inference_kernel(B, dev):
    m = _model(cases.weights()[0], dev)
    x = torch.from_numpy(_x(B, B)).to(dev)
    out = m(x)
    assert out.requires_grad and out.shape == (B, 4)
    ref = nb.nerf_forward_fused(m, x)
    assert torch.equal(out.detach(), ref)


# ------------------------------------------------------------------------------------------------ 2. stages
STAGE_CASES = {
    "random_both": dict(n=3000, weights="random", g="both"),
    "random_rgb_only": dict(n=1000, weights="random", g="rgb"),
    "random_sigma_only": dict(n=1000, weights="random", g="sigma"),
    "trained_both": dict(n=3000, weights="trained", g="both"),
    # samples 0..255 carry ~1e-4 upstream gradients, the rest ~0.3; 157 tiles, more than the probe visits
    "skewed_20000": dict(n=20000, weights="random", g="skewed"),
}


def _upstream(n, kind, seed):
    rs = np.random.RandomState(seed)
    g = (rs.randn(n, 4) * 0.3).astype(np.float32)
    if kind == "rgb":
        g[:, 3] = 0
    elif kind == "sigma":
        g[:, :3] = 0
    elif kind == "skewed":
        g[:256] *= 1e-4 / 0.3
    return g


@pytest.mark.parametrize("name", list(STAGE_CASES))
def test_backward_stages(name, dev):
    c = STAGE_CASES[name]
    n, seed = c["n"], 500 + list(STAGE_CASES).index(name)
    w = (cases.trained_weights() if c["weights"] == "trained" else cases.weights())[0]
    m = _model(w, dev)
    x = torch.from_numpy(_x(n, seed)).to(dev)
    g = _upstream(n, c["g"], seed)
    out = m(x)
    ws = _workspace(out)
    out.backward(torch.from_numpy(g).to(dev))
    torch.cuda.synchronize()
    assert _lib.load().nerfb200_check_status() == 0
    raw = ws.buf.cpu().numpy()
    grads = {k: p.grad.cpu().numpy() for k, p in m.named_parameters()}
    P = _layout(n)
    full = tt.WorkspaceTape(raw, P)
    nt = P["n_pad"] // 128
    sub = full if nt <= 24 else tt.WorkspaceTape(raw, P, np.unique([0, 1, nt // 2, nt - 1, *range(3, nt, nt // 6)]))
    bad = []
    # what the forward stored: the inference output, the fp16 rows of x it consumed
    o = out.detach().cpu().numpy()
    if not (np.array_equal(full.sigma(), o[:, 3]) and np.array_equal(full.rgb(), o[:, :3])):
        bad.append("stored sigma / rgb differ from the returned output")
    xs = x.cpu().numpy()
    xdir = _xdir(raw, P)
    if not (np.array_equal(full.enc()[:, :63], xs[:, :63].astype(np.float16)) and not full.enc()[:, 63].any()):
        bad.append("stored encoded rows are not the fp16 rows of x[:, :63]")
    if not (np.array_equal(xdir[:, :27], xs[:, 63:].astype(np.float16)) and not xdir[:, 27:].any()):
        bad.append("stored direction rows are not the fp16 rows of x[:, 63:]")
    # seed: d sigma = g_sigma, d rgb_pre = g_rgb rgb (1 - rgb)
    rgb = full.rgb().astype(np.float64)
    dp_ref = g[:, :3] * rgb * (1 - rgb)
    seed_err = float(np.abs(full.dprergb() - dp_ref).max() / max(np.abs(dp_ref).max(), 1e-30))
    if not np.array_equal(full.dsigma(), g[:, 3]) or not seed_err < 1e-6:
        bad.append(f"seed: d sigma exact {np.array_equal(full.dsigma(), g[:, 3])}, d rgb_pre {seed_err:.3g}")
    # MLP mode: the direction slice is an fp16 x fp16 tensor-core term
    net = tt.Net(w)
    net.Wdir = tt.r16(net.Wdir)
    fwd = tt.check_forward(sub, net, xdir[:, :27].astype(np.float64))
    masks = tt.check_masks(sub)
    chain = tt.check_chain(sub, net)
    ref = tt.reference_grads(full, net, chain["scales"], xdir[:, :27].astype(np.float64))
    dd = full.dd().astype(np.float64) / chain["scales"][0]
    ref["dir_encoding.0.weight"][:, 256:] = dd.T @ xdir[:, :27].astype(np.float64)
    gr = tt.check_grads(grads, ref)
    bad += tt.failures(fwd, masks, chain, None, gr)
    print(f"\n[{name}] forward " + " ".join(f"{k} {v:.3g}" for k, v in fwd.items()))
    print(f"seed {seed_err:.3g}; masks {masks}; scales log2 {[int(np.log2(s)) for s in chain['scales']]}")
    print("chain steps " + " ".join(f"{chain[f'step{v}']:.3g}" for v in range(9)) +
          " | acc " + " ".join(f"{chain[f'acc{v}']:.3g}" for v in range(1, 9)))
    wr = max(gr.items(), key=lambda kv: kv[1][0])
    wm = max(gr.items(), key=lambda kv: kv[1][1])
    print(f"grads worst rel {wr[1][0]:.3g} ({wr[0]}), worst max {wm[1][1]:.3g} ({wm[0]})")
    assert not bad, "\n".join(bad)


# ------------------------------------------------------------------------------------------------ 3. vs autograd
def _grad_bars(got, ref, whole=True):
    """DESIGN section 2's end-to-end bars: per tensor relative L2 < 8e-2, cosine > 0.997; whole gradient < 5e-3."""
    num = den = 0.0
    for k, r in ref.items():
        a, b = np.asarray(got[k], np.float64), np.asarray(r, np.float64)
        num += float(((a - b) ** 2).sum())
        den += float((b ** 2).sum())
        rel = np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30)
        cos = float((a * b).sum() / max(np.linalg.norm(a) * np.linalg.norm(b), 1e-30))
        assert rel < 8e-2 and cos > 0.997, f"{k}: rel {rel:.3e} cos {cos:.5f}"
    tot = (num / den) ** 0.5
    assert tot < 5e-3 or not whole, tot
    return tot


@pytest.mark.parametrize("weights", ["random", "trained"])
@pytest.mark.parametrize("loss", ["mse", "random_sign"])
def test_gradients_match_float64_autograd(weights, loss, dev):
    """Against torch autograd in float64 on the same inputs.  'mse': the upstream gradient of mean((out - t)^2) for
    a fixed target t, the regime of the render path's bars (per-sample terms add up coherently).  'random_sign':
    unit-variance random upstream gradients; the true parameter gradient is then a sum that cancels to ~1/sqrt(B)
    of its terms while the fp16 rounding / ReLU-flip errors of the terms do not cancel with it, so only the
    per-tensor bars apply (measured whole-gradient error ~2e-2 on an H100)."""
    w = (cases.trained_weights() if weights == "trained" else cases.weights())[1]
    n = 8192
    x = torch.from_numpy(_x(n, 77)).to(dev)
    m = _model(w, dev)
    if loss == "mse":
        with torch.no_grad():
            o = nb.nerf_forward_fused(m, x)
        g = (o - torch.tensor([0.8, 0.8, 0.8, 1.0], device=dev)) * (2.0 / o.numel())
    else:
        g = torch.from_numpy(_upstream(n, "both", 78)).to(dev)
    m(x).backward(g)
    m64 = _model(w, dev, "torch").double()
    nb.nerf_forward_torch(m64, x.double()).backward(g.double())
    got = {k: p.grad.cpu().numpy() for k, p in m.named_parameters()}
    ref = {k: p.grad.cpu().numpy() for k, p in m64.named_parameters()}
    print(f"\n{weights} {loss}: whole-gradient relative L2 {_grad_bars(got, ref, whole=loss == 'mse'):.3e}")


# ------------------------------------------------------------------------------------------------ 4. own renderer
def _embed(x, n_freqs):
    parts = [x]
    for k in range(n_freqs):
        parts += [torch.sin((2.0 ** k) * x), torch.cos((2.0 ** k) * x)]
    return torch.cat(parts, -1)


def _render_pass(model, rays, z, noise, noise_std, white_back):
    """models/rendering.py's inference() (:91-172) written with torch ops; the MLP call is model(x)."""
    n, S = z.shape
    o, d = rays[:, 0:3], rays[:, 3:6]
    xyz = (o[:, None, :] + d[:, None, :] * z[:, :, None]).reshape(-1, 3)
    x = torch.cat((_embed(xyz, 10), _embed(d, 4).repeat_interleave(S, dim=0)), -1)
    raw = model(x).view(n, S, 4)
    sig = raw[..., 3]
    delta = torch.cat((z[:, 1:] - z[:, :-1], torch.full_like(z[:, :1], 1e10)), -1) * d.norm(dim=-1, keepdim=True)
    if noise is not None:
        sig = sig + noise * noise_std
    alpha = 1 - torch.exp(-delta * torch.relu(sig))
    w = alpha * torch.cumprod(torch.cat((torch.ones_like(alpha[:, :1]), 1 - alpha + 1e-10), -1), -1)[:, :-1]
    rgb = (w[..., None] * raw[..., :3]).sum(-2)
    if white_back:
        rgb = rgb + 1 - w.sum(1)[:, None]
    return rgb


@pytest.mark.parametrize("name", list(cases.GRAD_CASES))
def test_own_renderer_matches_reference_golden(name, dev):
    """A renderer written here with torch ops whose MLP calls are model(x) on the fused path reproduces the
    reference's loss.backward() (tests/golden/grad_*.npz) within the render path's golden bars."""
    from oracle import nerf_oracle_grad as og
    n, kind, rseed, K, perturb, noise, wb = cases.GRAD_CASES[name]
    rays, target, randoms, ref_loss, ref_out, ref_grads = cases.load_grad_case(name)
    models = [_model(w, dev) for w in cases.weights()]
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    r, t = torch.from_numpy(rays).to(dev), torch.from_numpy(target).to(dev)
    rnd = {k: torch.from_numpy(v).to(dev) for k, v in randoms.items()}
    with torch.no_grad():      # the fine depths carry no gradient (models/rendering.py:225-227 .detach())
        z_fine = nb.render_rays(models, emb, r, 64, False, perturb, noise, K, 32768, wb, randoms=rnd,
                                extras=True)["z_vals_fine"]
    near, far = r[:, 6:7], r[:, 7:8]
    z = near * (1 - torch.linspace(0, 1, 64, device=dev)) + far * torch.linspace(0, 1, 64, device=dev)
    mid = 0.5 * (z[:, :-1] + z[:, 1:])
    upper, lower = torch.cat((mid, z[:, -1:]), -1), torch.cat((z[:, :1], mid), -1)
    z = lower + (upper - lower) * (perturb * rnd["perturb_rand"])
    nc = rnd.get("noise_coarse") if noise > 0 else None
    nf = rnd.get("noise_fine") if noise > 0 else None
    rgb_c = _render_pass(models[0], r, z, nc, noise, wb)
    rgb_f = _render_pass(models[1], r, z_fine, nf, noise, wb)
    loss = ((rgb_c - t) ** 2).mean() + ((rgb_f - t) ** 2).mean()
    loss.backward()
    torch.cuda.synchronize()
    assert abs(float(loss.detach()) - ref_loss) < 1e-3 * ref_loss, (float(loss.detach()), ref_loss)
    grads = {f"{tag}.{k}": p.grad.cpu().numpy() for tag, m in zip(("coarse", "fine"), models)
             for k, p in m.named_parameters()}
    rows, (rel, cos) = og.grad_compare(grads, ref_grads)
    worst = max(rows.items(), key=lambda kv: kv[1][0])
    print(f"\n{name}: global rel {rel:.3e} cos {cos:.6f}; worst {worst[0]} rel {worst[1][0]:.3e}")
    assert rel < 5e-3 and cos > 0.9999, (rel, cos)
    for k, (rr, cc) in rows.items():
        assert np.isfinite(grads[k]).all(), k
        assert rr < 8e-2 and cc > 0.997, f"{k}: rel {rr:.3e} cos {cc:.5f}"


# ------------------------------------------------------------------------------------------------ 5. accumulation
def _grads(m):
    return [p.grad.clone() for p in m.parameters()]


def test_accumulation_is_the_sum_of_single_backwards(dev):
    ws = cases.weights()
    x = [torch.from_numpy(_x(n, 90 + n)).to(dev) for n in (3000, 1700)]
    g = [torch.from_numpy(_upstream(xi.shape[0], "both", 95 + i)).to(dev) for i, xi in enumerate(x)]
    single = []
    for i in range(2):
        m = _model(ws[i], dev)
        m(x[i]).backward(g[i])
        single.append(_grads(m))
    # two different models, one backward
    a, b = _model(ws[0], dev), _model(ws[1], dev)
    ((a(x[0]) * g[0]).sum() + (b(x[1]) * g[1]).sum()).backward()
    for got, want in ((_grads(a), single[0]), (_grads(b), single[1])):
        assert all(torch.equal(p, q) for p, q in zip(got, want))
    # one model called twice, one backward
    one = []
    for i in range(2):
        m = _model(ws[0], dev)
        m(x[i]).backward(g[i])
        one.append(_grads(m))
    m = _model(ws[0], dev)
    ((m(x[0]) * g[0]).sum() + (m(x[1]) * g[1]).sum()).backward()
    for i, p in enumerate(m.parameters()):
        assert torch.equal(p.grad, one[0][i] + one[1][i]), i
    # repeating a step gives bit-identical gradients
    m2 = _model(ws[0], dev)
    ((m2(x[0]) * g[0]).sum() + (m2(x[1]) * g[1]).sum()).backward()
    assert all(torch.equal(p.grad, q.grad) for p, q in zip(m.parameters(), m2.parameters()))
    torch.cuda.synchronize()
    assert _lib.load().nerfb200_check_status() == 0


# ------------------------------------------------------------------------------------------------ 6. overflow
def _probed_tiles(span, probe_tiles):
    """The tiles the chain kernel's probe visits (csrc/capi.cu launch_chain: visit j -> j * stride mod span)."""
    s = span // probe_tiles if span > probe_tiles else 1
    while span > 1 and np.gcd(s, span) != 1:
        s += 1
    return {j * s % span for j in range(min(probe_tiles, span))}


def test_overflow_in_unprobed_tiles_is_reported(dev):
    """Upstream gradients 1e5 times larger than elsewhere, only in tiles the probe does not visit: the per-level
    scales cannot hold them; the backward reports status 102 (RuntimeError on the next call), not clamped gradients."""
    sm = torch.cuda.get_device_properties(dev).multi_processor_count
    span = 3 * sm + 1
    n = 128 * span
    probed = _probed_tiles(span, min(span, sm))
    hot = [t for t in range(span) if t not in probed][:3]
    assert len(hot) == 3
    g = _upstream(n, "both", 61) * 1e-5
    for t in hot:
        g[t * 128:(t + 1) * 128] *= 1e5
    m = _model(cases.weights()[0], dev)
    x = torch.from_numpy(_x(n, 60)).to(dev)
    lib = _lib.load()
    assert lib.nerfb200_check_status() == 0
    out = m(x)
    ws = _workspace(out)
    out.backward(torch.from_numpy(g).to(dev))
    torch.cuda.synchronize()
    sat = tt.WorkspaceTape(ws.buf.cpu().numpy(), _layout(n)).saturated()
    print(f"\nhot tiles {hot}: saturated elements {sat}")
    assert sat > 0
    with pytest.raises(RuntimeError, match="102"):
        m(x)
    assert lib.nerfb200_check_status() == 0


# ------------------------------------------------------------------------------------------------ 7. lifetime
def test_workspace_pool_stays_bounded(dev):
    NerfTrainWorkspace.clear()
    m = _model(cases.weights()[0], dev)
    x = torch.from_numpy(_x(5000, 3)).to(dev)
    for _ in range(100):             # outputs used under grad mode without a backward
        out = m(x)
        float(out[:, 3].mean())
        del out
    assert NerfTrainWorkspace.pool_size(dev) == 1
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(dev)
    lib = _lib.load()
    for i in range(100):             # a point loop whose batch size varies
        B = 5000 - 37 * i
        m(x[:B]).sum().backward()
        assert NerfTrainWorkspace.pool_size(dev) <= 1
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated(dev) <= base + lib.nerfb200_nerf_train_workspace_bytes(5000)
    outs = [m(x[:B]) for B in (5000, 4000, 5000)]       # pending backwards each hold their own workspace
    assert NerfTrainWorkspace.pool_size(dev) == 3
    del outs
    m(x[:100]).sum().backward()
    assert NerfTrainWorkspace.pool_size(dev) == 1


# ------------------------------------------------------------------------------------------------ 8. errors
def test_errors(dev):
    m = _model(cases.weights()[0], dev)
    x = torch.from_numpy(_x(300, 4)).to(dev)
    with pytest.raises(ValueError, match="sigma_only"):
        m(x[:, :63], sigma_only=True)
    with pytest.raises(ValueError, match="gradient with respect to x"):
        m(x.clone().requires_grad_(True))
    with pytest.raises(ValueError, match=r"\(B, 90\)"):
        m(x[:, :80])
    odd = nb.NeRF(D=4, skips=(2,)).to(dev)
    odd.autograd_impl = "fused"
    with pytest.raises(ValueError, match="default"):
        odd(x)
    m.autograd_impl = "tensorrt"
    with pytest.raises(ValueError, match="autograd_impl"):
        m(x)
    m.autograd_impl = "fused"
    with pytest.raises(RuntimeError):
        m(x.cpu())
    out = m(x)
    out.sum().backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="already run"):
        out.sum().backward()
    # the default path is untouched
    m.autograd_impl = "torch"
    assert m(x).grad_fn.name() != "FusedNerfFunctionBackward"
    with torch.no_grad():
        assert torch.equal(m(x), nb.nerf_forward_fused(m, x))
