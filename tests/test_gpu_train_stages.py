"""The training step's backward, stage by stage, on the device's own stored values (pytest -m gpu).

One fused training step per case; then every stage is compared in float64 with the values the device stored as
THAT stage's inputs (tests/train_tape.py reads them from the training workspace).  Each comparison isolates one
kernel, so its bar is set by fp32 / fp16 rounding instead of by the ReLU-mask flips that make the end-to-end
gradient tests of test_gpu_parity.py loose.  The last comparison covers every element of all 24 (48) .grad
tensors against float64 contractions of exactly the operands the wgrad / reduction / unfold kernels read: a
dropped chunk, a wrong piece range, a wrong partial slot, a wrong un-scale level or a missing direction slice
shows up there as an error far above fp32 summation error.

The bars and the values measured on an H100 stand in tests/train_tape.py BARS.
"""
import numpy as np
import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib
from oracle import nerf_oracle as orc
from tests import cases, philox
from tests import train_tape as tt

pytestmark = pytest.mark.gpu

DEFAULTS = dict(S=64, K=64, use_disp=False, perturb=1.0, noise_std=0.0, white_back=True, rng="tensors",
                weights="random", loss="fused", golden=None)
# name: one training step's configuration (ray seed = the case's index + 70)
CASES = {
    "anchor_64": dict(n=64, golden="grad_blender_noise0"),
    "one_ray_coarse_only": dict(n=1, K=0, loss="mse"),          # half the only tile is padding; 63 empty dir slices
    "disp_33": dict(n=33, S=32, K=32, use_disp=True, white_back=False),
    "sf192_75": dict(n=75, S=128, K=64),                         # S_f = 192: 6 samples per lane in composite_bwd
    "k160_50": dict(n=50, S=32, K=160),
    "noise_48": dict(n=48, K=128, noise_std=1.0),
    "all_outputs_130": dict(n=130, loss="all6"),                 # upstream g_rgb / g_depth / g_opac
    "bench_1024_seed": dict(n=1024, rng="seed"),                 # in-kernel Philox uniforms; probe sees a subset
    "trained_1024": dict(n=1024, weights="trained"),
    # rays 0..255 carry residuals ~1e-4 (their target is the rendered colour), the rest ~0.3: the probe of the
    # chain kernel picks the per-layer scales from one tile per SM spread over each pass, so it must not take
    # them from the first tiles alone
    "skewed_1024": dict(n=1024, loss="skewed"),
}
MAX_TILES = 24          # per-layer tape and chain checks: all tiles up to this many, else a fixed subset


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
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        out.append(m.to(dev))
    return out


def _to_dev(d, dev):
    return {k: torch.from_numpy(np.ascontiguousarray(v, np.float32)).to(dev) for k, v in d.items()}


def _tiles(n_pad, seed):
    """All tiles of a small pass; else first, second, middle, last and six seeded random ones (the chain kernel's
    probe visits ceil(SMs / 2) tiles spread over each pass, so most of these are tiles it did not see)."""
    nt = n_pad // 128
    if nt <= MAX_TILES:
        return None
    rs = np.random.RandomState(seed)
    return np.unique(np.concatenate([[0, 1, nt // 2, nt - 1], rs.choice(nt, 6, replace=False)]))


def run_step(name, dev, emb):
    return run_train(dict(DEFAULTS, **CASES[name]), 70 + list(CASES).index(name), dev, emb)


def run_train(c, seed, dev, emb):
    """One training step of configuration `c` (DEFAULTS' keys) on rays and random numbers drawn from `seed`.
    Returns the inputs, the workspace bytes, the gradients and the upstream gradient seeds of each pass."""
    n, S, K = c["n"], c["S"], c["K"]
    ws_np = cases.trained_weights() if c["weights"] == "trained" else cases.weights()
    if c["golden"]:
        rays, target, randoms, *_ = cases.load_grad_case(c["golden"])
    else:
        rays = orc.make_rays(n, seed)
        rs = np.random.RandomState(seed)
        target = rs.uniform(0, 1, (n, 3)).astype(np.float32)
        randoms = {"perturb_rand": rs.rand(n, S).astype(np.float32)}
        if K:
            randoms["u_rand"] = rs.rand(n, K).astype(np.float32)
        if c["noise_std"] > 0:
            randoms["noise_coarse"] = rs.randn(n, S).astype(np.float32)
            if K:
                randoms["noise_fine"] = rs.randn(n, S + K).astype(np.float32)
    if c["rng"] == "seed":             # the uniforms from the kernel's Philox stream, the noise still from tensors
        noise = {k: v for k, v in randoms.items() if k.startswith("noise")}
        rnd = dict(_to_dev(noise, dev), seed=1000 + seed)
        randoms = dict(philox.randoms(1000 + seed, n, S, K), **noise)
    else:
        rnd = _to_dev(randoms, dev)
    models = _models(ws_np, dev)
    r, t = torch.from_numpy(rays).to(dev), torch.from_numpy(target).to(dev)
    args = (S, c["use_disp"], c["perturb"], c["noise_std"], K, 32768, c["white_back"])
    with torch.no_grad():
        inf = nb.render_rays(models, emb, r, *args, randoms=rnd, extras=True)
    passes = ("coarse", "fine") if K else ("coarse",)
    if c["loss"] == "fused":
        out = nb.render_rays_loss(models, emb, r, t, *args[:5], 32768, c["white_back"], randoms=rnd)
        loss = out["loss"]
    else:
        out = nb.render_rays(models, emb, r, *args, randoms=rnd)
        for k in out:
            out[k].retain_grad()
        if c["loss"] == "mse":
            loss = sum(((out[f"rgb_{p}"] - t) ** 2).mean() for p in passes)
        elif c["loss"] == "all6":
            g = torch.Generator(device=dev).manual_seed(seed)
            loss = sum((v * torch.randn(v.shape, device=dev, generator=g)).sum() for v in out.values()) / n
        else:                     # skewed
            tg = {}
            for p in passes:
                tp = t.clone()
                off = torch.from_numpy(np.random.RandomState(seed + 1).uniform(-1e-4, 1e-4, (256, 3)).astype(np.float32))
                tp[:256] = inf[f"rgb_{p}"][:256] + off.to(dev)
                tg[p] = tp
            loss = sum(((out[f"rgb_{p}"] - tg[p]) ** 2).mean() for p in passes)
    ws = out["rgb_coarse"].grad_fn.keep[-1]           # the TrainWorkspace of this forward
    loss.backward()
    torch.cuda.synchronize()
    assert _lib.load().nerfb200_check_status() == 0
    raw = ws.buf.cpu().numpy()
    grads = [{k: p.grad.detach().cpu().numpy() for k, p in m.named_parameters()} for m in models[:len(passes)]]
    seeds = []
    for p in passes:
        if c["loss"] == "fused":
            rgb_out = out[f"rgb_{p}"].detach().cpu().numpy().astype(np.float64)
            g_rgb = (2.0 * (rgb_out - target) / (3 * n)).astype(np.float32)
            seeds.append((g_rgb, None, None))
        else:
            gr = [out.get(f"{k}_{p}") for k in ("rgb", "depth", "opacity")]
            seeds.append(tuple(None if x is None or x.grad is None else x.grad.cpu().numpy() for x in gr))
    noise = [randoms.get("noise_coarse"), randoms.get("noise_fine")] if c["noise_std"] > 0 else [None, None]
    z_fine = inf["z_vals_fine"].cpu().numpy() if K else None
    return dict(c=c, n=n, S=S, K=K, rays=rays, randoms=randoms, raw=raw, grads=grads, seeds=seeds, noise=noise,
                ws=ws_np, z_fine=z_fine, seed=seed)


def stage_report(run, device="cpu"):
    """All stage comparisons of one step: (printable lines, violations of the bars).  `device`: the torch device of
    the float64 gradient contractions (tt.reference_grads)."""
    c, n, S, K, rays = run["c"], run["n"], run["S"], run["K"], run["rays"]
    dir_emb = orc.embed(rays[:, 3:6], 4)
    lines, bad = [], []
    L = tt.layout(n, S, K)
    for ps, P in enumerate(L):
        tag = ("coarse", "fine")[ps]
        net = tt.Net(run["ws"][ps])
        full = tt.WorkspaceTape(run["raw"], P)
        sub = tt.WorkspaceTape(run["raw"], P, _tiles(P["n_pad"], run["seed"] + ps))
        # depths: coarse from the oracle on the same uniforms, fine from the inference kernel
        z = full.z()
        zref = (orc.coarse_depths(rays, S, c["use_disp"], c["perturb"], run["randoms"]["perturb_rand"]) if ps == 0
                else run["z_fine"])
        if not np.array_equal(z, zref):
            bad.append(f"{tag} depths: {int((z != zref).sum())} differ from the reference")
        # encoding of the device's depths
        o, d = rays[:, :3], rays[:, 3:6]
        ray = sub.ray_of_rows()
        xyz = (o[ray] + d[ray] * z.reshape(-1)[sub.rows][:, None]).astype(np.float32)
        enc_ref = orc.embed(xyz, 10)
        enc_err = float((np.abs(sub.enc()[:, :63].astype(np.float64) - enc_ref) /
                         (tt.ulp16(enc_ref) + 2.0 ** -20)).max())
        if not enc_err <= tt.BARS["enc"]:
            bad.append(f"{tag} enc: {enc_err:.3g}")
        fwd = tt.check_forward(sub, net, dir_emb)
        masks = tt.check_masks(sub)
        comp = tt.check_composite(full, rays, *run["seeds"][ps], run["noise"][ps], c["noise_std"], c["white_back"])
        chain = tt.check_chain(sub, net)
        ref = tt.reference_grads(full, net, chain["scales"], dir_emb, device)
        gr = tt.check_grads(run["grads"][ps], ref)
        bad += [f"{tag} {b}" for b in tt.failures(fwd, masks, chain, comp, gr, noise=c["noise_std"] > 0)]
        lines.append(f"{tag}: enc {enc_err:.3g} ulp; " + " ".join(f"{k} {v:.3g}" for k, v in fwd.items()))
        lines.append(f"{tag}: masks illegal {masks['illegal']} legal {masks['legal_frac']:.3g}; composite " +
                     " ".join(f"{k} {v:.3g}" for k, v in comp.items()))
        lines.append(f"{tag}: scales log2 {[int(np.log2(s)) for s in chain['scales']]} saturated {chain['saturated']}")
        lines.append(f"{tag}: chain steps (ulp) " + " ".join(f"{chain[f'step{v}']:.3g}" for v in range(9)))
        lines.append(f"{tag}: chain accumulated rel L2 " + " ".join(f"{chain[f'acc{v}']:.3g}" for v in range(1, 9)) +
                     " | max " + " ".join(f"{chain[f'accmax{v}']:.3g}" for v in range(1, 9)))
        wr = max(gr.items(), key=lambda kv: kv[1][0])
        wm = max(gr.items(), key=lambda kv: kv[1][1])
        lines.append(f"{tag}: grads worst rel L2 {wr[1][0]:.3g} ({wr[0]}), worst max {wm[1][1]:.3g} ({wm[0]})")
        lines += [f"{tag}:   {k:32s} rel {r:.3g} max {m:.3g}" for k, (r, m) in gr.items()]
    return lines, bad


@pytest.mark.parametrize("name", list(CASES))
def test_backward_stages(name, dev, emb):
    run = run_step(name, dev, emb)
    lines, bad = stage_report(run)
    print(f"\n[{name}]")
    print("\n".join(lines))
    assert not bad, "\n".join(bad)


def test_gradient_accumulation_is_the_sum_of_single_steps(dev, emb):
    """Two forwards (two workspaces: the first is still busy when the second runs), one backward of the summed
    losses: every gradient equals the sum of the two batches' gradients taken one step at a time, bit for bit."""
    ws_np = cases.weights()
    n = 64
    batches = []
    for s in (91, 92):
        rs = np.random.RandomState(s)
        batches.append((torch.from_numpy(orc.make_rays(n, s)).to(dev),
                        torch.from_numpy(rs.uniform(0, 1, (n, 3)).astype(np.float32)).to(dev),
                        _to_dev({"perturb_rand": rs.rand(n, 64), "u_rand": rs.rand(n, 64)}, dev)))

    def loss_of(models, b):
        return nb.render_rays_loss(models, emb, b[0], b[1], 64, False, 1.0, 0.0, 64, 32768, True, randoms=b[2])["loss"]

    single = []
    for b in batches:
        m = _models(ws_np, dev)
        loss_of(m, b).backward()
        single.append([p.grad.clone() for net in m for p in net.parameters()])
    m = _models(ws_np, dev)
    l1 = loss_of(m, batches[0])
    l2 = loss_of(m, batches[1])
    (l1 + l2).backward()
    torch.cuda.synchronize()
    assert _lib.load().nerfb200_check_status() == 0
    for i, p in enumerate(p for net in m for p in net.parameters()):
        assert torch.equal(p.grad, single[0][i] + single[1][i]), i


def _probed_tiles(span, probe_tiles):
    """The tiles the chain kernel's probe visits in a pass (csrc/capi.cu: visit j -> j * stride mod span)."""
    s = span // probe_tiles if span > probe_tiles else 1
    while span > 1 and np.gcd(s, span) != 1:
        s += 1
    return {j * s % span for j in range(min(probe_tiles, span))}


def test_overflow_in_unprobed_tiles_is_reported(dev, emb):
    """A batch whose large gradients sit only in tiles the probe does not visit: every ray's target is its rendered
    colour to ~1e-5 except four rays, chosen so that neither their coarse nor their fine tile is probed, whose
    targets are random (residual ~0.3, 3e4 times more).  The scales the probe picks cannot hold those rays'
    gradients; the step must say so (status 102 through nerfb200_check_status), not hand back wrong gradients."""
    n, S, K = 1024, 64, 64
    half = (torch.cuda.get_device_properties(dev).multi_processor_count + 1) // 2
    L = tt.layout(n, S, K)
    spans = [P["n_pad"] // 128 for P in L]
    pc, pf = (_probed_tiles(sp, min(sp, half)) for sp in spans)
    hot = [r for r in range(n) if (r * S) // 128 not in pc and (r * (S + K)) // 128 not in pf]
    hot = hot[len(hot) // 8::len(hot) // 4][:4]
    assert len(hot) == 4
    rays = torch.from_numpy(orc.make_rays(n, 95)).to(dev)
    models = _models(cases.weights(), dev)
    rnd = {"seed": 95}
    with torch.no_grad():
        inf = nb.render_rays(models, emb, rays, S, False, 1.0, 0.0, K, 32768, True, randoms=rnd)
    rs = np.random.RandomState(95)
    targets = {}
    for p in ("coarse", "fine"):
        t = inf[f"rgb_{p}"] + torch.from_numpy(rs.uniform(-1e-5, 1e-5, (n, 3)).astype(np.float32)).to(dev)
        t[hot] = torch.from_numpy(rs.uniform(0, 1, (len(hot), 3)).astype(np.float32)).to(dev)
        targets[p] = t
    assert _lib.load().nerfb200_check_status() == 0
    out = nb.render_rays(models, emb, rays, S, False, 1.0, 0.0, K, 32768, True, randoms=rnd)
    ws = out["rgb_coarse"].grad_fn.keep[-1]
    sum(((out[f"rgb_{p}"] - targets[p]) ** 2).mean() for p in targets).backward()
    torch.cuda.synchronize()
    lib = _lib.load()
    rc = lib.nerfb200_check_status()
    msg = lib.nerfb200_last_error().decode()
    raw = ws.buf.cpu().numpy()
    sat = [tt.WorkspaceTape(raw, P).saturated() for P in L]
    print(f"\nhot rays {hot}: saturated elements {sat}, status rc {rc}: {msg}")
    assert sum(sat) > 0                  # the case does overflow ...
    assert rc != 0 and "102" in msg      # ... and the step reports it
    assert lib.nerfb200_check_status() == 0
