"""The renderer's forward, stage by stage, on the device's own values (pytest -m gpu).

Per case: one inference render with extras (weights and fine depths), one test_time render, and one training
forward with the fused loss on the same rays and random numbers.  The training workspace holds each pass's depths,
sigma and rgb (tests/train_tape.py reads it).  Then:

  1. mode invariance, bitwise: training outputs == inference outputs, workspace fine depths == z_vals_fine,
     test_time=True (sigma-only coarse MLP) == test_time=False for everything both return;
  2. resampling, bitwise: z_vals_fine == tests/render_tape.py z_fine on the device's weights_coarse and coarse
     depths; the emulation against float64 sample_pdf (0 unflagged samples outside its bar);
  3. compositing: weights against float64 compositing of the workspace's sigma / depths, rgb / depth / opacity
     against float64 sums of the device's own weights;
  4. the fused loss epilogue against float64 sums of the device's rendered rgb.

Plus the stand-alone sample_pdf (bit for bit, up to n_weights = 4096) and volume_render (float64, edge inputs).
The bars and the values measured on an H100 stand in tests/render_tape.py BARS.
"""
import subprocess

import numpy as np
import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200.training import TrainWorkspace
from oracle import nerf_oracle as orc
from tests import cases
from tests import render_tape as rt
from tests import train_tape as tt

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
U32 = 2.0 ** -24
DEFAULTS = dict(n=65, S=64, K=64, use_disp=False, perturb=1.0, noise_std=0.0, white_back=True, rng="tensors",
                weights="random", kind="blender", edge=None)
# name: one case (ray seed = the case's index + 200)
CASES = {
    "s32_k32_disp": dict(n=33, S=32, K=32, use_disp=True, white_back=False),
    "s64_k64_det": dict(perturb=0.0),                               # u = linspace: u = 1 on the last knot
    "s64_k0": dict(n=31, K=0),
    "s128_k64_sf192": dict(n=75, S=128),
    "s32_k160_sf192": dict(n=51, S=32, K=160),
    "s64_k128_noise": dict(n=49, K=128, noise_std=1.0),
    "ndc_seed": dict(n=97, kind="ndc", rng="seed", white_back=False),
    "ndc_noise_det": dict(n=45, kind="ndc", perturb=0.0, noise_std=1.0, white_back=False),
    "trained_k64": dict(n=129, weights="trained"),
    "trained_det_k128": dict(n=63, weights="trained", perturb=0.0, K=128),
    "trained_s128_seed": dict(n=41, S=128, K=64, weights="trained", rng="seed"),
    "many_groups_2075": dict(n=148 * 14 + 3, rng="seed"),         # each CTA walks several groups
    "edge_near_eq_far": dict(n=41, edge="equal"),                  # all ties, zero deltas
    "edge_far_below_near": dict(n=41, edge="below"),              # decreasing coarse depths
    "edge_disp_near_far": dict(n=41, edge="close", use_disp=True, perturb=0.0),
    "large_coords": dict(n=65, kind="large"),                      # |o + d z| up to 64
}


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def emb():
    return [nb.Embedding(3, 10), nb.Embedding(3, 4)]


@pytest.fixture(scope="module", autouse=True)
def card(dev):
    name = torch.cuda.get_device_name(dev)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(dev.index)],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    print(f"\ncard: {name}, power limit {pl}")


def _models(ws, dev):
    out = []
    for w in ws:
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        out.append(m.to(dev))
    return out


def _rays(c, seed):
    n = c["n"]
    rs = np.random.RandomState(seed + 1)
    if c["kind"] == "large":
        rays = orc.make_rays(n, seed)
        rays[:, :3] = rs.uniform(-58, 58, (n, 3))
        return rays.astype(F32)
    rays = orc.make_rays(n, seed, "ndc" if c["kind"] == "ndc" else "blender")
    if c["edge"] == "equal":
        rays[:, 7] = rays[:, 6]
    elif c["edge"] == "below":       # far 1 ulp .. 1e-2 below near
        gap = np.where(np.arange(n) % 2 == 0, np.spacing(rays[:, 6]), rs.uniform(1e-6, 1e-2, n)).astype(F32)
        rays[:, 7] = rays[:, 6] - gap
    elif c["edge"] == "close":       # near ~ far: 1/(1/near (1 - t) + 1/far t) rounds non-monotonically
        rays[:, 7] = rays[:, 6] + (np.arange(n) % 8).astype(F32) * np.spacing(rays[:, 6])
    return rays


def _lists_inverted(z):
    return bool((z[:, 1:] < z[:, :-1]).any())


def run_case(name, dev, emb):
    return run_render(dict(DEFAULTS, **CASES[name]), 200 + list(CASES).index(name), dev, emb)


def run_render(c, seed, dev, emb, rays=None, rnd=None):
    """The three renders of configuration `c` (DEFAULTS' keys) on rays and random numbers drawn from `seed`; `rays`
    (n, 8) and `rnd` (numpy random tensors keyed as render_rays' randoms) replace the drawn ones when given."""
    n, S, K = c["n"], c["S"], c["K"]
    rays = _rays(c, seed) if rays is None else rays
    rs = np.random.RandomState(seed)
    target = rs.uniform(0, 1, (n, 3)).astype(F32)
    rnd_np = {}
    if rnd is not None:
        rnd_np = dict(rnd)
    elif c["perturb"] > 0:
        rnd_np["perturb_rand"] = rs.rand(n, S).astype(F32)
        if K:
            rnd_np["u_rand"] = rs.rand(n, K).astype(F32)
    if c["noise_std"] > 0 and rnd is None:
        rnd_np["noise_coarse"] = rs.randn(n, S).astype(F32)
        if K:
            rnd_np["noise_fine"] = rs.randn(n, S + K).astype(F32)
    tensors = {k: torch.from_numpy(v).to(dev) for k, v in rnd_np.items()}
    rng_seed = None
    if c["rng"] == "seed":
        rng_seed = 1000 + seed
        from tests import philox
        ph = philox.randoms(rng_seed, n, S, K)
        rnd_np.update({k: v for k, v in ph.items() if c["perturb"] > 0})
        tensors = {k: v for k, v in tensors.items() if k.startswith("noise")}
        tensors["seed"] = rng_seed
    ws_np = cases.trained_weights() if c["weights"] == "trained" else cases.weights()
    models = _models(ws_np, dev)
    r, t = torch.from_numpy(rays).to(dev), torch.from_numpy(target).to(dev)
    args = (S, c["use_disp"], c["perturb"], c["noise_std"], K, 32768, c["white_back"])
    with torch.no_grad():
        inf = nb.render_rays(models, emb, r, *args, randoms=tensors, extras=True)
        tst = nb.render_rays(models, emb, r, *args, test_time=True, randoms=tensors, extras=True)
    out = nb.render_rays_loss(models, emb, r, t, *args[:5], 32768, c["white_back"], randoms=tensors)
    ws = out["rgb_coarse"].grad_fn.keep[-1]
    torch.cuda.synchronize()
    raw = ws.buf.cpu().numpy()
    res = dict(c=c, n=n, S=S, K=K, rays=rays, target=target, rnd=rnd_np, raw=raw, rng_seed=rng_seed,
               inf={k: v.cpu().numpy() for k, v in inf.items()}, tst={k: v.cpu().numpy() for k, v in tst.items()},
               train={k: v.detach().cpu().numpy() for k, v in out.items()})
    del out
    TrainWorkspace.clear()           # no backward follows: drop the workspace with its graph
    return res


def mode_findings(run):
    """Bitwise mode invariance; returns the list of differences."""
    inf, tst, tr = run["inf"], run["tst"], run["train"]
    bad = []
    for k in ("rgb_coarse", "depth_coarse", "opacity_coarse", "rgb_fine", "depth_fine", "opacity_fine"):
        if k in inf and not np.array_equal(tr[k], inf[k], equal_nan=True):
            bad.append(f"training {k} differs from inference in {int((tr[k] != inf[k]).sum())} elements")
    for k in ("opacity_coarse", "weights_coarse", "rgb_fine", "depth_fine", "opacity_fine", "z_vals_fine",
              "weights_fine"):
        if k in inf and not np.array_equal(tst[k], inf[k], equal_nan=True):
            bad.append(f"test_time {k} differs from test_time=False in {int((tst[k] != inf[k]).sum())} elements")
    if run["K"]:
        zf = tt.WorkspaceTape(run["raw"], tt.layout(run["n"], run["S"], run["K"])[1]).z()
        if not np.array_equal(zf, inf["z_vals_fine"], equal_nan=True):
            bad.append(f"workspace fine depths differ from z_vals_fine in {int((zf != inf['z_vals_fine']).sum())}")
    return bad


def composite_report(run):
    """Stage 3: {metric: worst value in units of its bar} per pass."""
    c, n, S, K, rays = run["c"], run["n"], run["S"], run["K"], run["rays"]
    out = {}
    for ps, P in enumerate(tt.layout(n, S, K)):
        tag = ("coarse", "fine")[ps]
        Sp = P["S"]
        tape = tt.WorkspaceTape(run["raw"], P)
        sig = tape.sigma().reshape(n, Sp)
        rgb = tape.rgb().reshape(n, Sp, 3)
        z = tape.z()
        noise = run["rnd"].get(("noise_coarse", "noise_fine")[ps]) if c["noise_std"] > 0 else None
        w_dev = run["inf"][f"weights_{tag}"].astype(F64)
        w64, _, _, _ = rt.composite64(sig, z, rays[:, 3:6], None, noise, c["noise_std"])
        dw = np.abs(w_dev - w64) / rt.weight_units(Sp)
        out[f"{tag}.weights"] = float(dw[:, :-1].max())
        out[f"{tag}.weights_last"] = float(dw[:, -1].max())
        opac = w_dev.sum(1)
        wsum = np.abs(w_dev).sum(1)
        e = np.abs(run["inf"][f"opacity_{tag}"] - opac) / rt.sum_bar_units(Sp, wsum)
        out[f"{tag}.opacity"] = float(e.max())
        dep = (w_dev * z).sum(1)
        e = np.abs(run["inf"][f"depth_{tag}"] - dep) / rt.sum_bar_units(Sp, (np.abs(w_dev * z)).sum(1))
        out[f"{tag}.depth"] = float(e.max())
        col = (w_dev[..., None] * rgb).sum(1)
        absc = (np.abs(w_dev[..., None] * rgb)).sum(1)
        extra = 0.0
        if c["white_back"]:
            col = col + (1 - opac)[:, None]
            absc = absc + wsum[:, None]
            extra = 2 * U32 * (np.abs(col) + 1)
        e = np.abs(run["inf"][f"rgb_{tag}"] - col) / rt.sum_bar_units(Sp, absc, extra)
        out[f"{tag}.rgb"] = float(e.max())
    return out


def loss_report(n, S, K, rgb_c, rgb_f, target, loss4, sm_count):
    """Stage 4: errors of mse_coarse / mse_fine / loss / psnr in units of their bars (rays per helper warp m:
    m + 8 fp32 roundings of sums of squares; psnr: 10 / ln 10 times that relative bound + 4 ulp)."""
    grid = min(sm_count, (n + 1) // 2)
    m = -(-(-(-n // grid)) // 2)
    rel = (m + 8) * U32
    t = target.astype(F64)
    mc = ((rgb_c.astype(F64) - t) ** 2).sum() / (3 * n)
    mf = ((rgb_f.astype(F64) - t) ** 2).sum() / (3 * n) if K else 0.0
    fin = mf if K else mc
    ps = -10 * np.log10(fin)
    den = lambda v: max(rel * v, 1e-45)
    out = {"mse_coarse": abs(loss4["mse_coarse"] - mc) / den(mc),
           "mse_fine": abs(loss4["mse_fine"] - mf) / den(mf) if K else float(loss4["mse_fine"] != 0) * 1e9,
           "loss": abs(loss4["loss"] - (mc + mf)) / ((rel + U32) * (mc + mf)),
           "psnr": abs(loss4["psnr"] - ps) / (10 / np.log(10) * rel + 4 * float(np.spacing(F32(abs(ps)))))}
    return {k: float(v) for k, v in out.items()}


def enc_report(run):
    """Positional encoding of the workspace against float64 sin / cos of the device's own fp32 point o + d z (the
    factor 2^k is exact), in units of (fp16 ulp + 2^-20) as test_gpu_train_stages applies it; with max |x|."""
    n, S, K, rays = run["n"], run["S"], run["K"], run["rays"]
    worst, xmax = 0.0, 0.0
    for P in tt.layout(n, S, K):
        nt = P["n_pad"] // 128
        tape = tt.WorkspaceTape(run["raw"], P, None if nt <= 24 else np.arange(24))
        ray = tape.ray_of_rows()
        z = tape.z().reshape(-1)[tape.rows]
        x = (rays[ray, :3] + (rays[ray, 3:6] * z[:, None]).astype(F32)).astype(F32).astype(F64)
        ref = [x]
        for k in range(10):
            ref += [np.sin(2.0 ** k * x), np.cos(2.0 ** k * x)]
        ref = np.concatenate(ref, 1)
        err = np.abs(tape.enc()[:, :63].astype(F64) - ref) / (tt.ulp16(ref) + 2.0 ** -20)
        worst = max(worst, float(err.max()))
        xmax = max(xmax, float(np.abs(x).max()))
    return worst, xmax


def forward_report(run, sm_count):
    """Stages 1-4 of one run_render result against their bars: (printable lines, violations)."""
    c, n, S, K = run["c"], run["n"], run["S"], run["K"]
    bad = mode_findings(run)
    lines = []
    # coarse depths: the existing bitwise pin
    zc = tt.WorkspaceTape(run["raw"], tt.layout(n, S, K)[0]).z()
    zref = orc.coarse_depths(run["rays"], S, c["use_disp"], c["perturb"], run["rnd"].get("perturb_rand"))
    if not np.array_equal(zc, zref, equal_nan=True):
        bad.append(f"coarse depths: {int((zc != zref).sum())} differ from the oracle")
    if K:
        u = rt.fine_uniforms(n, K, c["perturb"], run["rnd"].get("u_rand"))
        rep = rt.check_resampling(run["inf"]["z_vals_fine"], run["inf"]["weights_coarse"], zc, u)
        lines.append(f"resampling: {rep['differ']} of {n * (S + K)} depths differ from the emulation; "
                     f"float64: {rep['f64_bad']} unflagged outside the bar, {rep['flagged']} flagged of {n * K}; "
                     f"exhaustive merge on {rep['exhaustive']} rays; coarse list inverted {_lists_inverted(zc)}")
        if rep["differ"]:
            bad.append(f"z_vals_fine: {rep['differ']} depths differ from the emulation")
        if rep["nonfinite_mismatch"]:
            bad.append(f"resampling: {rep['nonfinite_mismatch']} depths finite in one of fp32 / float64")
        if c["edge"] is None and rep["f64_bad"] > rt.BARS["sample_pdf64"]:
            bad.append(f"resampling: {rep['f64_bad']} unflagged samples outside the float64 bar")
    comp = composite_report(run)
    lines.append("compositing: " + " ".join(f"{k} {v:.3g}" for k, v in comp.items()))
    for k, v in comp.items():
        bar = rt.BARS["weights_last" if k.endswith("last") else "weights" if k.endswith("weights") else "sums"]
        if not v <= bar:
            bad.append(f"compositing {k}: {v:.3g} > {bar}")
    tr = run["train"]
    lr = loss_report(n, S, K, tr["rgb_coarse"], tr.get("rgb_fine"), run["target"], tr, sm_count)
    lines.append("loss: " + " ".join(f"{k} {v:.3g}" for k, v in lr.items()))
    for k, v in lr.items():
        if not v <= rt.BARS["psnr" if k == "psnr" else "loss"]:
            bad.append(f"loss {k}: {v:.3g}")
    enc, xmax = enc_report(run)
    lines.append(f"enc: {enc:.3g} (max |x| {xmax:.3g})")
    if not enc <= tt.BARS["enc"]:
        bad.append(f"enc: {enc:.3g} > {tt.BARS['enc']} at max |x| {xmax:.3g}")
    return lines, bad


@pytest.mark.parametrize("name", list(CASES))
def test_forward_stages(name, dev, emb):
    run = run_case(name, dev, emb)
    lines, bad = forward_report(run, torch.cuda.get_device_properties(dev).multi_processor_count)
    print(f"\n[{name}] n {run['n']} S {run['S']} K {run['K']}\n" + "\n".join(lines))
    assert not bad, "\n".join(bad)


def test_loss_epilogue_over_batch_sizes(dev, emb):
    """The fused loss at 1 ray, 3 rays (fewer rays than CTAs), coarse only (psnr from the coarse pass, mse_fine 0) and
    16,385 rays (62 per CTA on 132 SMs); each shape twice back to back on the same workspace (its ticket counter
    must be back at 0), and shapes interleaved.  16,385 rays at S = 32 keep the training workspace at 4.8 GB; the
    196,608-ray batch of bench.py's render would need 57 GB even at S = 32, K = 0."""
    sm = torch.cuda.get_device_properties(dev).multi_processor_count
    models = _models(cases.weights(), dev)
    seq = [(1, 64, 64), (3, 64, 64), (3, 64, 64), (16385, 32, 0), (16385, 32, 0), (1, 32, 0), (3, 64, 64)]
    bad, prev = [], {}
    for i, (n, S, K) in enumerate(seq):
        rays = torch.from_numpy(orc.make_rays(n, 300 + n)).to(dev)
        tgt = torch.from_numpy(np.random.RandomState(n).uniform(0, 1, (n, 3)).astype(F32)).to(dev)
        out = nb.render_rays_loss(models, emb, rays, tgt, S, False, 1.0, 0.0, K, 32768, True, randoms={"seed": n})
        out["rgb_coarse"].grad_fn.keep[-1].busy = False      # no backward: the next call of this shape reuses it
        torch.cuda.synchronize()
        o = {k: v.detach().cpu().numpy() for k, v in out.items()}
        lr = loss_report(n, S, K, o["rgb_coarse"], o.get("rgb_fine"), tgt.cpu().numpy(), o, sm)
        print(f"\nloss n {n} S {S} K {K}: " + " ".join(f"{k} {v:.3g}" for k, v in lr.items()))
        bad += [f"n {n} K {K} {k}: {v:.3g}" for k, v in lr.items() if not v <= rt.BARS["psnr" if k == "psnr" else "loss"]]
        key = (n, S, K)
        if key in prev:
            for k in ("loss", "psnr", "mse_coarse", "mse_fine"):
                if not np.array_equal(prev[key][k], o[k]):
                    bad.append(f"n {n} K {K}: {k} of a repeated launch differs")
        prev[key] = o
        del out
    TrainWorkspace.clear()
    assert not bad, "\n".join(bad)


# ------------------------------------------------------------------------------------------ stand-alone rows
def _pdf_inputs(nw, R=8, K=40, seed=0):
    rs = np.random.RandomState(seed + nw)
    w = rs.dirichlet(np.ones(nw) * 0.5, R).astype(F32)
    w[0] = 0                                        # uniform cdf
    w[1] = 0
    w[1, nw // 2] = 1                               # one-hot: denom branch elsewhere
    w[2, rs.rand(nw) < 0.7] = 0                     # flat runs
    bins = np.sort(rs.uniform(2, 6, (R, nw + 1)), 1).astype(F32)
    cdf = rt.cdf_standalone(w)
    u = rs.rand(R, K).astype(F32)
    u[:, 0], u[:, 1] = 0.0, 1.0
    k = np.minimum(np.arange(2, 10) * max(nw // 9, 1), nw)
    u[:, 2:10] = cdf[:, k]                          # on knots
    return bins, w, u


@pytest.mark.parametrize("nw", [1, 2, 31, 32, 33, 63, 126, 1000, 3071, 3072, 4096])
def test_sample_pdf_bitwise(nw, dev):
    """nerfb200_sample_pdf against cdf_standalone + inverse_cdf, bit for bit, up to the header's n_weights <= 4096
    (from 3072 the kernel's cdfs need more than the 48 KB of shared memory a launch gets without opting in)."""
    bins, w, u = _pdf_inputs(nw)
    got = nb.sample_pdf(torch.from_numpy(bins).to(dev), torch.from_numpy(w).to(dev), u.shape[1],
                        u=torch.from_numpy(u).to(dev)).cpu().numpy()
    ref = rt.inverse_cdf(rt.cdf_standalone(w), bins, u)
    diff = int((got != ref).sum())
    z64, flagged, bar = rt.sample_pdf64(bins, w, u, sequential=True)
    far = int((~(np.abs(got - z64) <= bar) & ~flagged).sum())
    print(f"\nsample_pdf nw {nw}: {diff} of {got.size} differ from the emulation; float64 {far} unflagged outside "
          f"the bar, {int(flagged.sum())} flagged")
    assert diff == 0 and far == 0


def _vr_inputs(S, seed):
    rs = np.random.RandomState(seed)
    n = 97
    sig = (rs.randn(n, S) * 3).astype(F32)
    sig[0] = 1e30                                   # alpha = 1 (delta sigma overflows to inf)
    sig[1] = -1e3                                   # negative sigma (also under noise): alpha = 0
    sig[2, ::3] = 3e4
    rgb = rs.rand(n, S, 3).astype(F32)
    z = np.sort(rs.uniform(2, 6, (n, S)).astype(F32), -1)
    z[3:8, 5:9] = z[3:8, 5:6]                       # duplicate depths: zero deltas
    z[8] = z[8, 0]                                  # one depth for the whole ray
    d = (rs.randn(n, 3) * rs.uniform(0.2, 3, (n, 1))).astype(F32)   # non-unit directions
    noise = rs.randn(n, S).astype(F32)
    return sig, rgb, z, d, noise


@pytest.mark.parametrize("S", [32, 64, 96, 128, 160, 192])
@pytest.mark.parametrize("noise_std,wb", [(0.0, False), (1.0, True)])
def test_volume_render_vs_float64(S, noise_std, wb, dev):
    sig, rgb, z, d, noise = _vr_inputs(S, S)
    nz = noise if noise_std > 0 else None
    T = lambda a: None if a is None else torch.from_numpy(a).to(dev)
    w, c, dp, op = [x.cpu().numpy() for x in nb.volume_render(T(sig), T(rgb), T(z), T(d), T(nz), noise_std, wb)]
    w64, _, _, _ = rt.composite64(sig, z, d, None, nz, noise_std)
    e = rt.composite_errors(sig, rgb, z, d, nz, noise_std, wb, w, c, dp, op)
    print(f"\nvolume_render S {S} noise {noise_std}: " + " ".join(f"{k} {v:.3g}" for k, v in e.items()))
    assert np.all(np.isfinite(w)) and w[0, 0] == 1 and np.all(w[1] == 0)
    np.testing.assert_allclose(op, w64.sum(1), rtol=0, atol=S * 4 * U32)     # weights sum to the opacity
    assert not rt.composite_violations(e), rt.composite_violations(e)
