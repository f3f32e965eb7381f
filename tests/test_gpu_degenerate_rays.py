"""The fused renderer on degenerate and non-finite rays (pytest -m gpu): every ray isolated, independent of the launch
shape, and held to float64.

A fixed catalogue of poisoned rays (NaN / +inf / -inf in each of the 8 columns, which includes far = +inf with a
finite near; d = 0, |d| ~ 1e-30 and subnormal, |d| ~ 1e20, an NDC ray, near < 0, far = 1e10 and 3e38) plus two rays
with a NaN in their perturb_rand or u_rand row is mixed into 1200 ordinary rays; each poisoned ray sits at an even
and an odd index, inside a multi-group CTA range.  Each S/K, perturb, noise mode (and use_disp, where the NDC ray
has near = 0) renders the batch for inference with extras, test_time and training with the fused loss, then:

  1. isolation, bitwise: every clean ray's outputs, weights and z_vals_fine equal the render of the clean rays
     alone with the same per-ray random rows, which also meets the stage bars of test_gpu_render_stages; so do the
     poisoned rays whose depths are finite (d = 0, tiny d, NDC, near < 0), rendered alone;
  2. launch shape and position: max_ctas 1, 3 and all SMs, the batch reversed, and sub-batches with each poisoned ray
     first, second and last in its sub-batch give the same values, NaN equal to NaN; culled rendering on a trained
     occupancy grid equals the full render on every live ray (test_culled_equals_full);
  3. semantics: z_vals_fine equals tests/render_tape.py z_fine (torch.sort's NaN-last order, the reference's own fp32
     mid-points) bitwise; every other output's finiteness pattern equals that of the float64 restatement
     tests/test_degenerate_rays_ref.py render64 with sigma -> fmax(sigma, 0), on rays whose points stay within
     |x| <= 64 (the range the fp16 forward's encoding bar is pinned over; larger |x| is test 5's);
  4. no silent finite gradients: a training step on a batch with a non-finite ray, on the render path and through
     NeRF.forward(autograd_impl='fused'), reports through the device status word (test_nonfinite_ray_gradients,
     test_nonfinite_point_gradients_nerf_forward);
  5. large coordinates: the first |x| at which the kernel's sigma or rgb stops being finite where fp32 is finite, for
     random and trained weights, printed and pinned with the range over which the encoding holds its bar
     (test_large_coordinates).
"""
import ctypes

import numpy as np
import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib
from nerf_pl_b200.nerf import packed_weights
from nerf_pl_b200.rendering import _render_args
from oracle import nerf_oracle as orc
from tests import cases
from tests import render_tape as rt
from tests import test_degenerate_rays_ref as dr
from tests import test_gpu_render_stages as ts
from tests import train_tape as tt

pytestmark = pytest.mark.gpu

F32 = np.float32
N = 1200
SUB = 7                      # sub-batch length of the position check
XLIM = 64.0                  # |x| up to which the finiteness pattern is held to render64
COLS = ("ox", "oy", "oz", "dx", "dy", "dz", "near", "far")
# (S, K, perturb, noise_std, use_disp)
MODES = [(S, K, p, nz, False) for S, K in ((64, 64), (64, 128), (32, 160)) for p in (0.0, 1.0) for nz in (0.0, 1.0)]
MODES.append((64, 64, 1.0, 0.0, True))
dev = ts.dev
emb = ts.emb
card = ts.card


def catalogue():
    """[(family, name, ray (8,) | None)]; None: an ordinary ray whose random row is poisoned instead."""
    base = orc.make_rays(1, 11)[0]
    out = []
    for c in range(8):
        for v in (np.nan, np.inf, -np.inf):
            r = base.copy()
            r[c] = v
            out.append(("nonfinite", f"{COLS[c]}={v}", r))
    deg = {
        "d=0": lambda r: r.__setitem__(slice(3, 6), 0.0),
        "|d|=1e-30": lambda r: r.__setitem__(slice(3, 6), r[3:6] * F32(1e-30)),   # fp32 |d|^2 underflows: |d| = 0
        "d_subnormal": lambda r: r.__setitem__(slice(3, 6), r[3:6] * F32(1e-39)),
        "|d|=1e20": lambda r: r.__setitem__(slice(3, 6), r[3:6] * F32(1e20)),     # fp32 |d|^2 overflows: |d| = inf
        "ndc": lambda r: r.__setitem__(slice(0, 8), orc.make_rays(1, 12, "ndc")[0]),
        "near<0": lambda r: r.__setitem__(6, -1.5),
        "far=1e10": lambda r: r.__setitem__(7, 1e10),
        "far=3e38": lambda r: r.__setitem__(7, 3e38),                              # fp32 mid-points overflow
    }
    for name, f in deg.items():
        r = base.copy()
        f(r)
        out.append(("degenerate", name, r.astype(F32)))
    out += [("random", "perturb_rand NaN", None), ("random", "u_rand NaN", None)]
    return out


def build_batch(S, K, perturb, noise_std, seed):
    """(rays (N, 8), rnd {name: (N, ..)}, poisoned {index: catalogue entry})."""
    cat = catalogue()
    rays = orc.make_rays(N, seed)
    rs = np.random.RandomState(seed)
    rnd = {}
    if perturb > 0:
        rnd["perturb_rand"] = rs.rand(N, S).astype(F32)
        rnd["u_rand"] = rs.rand(N, K).astype(F32)
    if noise_std > 0:
        rnd["noise_coarse"] = rs.randn(N, S).astype(F32)
        rnd["noise_fine"] = rs.randn(N, S + K).astype(F32)
    poisoned = {}
    for j, (fam, name, r) in enumerate(cat):
        e = 20 + 26 * j
        for p in (e, e + 13):                       # an even and an odd index
            poisoned[p] = (fam, name)
            if r is not None:
                rays[p] = r
            elif perturb > 0:
                rnd["perturb_rand" if name.startswith("perturb") else "u_rand"][p, 9] = np.nan
    return rays, rnd, poisoned


def _models(weights):
    return ts._models(cases.trained_weights() if weights == "trained" else cases.weights(), torch.device("cuda:0"))


def infer(models, rays, rnd, S, K, perturb, noise_std, use_disp, max_ctas=0):
    """One inference render with extras through the C ABI at a given max_ctas; numpy results keyed as render_rays."""
    d = torch.device("cuda:0")
    n = len(rays)
    f32 = dict(dtype=torch.float32, device=d)
    shapes = dict(rgb_coarse=(n, 3), depth_coarse=(n,), opacity_coarse=(n,), rgb_fine=(n, 3), depth_fine=(n,),
                  opacity_fine=(n,), z_fine=(n, S + K), weights_coarse=(n, S), weights_fine=(n, S + K))
    outs = {k: torch.empty(s, **f32) for k, s in shapes.items()}
    T = lambda k: torch.from_numpy(np.ascontiguousarray(rnd[k])).to(d) if k in rnd else None  # noqa: E731
    r = torch.from_numpy(np.ascontiguousarray(rays)).to(d)
    packed = (packed_weights(models[0]), packed_weights(models[1]))
    args = _render_args(r, S, K, use_disp, perturb, noise_std, True, False, packed,
                        (T("perturb_rand"), T("noise_coarse"), T("u_rand"), T("noise_fine")), outs, None)
    args.max_ctas = max_ctas
    _lib.call("nerfb200_render_rays", d, ctypes.byref(args))
    torch.cuda.synchronize()
    res = {k: v.cpu().numpy() for k, v in outs.items()}
    res["z_vals_fine"] = res.pop("z_fine")
    return res


def _rows(rnd, idx):
    return {k: np.ascontiguousarray(v[idx]) for k, v in rnd.items()}


def _scalars_out(d):
    return {k: v for k, v in d.items() if np.ndim(v) > 0}


@pytest.mark.parametrize("S,K,perturb,noise_std,use_disp", MODES,
                         ids=[f"s{S}_k{K}_p{int(p)}_n{int(nz)}" + ("_disp" if ud else "") for S, K, p, nz, ud in MODES])
def test_degenerate_batch(S, K, perturb, noise_std, use_disp, dev, emb):
    seed = 700 + MODES.index((S, K, perturb, noise_std, use_disp))
    rays, rnd, poisoned = build_batch(S, K, perturb, noise_std, seed)
    pidx = np.array(sorted(poisoned))
    cidx = np.setdiff1d(np.arange(N), pidx)
    c = dict(ts.DEFAULTS, n=N, S=S, K=K, perturb=perturb, noise_std=noise_std, use_disp=use_disp, white_back=True,
             rng="tensors")
    models = _models("random")
    with np.errstate(all="ignore"):
        full = ts.run_render(c, seed, dev, emb, rays=rays, rnd=rnd)
    bad = [f"modes: {m}" for m in ts.mode_findings(full)]
    lines = []

    # 1. isolation: the clean rays alone, same random rows
    clean = ts.run_render(dict(c, n=len(cidx)), seed, dev, emb, rays=rays[cidx], rnd=_rows(rnd, cidx))
    for mode in ("inf", "tst", "train"):
        mm = dr.position_mismatch(_scalars_out(full[mode]), _scalars_out(clean[mode]), cidx, slice(None))
        bad += [f"isolation ({mode}): clean {k} differs from the clean-only render in {v}" for k, v in mm.items()]
    stage_lines, stage_bad = ts.forward_report(clean, torch.cuda.get_device_properties(dev).multi_processor_count)
    lines += ["clean rays: " + s for s in stage_lines]
    bad += ["clean rays: " + b for b in stage_bad]

    # 2. launch shape and position
    inf = full["inf"]
    for m in (1, 3, 0):
        mm = dr.position_mismatch(infer(models, rays, rnd, S, K, perturb, noise_std, use_disp, m), inf,
                                  slice(None), slice(None))
        bad += [f"max_ctas {m}: {k} differs in {v}" for k, v in mm.items()]
    rev = np.arange(N)[::-1].copy()
    mm = dr.position_mismatch(infer(models, rays[rev], _rows(rnd, rev), S, K, perturb, noise_std, use_disp), inf,
                              slice(None), rev)
    bad += [f"reversed batch: {k} differs in {v}" for k, v in mm.items()]
    for p in pidx[::2]:
        for a in (0, 1, SUB - 1):                  # the poisoned ray first, second, last in its sub-batch
            sl = np.arange(p - a, p - a + SUB)
            mm = dr.position_mismatch(infer(models, rays[sl], _rows(rnd, sl), S, K, perturb, noise_std, use_disp),
                                      inf, slice(None), sl)
            bad += [f"sub-batch at {p} (position {a}) {poisoned[p][1]}: {k} differs in {v}" for k, v in mm.items()]

    # 3. semantics: z_vals_fine against the emulation (NaN last), the rest against render64's finiteness
    zc = tt.WorkspaceTape(full["raw"], tt.layout(N, S, K)[0]).z()
    with np.errstate(all="ignore"):
        u = rt.fine_uniforms(N, K, perturb, rnd.get("u_rand"))
        zf, _, _ = rt.z_fine(inf["weights_coarse"], zc, u)
        d32 = torch.linalg.vector_norm(torch.from_numpy(rays[pidx, 3:6]).to(dev), dim=-1).cpu().numpy()
        ref = dr.render64(cases.weights(), rays[pidx], S, K, use_disp, perturb, noise_std, True,
                          _rows(rnd, pidx), dnorm=d32)
    mm = dr.position_mismatch({"z_vals_fine": inf["z_vals_fine"]}, {"z_vals_fine": zf}, slice(None), slice(None))
    bad += [f"z_vals_fine differs from the NaN-last emulation in {v}" for v in mm.values()]
    fams = {}
    for i, p in enumerate(pidx):
        fams.setdefault(poisoned[p][1], []).append(i)
    dev_p = {k: v[pidx] for k, v in inf.items()}
    for name, rows in fams.items():
        in_range = bool((ref["xmax"][rows] <= XLIM).all())
        nonfin = {k: int((~np.isfinite(dev_p[k][rows])).sum()) for k in dr.OUT_KEYS if k in dev_p}
        tag = ", ".join(f"{k} {v}" for k, v in nonfin.items() if v) or "all finite"
        if in_range:
            mm = dr.pattern_mismatch(dev_p, ref, rows)
            bad += [f"{name}: {k} finiteness differs from float64 in {v}" for k, v in mm.items()]
            lines.append(f"{name}: non-finite {tag}; pattern mismatches {sum(mm.values())}")
        else:
            lines.append(f"{name}: non-finite {tag}; |x| up to {ref['xmax'][rows].max():.3g} (beyond {XLIM})")

    # poisoned rays whose depths are finite, sorted and within XLIM (d = 0, tiny d, NDC, near < 0 where the mode
    # keeps them so) also meet the stage bars: rendered alone they are bitwise their rows of the batch
    fidx = np.array([p for i, p in enumerate(pidx) if poisoned[p][0] == "degenerate" and ref["xmax"][i] <= XLIM
                     and np.isfinite(zc[p]).all() and (np.diff(zc[p]) >= 0).all()
                     and np.isfinite(inf["z_vals_fine"][p]).all()])
    fin = ts.run_render(dict(c, n=len(fidx)), seed, dev, emb, rays=rays[fidx], rnd=_rows(rnd, fidx))
    mm = dr.position_mismatch(_scalars_out(fin["inf"]), inf, slice(None), fidx)
    bad += [f"finite-depth poisoned rays rendered alone: {k} differs in {v}" for k, v in mm.items()]
    stage_lines, stage_bad = ts.forward_report(fin, torch.cuda.get_device_properties(dev).multi_processor_count)
    names = sorted({poisoned[p][1] for p in fidx})
    lines += [f"finite-depth poisoned rays ({', '.join(names)}): " + s for s in stage_lines]
    bad += ["finite-depth poisoned rays: " + b for b in stage_bad]
    print(f"\n[N {N} S {S} K {K} perturb {perturb} noise {noise_std} use_disp {use_disp}]\n" + "\n".join(lines))
    assert not bad, "\n".join(bad[:60])


def test_culled_equals_full(dev, emb):
    """render_rays_culled on a trained occupancy grid equals the full render on every live ray; every ray with a
    non-finite value is live (the finite degenerate rays may be culled)."""
    rays, rnd, poisoned = build_batch(64, 64, 0.0, 0.0, 790)
    models = _models("trained")
    grid = nb.occupancy_grid(models[1], 128, *(((-1.5, 1.5),) * 3), 1.0, 1)
    r = torch.from_numpy(rays).to(dev)
    with torch.no_grad():
        full = nb.render_rays(models, emb, r, 64, False, 0, 0, 64, 32768, True, test_time=True)
        cul = nb.render_rays_culled(models, emb, r, grid, 64, False, 64, True, test_time=True)
    live = cul["live_idx"].cpu().numpy()
    assert {i for i, (fam, _) in poisoned.items() if fam == "nonfinite"} <= set(live.tolist())
    a = {k: v.cpu().numpy() for k, v in cul.items() if k in full}
    b = {k: v.cpu().numpy() for k, v in full.items()}
    mm = dr.position_mismatch(a, b, live, live)
    print(f"\nculled: {len(live)} of {N} rays live; mismatches {mm}")
    assert not mm


NONFINITE = {"o NaN": (0, np.nan), "d +inf": (4, np.inf), "far +inf": (7, np.inf)}


NONFINITE = {"none": None, "o NaN": (0, np.nan), "d +inf": (4, np.inf), "far +inf": (7, np.inf)}


def _step_report(backward, params):
    """Run `backward`; -> (the step was reported through the device status, names of parameters whose gradient is
    finite everywhere)."""
    reported = False
    try:
        backward()
        torch.cuda.synchronize()
        reported = _lib.load().nerfb200_check_status() != 0
    except _lib.NerfB200Error:
        reported = True
    return reported, [n for n, p in params if p.grad is not None and torch.isfinite(p.grad).all()]


@pytest.mark.parametrize("kind", list(NONFINITE))
def test_nonfinite_ray_gradients(kind, dev, emb):
    """One non-finite ray in a 64-ray training batch: the reference's gradients are NaN everywhere.  The fused
    backward reports it (device status 103) instead of returning finite bias gradients beside NaN weight
    gradients; a batch without one ("none") is not reported and has finite gradients."""
    rays = orc.make_rays(64, 31)
    if NONFINITE[kind] is not None:
        col, val = NONFINITE[kind]
        rays[33, col] = val
    models = _models("random")
    tgt = torch.from_numpy(np.random.RandomState(3).uniform(0, 1, (64, 3)).astype(F32)).to(dev)
    out = nb.render_rays_loss(models, emb, torch.from_numpy(rays).to(dev), tgt, 64, False, 1.0, 0.0, 64, 32768, True)
    loss = float(out["loss"].detach())
    reported, finite = _step_report(out["loss"].backward,
                                    [(f"{i}.{n}", p) for i, m in enumerate(models) for n, p in m.named_parameters()])
    print(f"\n{kind}: render path loss {loss:.3g}, status reported {reported}, {len(finite)} of 48 parameters with "
          f"finite gradients")
    if kind == "none":
        assert not reported and len(finite) == 48
    else:
        assert reported, f"not reported; finite gradients: {finite}"


@pytest.mark.parametrize("kind", list(NONFINITE))
def test_nonfinite_point_gradients_nerf_forward(kind, dev, emb):
    """NeRF.forward with autograd_impl='fused' on 512 points of which one is non-finite (the first point of the
    poisoned ray of test_nonfinite_ray_gradients): reported through the device status, as the render path; a batch
    without one is not reported and has finite gradients."""
    rays = orc.make_rays(64, 31)
    m = _models("random")[1]
    m.autograd_impl = "fused"
    o, d = torch.from_numpy(rays[:, :3]).to(dev), torch.from_numpy(rays[:, 3:6]).to(dev)
    z = torch.linspace(2, 6, 8, device=dev)
    if NONFINITE[kind] is not None:
        col, val = NONFINITE[kind]
        if col < 3:
            o[33, col] = val
        elif col < 6:
            d[33, col - 3] = val
        else:
            z = z.expand(64, 8).clone()
            z[33] = float("nan") if np.isnan(val) else torch.linspace(2, 6, 8, device=dev) * val  # 2 inf .. 6 inf
    x = (o[:, None] + d[:, None] * (z if z.dim() == 2 else z[None]).unsqueeze(-1)).reshape(-1, 3)
    xe = torch.cat([emb[0](x), emb[1](d).repeat_interleave(8, 0)], -1)
    reported, finite = _step_report(lambda: m(xe).sum().backward(), list(m.named_parameters()))
    print(f"\n{kind}: NeRF.forward status reported {reported}, {len(finite)} of 24 parameters with finite gradients")
    if kind == "none":
        assert not reported and len(finite) == 24
    else:
        assert reported, f"not reported; finite gradients: {finite}"


# The first |x| of MAGS at which the kernel's sigma or rgb stops being finite where the fp32 oracle is finite, and
# the |x| up to which the encoding holds tt.BARS['enc'] at every point (it does not depend on the weights; past it,
# meeting the bar depends on the point), measured on an H100 80GB HBM3 at a 700 W power limit (DESIGN.md section 8).
# The fp16-operand oracle predicts the first to the same magnitude.
MAGS = [64.0 * 2.0 ** k for k in range(11)] + [1e5]
FIRST_NONFINITE = {"random": 1e5, "trained": 8192.0}
ENC_HOLDS_TO = 256.0


def _oracle_finite(w, rays, x, S, fp16):
    """Whether the fp32 oracle (with the big layers' operands rounded to fp16 when `fp16`) gives finite sigma and
    rgb at the device's own points x (n S, 3)."""
    from tools.fp16_error_model import rounded_operands
    X = np.concatenate([orc.embed(x, 10), np.repeat(orc.embed(rays[:, 3:6], 4), S, 0)], -1)
    with np.errstate(all="ignore"):
        if fp16:
            with rounded_operands("wa"):
                out = orc.nerf_forward(w, X)
        else:
            out = orc.nerf_forward(w, X)
    return np.isfinite(out).all(1)


@pytest.mark.parametrize("weights", ["random", "trained"])
def test_large_coordinates(weights, dev, emb):
    n, S, K = 32, 64, 64
    ws = cases.trained_weights() if weights == "trained" else cases.weights()
    c = dict(ts.DEFAULTS, n=n, S=S, K=K, perturb=0.0, white_back=True, weights=weights)
    lines, first, enc_ok, first16 = [], None, None, None
    for i, M in enumerate(MAGS):
        rs = np.random.RandomState(900 + i)
        rays = orc.make_rays(n, 900 + i)
        o = rs.randn(n, 3)
        rays[:, :3] = (o / np.linalg.norm(o, axis=1, keepdims=True) * M).astype(F32)
        run = ts.run_render(c, 900 + i, dev, emb, rays=rays, rnd={})
        enc, xmax = ts.enc_report(run)
        kern, f32, f16 = [], [], []
        for P in tt.layout(n, S, K):
            tape = tt.WorkspaceTape(run["raw"], P)
            z = tape.z()
            Sp = z.shape[1]
            x = (rays[:, None, :3] + (rays[:, None, 3:6] * z[:, :, None]).astype(F32)).astype(F32).reshape(-1, 3)
            kern.append(np.isfinite(tape.sigma().reshape(-1)) & np.isfinite(tape.rgb().reshape(-1, 3)).all(1))
            w = ws[len(f32)]
            f32.append(_oracle_finite(w, rays, x, Sp, False))
            f16.append(_oracle_finite(w, rays, x, Sp, True))
        kern, f32, f16 = (np.concatenate(a) for a in (kern, f32, f16))
        lost = int((~kern & f32).sum())
        lost16 = int((~f16 & f32).sum())
        lines.append(f"|x| {xmax:9.4g}: enc {enc:8.3g}, kernel non-finite where fp32 finite {lost:5d} of {kern.size}, "
                     f"fp16-operand oracle {lost16:5d}")
        if enc <= tt.BARS["enc"] and (enc_ok if enc_ok is not None else -1) == i - 1:
            enc_ok = i                      # every magnitude up to this one holds the bar
        if lost and first is None:
            first = M
        if lost16 and first16 is None:
            first16 = M
    print(f"\n[{weights} weights] encoding holds its bar to |x| = {MAGS[enc_ok] if enc_ok is not None else None}; "
          f"first non-finite sigma / rgb at |x| = {first} (fp16-operand oracle: {first16})\n" + "\n".join(lines))
    assert enc_ok is not None and MAGS[enc_ok] >= ENC_HOLDS_TO
    assert first == first16, "the kernel leaves the fp16 range where the fp16-operand oracle does not"
    assert first == FIRST_NONFINITE[weights]
