"""Empty-sample skipping over its whole shape envelope and at its edges (pytest -m gpu), against float64 and autograd.

1. Every (N_samples, N_importance) pair the C ABI accepts on a partial grid with unequal and reversed ranges, the
   options rotated over the pairs (MATRIX), through three entries: culling.render_samples(per_sample=True) (the
   evaluated set is the float64 rule of tests/sample_skip_ref.py, evaluated samples are the full-grid path's bit for
   bit, z_vals_fine is render_tape.z_fine of the path's own coarse weights, compositing meets
   render_tape.composite_errors), render_rays_train_skip with the MSE target (train_skip_ref.forward / backward and
   the autograd composition of test_gpu_train_skip) and render_rays(..., occupancy=) with a random loss on every
   output (train_skip_seed_ref.backward and the autograd composition of test_gpu_render_rays_grid).
2. Patterned rays whose coarse evaluated sets are chosen exactly (pattern_case): single samples at 0, 31, 32 and
   S - 1, whole mask words, all but one word, alternating and random samples; the fine passes of 96, 160 and 192
   samples (3, 5 and 6 samples per lane in the sparse backward) show lane chunks straddling a mask word.
3. Per-pass row totals at the compacted MLP's 128-row tiles (0, 1, 127, 128, 129, 255, and a coarse pass with no
   row whose fine pass has some), the last row carrying a large gradient: counting the padding rows of the last
   tile would fail the gradient bars.
4. Grid edges: rays in a lattice plane, on a lattice line and through lattice corners, the box boundary and one ulp
   outside, reversed ranges, N = 2, 33, 34 and the largest grid (N = 1625: cell indices above 2^31).
5. Batch sizes 1, 2, 3, 5 and 4 k +- 1 around the per-ray kernels' blocks of four warps.

The 48 gradients against the autograd compositions: with random weights they meet all of DESIGN.md section 2's
bars, under the MSE loss and under a loss with random positive weights on every output (parts 1, 3 and 5).  With
trained weights, and on the patterned rays, whose points lie up to 128 from the origin (positional encodings of up
to 2^9 * 128 radians), they meet its per-tensor bars (relative L2 < 8e-2, cosine > 0.997); the whole-gradient bar
(5e-3, set on 1000-ray batches of random weights near the origin) is not asserted there.  The plain step on the
same rays exceeds it too with the trained weights: 3.5e-3 - 2.5e-2 at these 40-80 rays (H100 80GB HBM3, 700 W).

Each comparison names its reference and shows that its bar rejects a planted defect in that reference: a mask
shifted by one sample, rows starting one row off, the passes swapped, the padding rows counted.  The fixture `dev`
prints the module's wall time and peak device memory with the card it ran on.
"""
import subprocess
import time

import numpy as np
import pytest
import torch

from oracle import nerf_oracle as orc
from tests import cases
from tests import render_tape as rt
from tests import sample_skip_ref as sk
from tests import test_gpu_render_rays_grid as rg
from tests import test_gpu_train_skip as ts
from tests import train_skip_ref as tr
from tests import train_skip_seed_ref as seed_ref

pytestmark = pytest.mark.gpu
F32 = np.float32

# (N_samples, N_importance): batch size and options.  Every value of every option runs with a 96-sample and with a
# 160-sample fine pass (tests/test_skip_envelope_ref.py); use_disp only with Blender rays (NDC rays start at near = 0).
MATRIX = {
    (32, 0): dict(n=45, kind="blender", use_disp=True, perturb=1.0, noise_std=1.0, white_back=False, rng="seed",
                  weights="random"),
    (32, 32): dict(n=56, kind="ndc", use_disp=False, perturb=1.0, noise_std=0.0, white_back=True, rng="tensors",
                   weights="trained"),
    (32, 64): dict(n=41, kind="blender", use_disp=True, perturb=1.0, noise_std=1.0, white_back=False, rng="seed",
                   weights="trained"),
    (32, 96): dict(n=63, kind="blender", use_disp=True, perturb=0.0, noise_std=0.0, white_back=True, rng="tensors",
                   weights="random"),
    (32, 128): dict(n=77, kind="blender", use_disp=True, perturb=1.0, noise_std=0.0, white_back=True, rng="tensors",
                    weights="trained"),
    (32, 160): dict(n=50, kind="ndc", use_disp=False, perturb=1.0, noise_std=1.0, white_back=False, rng="tensors",
                    weights="random"),
    (64, 0): dict(n=79, kind="ndc", use_disp=False, perturb=0.0, noise_std=1.0, white_back=True, rng="tensors",
                  weights="trained"),
    (64, 32): dict(n=64, kind="ndc", use_disp=False, perturb=0.0, noise_std=0.0, white_back=True, rng="tensors",
                   weights="random"),
    (64, 64): dict(n=72, kind="blender", use_disp=True, perturb=1.0, noise_std=0.0, white_back=False, rng="seed",
                   weights="random"),
    (64, 96): dict(n=48, kind="ndc", use_disp=False, perturb=0.0, noise_std=1.0, white_back=False, rng="seed",
                   weights="random"),
    (64, 128): dict(n=61, kind="blender", use_disp=False, perturb=1.0, noise_std=0.0, white_back=True, rng="seed",
                    weights="trained"),
    (128, 0): dict(n=40, kind="blender", use_disp=False, perturb=1.0, noise_std=0.0, white_back=False, rng="tensors",
                   weights="random"),
    (128, 32): dict(n=53, kind="blender", use_disp=False, perturb=1.0, noise_std=1.0, white_back=True, rng="seed",
                    weights="random"),
    (128, 64): dict(n=67, kind="ndc", use_disp=False, perturb=0.0, noise_std=1.0, white_back=True, rng="tensors",
                    weights="trained"),
}
OPTIONS = {"kind": {"blender", "ndc"}, "use_disp": {False, True}, "perturb": {0.0, 1.0}, "noise_std": {0.0, 1.0},
           "white_back": {False, True}, "rng": {"tensors", "seed"}, "weights": {"random", "trained"}}
PAIRS = list(MATRIX)
PAIR_IDS = [f"s{S}_k{K}" for S, K in PAIRS]
# the partial grid of part 1: unequal ranges, y reversed; cells drawn at random
PARTIAL = dict(N=11, ranges=((-2.0, 2.0), (2.0, -2.0), (-1.5, 2.5)), fill=0.3)


def cell_words(N, fill, seed):
    """Bits of a grid of N points per axis with each cell occupied with probability `fill`; the bits past the last
    cell of the last word are set, so that reading them would show."""
    M3 = (N - 1) ** 3
    occ = np.random.default_rng(seed).random(M3) < fill
    pad = np.ones((M3 + 31) // 32 * 32, bool)
    pad[:M3] = occ
    return np.packbits(pad.reshape(-1, 32)[:, ::-1], axis=1).view(">u4").astype(np.uint32).reshape(-1).view(np.int32)


# ------------------------------------------------------------------------------------------ patterned rays
PAT_M = 128              # cells per axis of the pattern grid over [0, 128]^3: one unit cell per unit of x


def coarse_patterns(S, seed=0):
    """name -> (S,) bool: the designed coarse evaluated sets of part 2."""
    i = np.arange(S)
    W = S // 32
    sets = {"empty": [], "full": i, "first": [0], "last": [S - 1], "only31": [31], "even": i[::2], "odd": i[1::2]}
    if S > 32:
        sets.update({"only32": [32], "31and32": [31, 32]})
    for w in range(W):
        sets[f"word{w}"] = i[32 * w:32 * w + 32]
        if W > 1:
            sets[f"all_but_word{w}"] = i[i // 32 != w]
    sets["random"] = i[np.random.default_rng(seed + S).random(S) < 0.5]
    out = {}
    for k, v in sets.items():
        m = np.zeros(S, bool)
        m[np.asarray(v, int)] = True
        out[k] = m
    return out


def pattern_case(masks, rows=None):
    """Rays and grid bits that give ray j the coarse evaluated set masks[j] (R, S): ray j runs along +x through the
    centre of cell row (cy, cz) = rows[j] (default (j % 128, j // 128)) from x = 0.5 over near = 0, far = S - 1, so at
    perturb = 0 its coarse sample i lies near x = i + 0.5, inside cell i alone; row j's bits are the pattern."""
    masks = np.asarray(masks, bool)
    R, S = masks.shape
    M = PAT_M
    j = np.arange(R)
    cy, cz = (j % M, j // M) if rows is None else (np.asarray(rows)[:, 0], np.asarray(rows)[:, 1])
    rays = np.zeros((R, 8), F32)
    rays[:, 0], rays[:, 1], rays[:, 2], rays[:, 3], rays[:, 7] = 0.5, cy + 0.5, cz + 0.5, 1.0, S - 1
    words = np.zeros((M ** 3 + 31) // 32, np.uint32)
    rr, ii = np.nonzero(masks)
    c = (cz[rr] * M + cy[rr]) * M + ii
    np.bitwise_or.at(words, c >> 5, (np.uint32(1) << (c & 31).astype(np.uint32)))
    return rays, words.view(np.int32)


PAT_RANGES = (0.0, float(PAT_M), 0.0, float(PAT_M), 0.0, float(PAT_M))
# pattern pairs: coarse passes of 1, 2 and 4 words; fine passes of 3, 5 and 6 samples per lane
PAT_PAIRS = [(32, 0), (64, 32), (32, 128), (128, 32), (64, 96), (64, 128), (128, 64)]


def straddles(ev, P):
    """Whether some ray of ev (R, S) has a lane chunk [l P, l P + P) across a mask-word boundary with evaluated
    samples on both sides of it and a skipped sample in it.  This is weaker than evaluated and skipped samples on
    each side: with P = 3 one side of a straddling chunk holds a single sample, so that cannot happen."""
    R, S = ev.shape
    for lane in range(32):
        a, b = lane * P, lane * P + P
        w = (b - 1) // 32 * 32
        if a >= w:
            continue
        lo, hi = ev[:, a:w], ev[:, w:b]
        if (lo.any(1) & hi.any(1) & ~ev[:, a:b].all(1)).any():
            return True
    return False


def counted_masks(total, n, S):
    """(n, S) masks of `total` rows in ray-major order whose last row is alone in its ray (sample 0 of the last ray
    with rows, transmittance 1): full rays, a remainder, then one ray with one sample."""
    m = np.zeros((n, S), bool)
    if total == 0:
        return m
    rest, r = total - 1, 0
    while rest > 0:
        c = min(S, rest)
        m[r, :c] = True
        rest -= c
        r += 1
    m[r, 0] = True
    assert r < n
    return m


def _nb():
    import nerf_pl_b200 as nb
    return nb


@pytest.fixture(scope="module")
def dev():
    d = torch.device("cuda:0")
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    name = torch.cuda.get_device_name(d)
    torch.cuda.reset_peak_memory_stats(d)
    t0 = time.perf_counter()
    yield d
    print(f"\nskip envelope on {name} (power limit {pl}): {time.perf_counter() - t0:.0f} s wall, peak device memory "
          f"{torch.cuda.max_memory_allocated(d) / 2 ** 30:.2f} GiB")


@pytest.fixture(autouse=True)
def _status_and_workspaces():
    yield
    torch.cuda.synchronize()
    assert _nb()._lib.load().nerfb200_check_status() == 0
    from nerf_pl_b200.train_skip import SkipTrainWorkspace
    SkipTrainWorkspace.clear()
    torch.cuda.empty_cache()


def _grid(words, N, ranges):
    rg_ = [tuple(ranges[2 * a:2 * a + 2]) for a in range(3)] if len(ranges) == 6 else ranges
    return _nb().OccupancyGrid(torch.from_numpy(np.asarray(words).view(np.int32)).cuda(), N, *rg_)


def _partial_grid(seed=3):
    N = PARTIAL["N"]
    return _grid(cell_words(N, PARTIAL["fill"], seed), N, PARTIAL["ranges"])


_TRAINED = []


def _models(kind):
    if kind == "random":
        return ts._models()
    if not _TRAINED:
        _TRAINED.extend(cases.trained_weights())
    ms = []
    for w in _TRAINED:
        m = _nb().NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        ms.append(m.cuda())
    return ms


def _passes(S, K):
    return (("coarse", S), ("fine", S + K))[:2 if K else 1]


def _carries(rows, ds_ref, dp_ref):
    """Whether the reference's gradient at the samples `rows` exceeds the per-row bar (a defect that drops them shows)."""
    return any(np.abs(r[rows]).max(initial=0.0) > tr.BWD_BAR * np.abs(r).max(initial=0.0) for r in (ds_ref, dp_ref))


def _shift_rows(ref, ev):
    """The reference's per-row values with the rows starting one row late (a row0 off by one)."""
    rows = ref[ev]
    return np.concatenate([np.zeros_like(rows[:1]), rows[:-1]], 0)


def check_rows(tag, ev, ds, dp, ref_bwd, two_passes):
    """The device's per-row d sigma / d rgb_pre of one pass (the rows of ev) against the float64 reference
    ref_bwd(ev_, swapped=False) -> (R, S), (R, S, 3) within BWD_BAR; where the reference has a gradient for a defect
    to move, each planted defect of the reference exceeds the bar: rows starting one row late, the mask shifted by
    one sample (where the samples it drops carry gradient) and, with two passes, the other pass's seed.  Returns the
    errors."""
    ds_ref, dp_ref = ref_bwd(ev)
    errs = tr.backward_errors(ds, dp, ev, ds_ref, dp_ref)
    assert max(errs) <= tr.BWD_BAR, (tag, errs)
    if ds.shape[0] < 2 or ev.all() or not _carries(ev, ds_ref, dp_ref):
        return errs
    shifted = ev & np.roll(ev, 1, 1)
    defects = {"row0 off by one": (_shift_rows(ds_ref, ev), _shift_rows(dp_ref, ev))}
    if _carries(ev & ~shifted, ds_ref, dp_ref):
        defects["mask shifted by one sample"] = tuple(r[ev] for r in ref_bwd(shifted))
    if two_passes:
        defects["passes swapped"] = tuple(r[ev] for r in ref_bwd(ev, swapped=True))
    for what, (bds, bdp) in defects.items():
        bad = tr.backward_errors(bds, bdp, ev, ds_ref, dp_ref)
        assert max(bad) > tr.BWD_BAR, (tag, what, bad)
    return errs


# ------------------------------------------------------------------------------------------ the three entries
def check_render(models, rays, grid, S, K, use_disp, white_back, tag, frac=None):
    """culling.render_samples(per_sample=True) at perturb = 0 against the float64 rule on z_base's depths, the
    full-grid path, render_tape.z_fine and render_tape.composite_errors.  Returns the worst compositing metrics and the render."""
    nb = _nb()
    full = _grid(np.full(1, -1, np.int32), 2, ((-1e4, 1e4),) * 3)
    got = nb.culling.render_samples(models, rays, grid, S, use_disp, K, white_back, False, extras=True, per_sample=True)
    ref = nb.culling.render_samples(models, rays, full, S, use_disp, K, white_back, False, extras=True, per_sample=True)
    rn, words = rays.cpu().numpy(), grid.bits.cpu().numpy()
    n = rn.shape[0]
    zc = sk.z_base(rn, S, use_disp)
    ev_c = sk.mask_bits(got["mask_coarse"].cpu().numpy(), S)
    want_c = sk.evaluated(rn, zc, words, grid.N, grid.ranges)
    assert np.array_equal(ev_c, want_c), (tag, "coarse set")
    if want_c.any() and not want_c.all():
        assert not np.array_equal(np.roll(want_c, 1, 1), ev_c)          # planted: the mask shifted by one sample
    if frac is not None:
        assert frac[0] < ev_c.mean() < frac[1], (tag, ev_c.mean())
    assert sk.mask_bits(ref["mask_coarse"].cpu().numpy(), S).all()
    sc, rc = got["samples_coarse"].cpu().numpy(), ref["samples_coarse"].cpu().numpy()
    assert np.array_equal(sc[ev_c].view(np.int32), rc[ev_c].view(np.int32)) and not sc[~ev_c].any(), tag
    wc = got["weights_coarse"].cpu().numpy()
    assert not wc[~ev_c].any(), tag
    live = [int(ev_c.sum()), 0]
    d = rn[:, 3:6]
    worst = {}
    comps = [("coarse", sc, zc, wc, ev_c)]
    if K:
        zf = got["z_vals_fine"].cpu().numpy()
        ev_f = sk.mask_bits(got["mask_fine"].cpu().numpy(), S + K)
        assert np.array_equal(ev_f, sk.evaluated(rn, zf, words, grid.N, grid.ranges)), (tag, "fine set")
        live[1] = int(ev_f.sum())
        want_z, _, _ = rt.z_fine(wc, zc, rt.fine_uniforms(n, K, 0.0))
        assert np.array_equal(zf, want_z), (tag, "z_vals_fine")
        sf, wf = got["samples_fine"].cpu().numpy(), got["weights_fine"].cpu().numpy()
        assert not sf[~ev_f].any() and not wf[~ev_f].any(), tag
        # evaluated fine samples at depths the full-grid path also sampled are its values bit for bit
        same = (zf == ref["z_vals_fine"].cpu().numpy()) & ev_f
        rf = ref["samples_fine"].cpu().numpy()
        assert np.array_equal(sf[same].view(np.int32), rf[same].view(np.int32)), tag
        comps.append(("fine", sf, zf, wf, ev_f))
    assert got["live_samples"] == tuple(live), tag
    for name, s_all, z_, w_, ev in comps:
        out = [got[f"{k}_{name}"].cpu().numpy() for k in ("rgb", "depth", "opacity")]

        def errs(ev_=ev):
            return rt.composite_errors(np.where(ev_, s_all[..., 3], 0), s_all[..., :3], z_, d, None, 0.0, white_back,
                                       w_, *out)
        e = errs()
        assert not rt.composite_violations(e), (tag, name, e)
        worst.update({f"{name}.{k}": v for k, v in e.items()})
        if (w_[ev & ~np.roll(ev, 1, 1)] > 1e-3).any():   # planted: sigma of a mask shifted by one sample
            assert rt.composite_violations(errs(ev & np.roll(ev, 1, 1))), (tag, name)
    return worst, got


def _train_inputs(n, S, K, o, seed):
    rnd = ts._randoms(n, S, K, seed)
    kernel = o["rng"] == "seed"
    per = o["perturb"] > 0 and not kernel
    pr = rnd["perturb_rand"] if per else None
    ur = rnd.get("u_rand") if per else None
    nc = rnd["noise_coarse"] if o["noise_std"] else None
    nf = rnd.get("noise_fine") if o["noise_std"] else None
    noise = {k: v for k, v in (("noise_coarse", nc), ("noise_fine", nf)) if v is not None}
    return (pr, nc, ur, nf), (4000 + seed if kernel and o["perturb"] > 0 else None), noise


def _rays(kind, n, seed):
    if kind == "ndc":
        return torch.from_numpy(orc.make_rays(n, seed, "ndc")).cuda()
    return ts._rays(kind, n, seed)


def grad_errors(got, ref):
    """DESIGN section 2's measures of the gradients `got` against `ref`: (whole-gradient relative L2, worst
    per-tensor relative L2, lowest per-tensor cosine)."""
    num = sum(float(((got[k] - r) ** 2).sum()) for k, r in ref.items())
    den = sum(float((r ** 2).sum()) for r in ref.values())
    rel = [np.linalg.norm(got[k] - r) / max(np.linalg.norm(r), 1e-30) for k, r in ref.items()]
    cos = [float((got[k] * r).sum() / max(np.linalg.norm(got[k]) * np.linalg.norm(r), 1e-30)) for k, r in ref.items()]
    return (num / den) ** 0.5, max(rel), min(cos)


def _grads_close(gg, ref, live, K, tag, bars="all"):
    """A network without evaluated rows (or whose reference gradient is 0) has exact-zero gradients; the others meet
    DESIGN section 2's bars: all of them (bars="all"), or the per-tensor ones, relative L2 < 8e-2 and cosine > 0.997
    (bars="tensor").  Returns grad_errors of the others."""
    zero = [live[ps] == 0 or not any(v.any() for k, v in ref.items() if k.startswith(f"{ps}."))
            for ps in range(2 if K else 1)]
    for k, v in gg.items():
        if zero[int(k[0])]:              # no row, or rows whose every reference gradient is 0
            assert not v.any() and not ref[k].any(), (tag, k)
    keep = {k: v for k, v in ref.items() if not zero[int(k[0])]}
    if not keep:
        return 0.0, 0.0, 1.0
    if bars == "all":
        ts._grad_bars(gg, keep)
    e = grad_errors(gg, keep)
    if bars == "tensor":
        assert e[1] < 8e-2 and e[2] > 0.997, (tag, e)
    return e


def check_train(models, rays, rgbs, grid, S, K, o, seed, tag, frac=None, copies_fail=False, bars="all"):
    """render_rays_train_skip with the MSE target and extras: evaluated sets against the float64 rule on the device's
    own depths, the forward against train_skip_ref.forward, the per-row d sigma / d rgb_pre against
    train_skip_ref.backward (BWD_BAR), the 24 / 48 gradients against test_gpu_train_skip's autograd composition.
    Returns the worst errors."""
    from nerf_pl_b200.train_skip import render_rays_train_skip
    n = rays.shape[0]
    randoms, rng_seed, noise = _train_inputs(n, S, K, o, seed)
    for m in models:
        m.zero_grad(set_to_none=True)
    got = render_rays_train_skip(models, rays, S, o["use_disp"], o["perturb"], o["noise_std"], K, o["white_back"],
                                 *randoms, rgbs, grid, rng_seed=rng_seed, extras=True)
    got["loss"].backward()
    gg = rg._grads(models, K)
    rn, words, tn = rays.cpu().numpy(), grid.bits.cpu().numpy(), rgbs.cpu().numpy()
    worst = {}
    live = []
    for ps, (name, Sp) in enumerate(_passes(S, K)):
        z = got["z_vals_" + name].cpu().numpy()
        ev = sk.mask_bits(got["mask_" + name].cpu().numpy(), Sp)
        assert np.array_equal(ev, sk.evaluated(rn, z, words, grid.N, grid.ranges)), (tag, name, "set")
        if ps == 0 and frac is not None:
            assert frac[0] < ev.mean() < frac[1], (tag, ev.mean())
        live.append(int(ev.sum()))
        smp = got["samples_" + name].cpu().numpy()
        w = got["weights_" + name].cpu().numpy()
        assert not smp[~ev].any() and not w[~ev].any(), (tag, name)
        nz = noise["noise_" + name].cpu().numpy() if o["noise_std"] else None
        outs = {k: got[f"{k}_{name}"].detach().cpu().numpy() for k in ("rgb", "depth", "opacity")}
        tr.assert_close(tr.forward(z, smp, ev, rn, nz, o["noise_std"], o["white_back"]), outs, w, ref_weights=True)
        rows = live[-1]
        ds = got["dsigma_" + name][:rows].cpu().numpy()
        dp = got["dprergb_" + name][:rows].cpu().numpy()
        other = "fine" if ps == 0 else "coarse"

        def ref_bwd(ev_, swapped=False, z=z, smp=smp, nz=nz, out=name, other=other):
            rgb_out = got["rgb_" + (other if swapped else out)].detach().cpu().numpy()
            return tr.backward(z, smp[..., 3], smp[..., :3], ev_, rn[:, 3:6], nz, o["noise_std"], o["white_back"],
                               rgb_out, tn, n)
        worst[f"{name}.dsigma"], worst[f"{name}.dprergb"] = check_rows(f"{tag} {name}", ev, ds, dp, ref_bwd, K > 0)
    ref = ts._autograd_reference(models, rays, rgbs, got, S, K, o["noise_std"], o["white_back"], noise)
    worst["grad.total"], worst["grad.worst_tensor"], worst["grad.min_cos"] = _grads_close(gg, ref, live, K, tag, bars)
    if copies_fail:       # planted: the padding rows of the last coarse tile counted in the weight gradients
        copies = -live[0] % 128
        bad = ts._autograd_reference(models, rays, rgbs, got, S, K, o["noise_std"], o["white_back"], noise,
                                     copies=(copies, 0))
        with pytest.raises(AssertionError):
            ts._grad_bars(gg, bad)
    return worst, tuple(live)


def check_seed(models, rays, grid, S, K, o, seed, tag, frac=None, copies_fail=False, weights=None, bars="all"):
    """render_rays(..., occupancy=) with sum_k <w_k, out_k>, then the same step through render_rays_train_skip(
    target=None, extras=True): the same outputs bit for bit; per-row gradients against
    train_skip_seed_ref.backward (BWD_BAR), both paths' 24 / 48 gradients against test_gpu_render_rays_grid's
    autograd composition."""
    from nerf_pl_b200.train_skip import render_rays_train_skip
    n = rays.shape[0]
    randoms, rng_seed, noise = _train_inputs(n, S, K, o, seed)
    w = rg._weights(n, K, seed) if weights is None else weights
    rr = dict(zip(("perturb_rand", "noise_coarse", "u_rand", "noise_fine"), randoms))
    rr = {k: v for k, v in rr.items() if v is not None}
    if rng_seed is not None:
        rr["seed"] = rng_seed
    for m in models:
        m.zero_grad(set_to_none=True)
    res = _nb().render_rays(models, ts._emb(), rays, S, o["use_disp"], o["perturb"], o["noise_std"], K, 32768,
                            o["white_back"], randoms=rr, occupancy=grid)
    rg._wloss(res, w).backward()
    g_rr = rg._grads(models, K)
    for m in models:
        m.zero_grad(set_to_none=True)
    got = render_rays_train_skip(models, rays, S, o["use_disp"], o["perturb"], o["noise_std"], K, o["white_back"],
                                 *randoms, None, grid, rng_seed=rng_seed, extras=True)
    rg._wloss(got, w).backward()
    gg = rg._grads(models, K)
    for k in res:
        assert ts._same(res[k].detach(), got[k].detach()), (tag, k)
    rn, words = rays.cpu().numpy(), grid.bits.cpu().numpy()
    wn = {k: v.cpu().numpy() for k, v in w.items()}
    worst, live = {}, []
    for ps, (name, Sp) in enumerate(_passes(S, K)):
        z = got["z_vals_" + name].cpu().numpy()
        ev = sk.mask_bits(got["mask_" + name].cpu().numpy(), Sp)
        assert np.array_equal(ev, sk.evaluated(rn, z, words, grid.N, grid.ranges)), (tag, name, "set")
        if ps == 0 and frac is not None:
            assert frac[0] < ev.mean() < frac[1], (tag, ev.mean())
        live.append(int(ev.sum()))
        smp = got["samples_" + name].cpu().numpy()
        nz = noise["noise_" + name].cpu().numpy() if o["noise_std"] else None
        rows = live[-1]
        ds = got["dsigma_" + name][:rows].cpu().numpy()
        dp = got["dprergb_" + name][:rows].cpu().numpy()
        other = "fine" if ps == 0 else "coarse"

        def ref_bwd(ev_, swapped=False, z=z, smp=smp, nz=nz, seeds=name, other=other):
            k = other if swapped else seeds
            return seed_ref.backward(z, smp[..., 3], smp[..., :3], ev_, rn[:, 3:6], nz, o["noise_std"],
                                     o["white_back"], wn["rgb_" + k], wn["depth_" + k], wn["opacity_" + k])
        worst[f"{name}.dsigma"], worst[f"{name}.dprergb"] = check_rows(f"{tag} {name}", ev, ds, dp, ref_bwd, K > 0)
    ref = rg._autograd_reference(models, rays, got, S, K, o["noise_std"], o["white_back"], noise, w)
    worst["grad.total"], worst["grad.worst_tensor"], worst["grad.min_cos"] = _grads_close(gg, ref, live, K, tag, bars)
    worst["render_rays.grad.total"] = _grads_close(g_rr, ref, live, K, tag, bars)[0]
    if copies_fail:
        bad = rg._autograd_reference(models, rays, got, S, K, o["noise_std"], o["white_back"], noise, w,
                                     copies=(-live[0] % 128, 0))
        with pytest.raises(AssertionError):
            ts._grad_bars(gg, bad)
    return worst, tuple(live)


def _positive_weights(n, K, seed):
    """rg._weights with every weight made positive: a random loss on every output whose weight-gradient sums do not
    cancel (with weights of random sign the rows' contributions cancel, and relative errors of the sums are no
    longer those DESIGN section 2's bars were set on)."""
    return {k: v.abs() for k, v in rg._weights(n, K, seed).items()}


def _fmt(d):
    return " ".join(f"{k} {v:.2e}" for k, v in d.items())


# ------------------------------------------------------------------------------------------ 1. the pair matrix
@pytest.mark.parametrize("S,K", PAIRS, ids=PAIR_IDS)
def test_pair_matrix_render(S, K, dev):
    c = MATRIX[(S, K)]
    seed = 500 + PAIRS.index((S, K))
    rays = _rays(c["kind"], c["n"], seed)
    worst, _ = check_render(_models(c["weights"]), rays, _partial_grid(), S, K, c["use_disp"], c["white_back"],
                            f"s{S}_k{K}", frac=(0.05, 0.95))
    print(f"\n[render s{S}_k{K}] {c}\n  worst (units of the render_tape bars): {_fmt(worst)}")


@pytest.mark.parametrize("S,K", PAIRS, ids=PAIR_IDS)
def test_pair_matrix_train(S, K, dev):
    c = MATRIX[(S, K)]
    seed = 520 + PAIRS.index((S, K))
    rays = _rays(c["kind"], c["n"], seed)
    rgbs = torch.rand(c["n"], 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed))
    worst, live = check_train(_models(c["weights"]), rays, rgbs, _partial_grid(), S, K, c, seed, f"s{S}_k{K}",
                              frac=(0.05, 0.95), bars="all" if c["weights"] == "random" else "tensor")
    print(f"\n[train s{S}_k{K}] {c} rows {live}\n  worst: {_fmt(worst)}")


@pytest.mark.parametrize("S,K", PAIRS, ids=PAIR_IDS)
def test_pair_matrix_general_seed(S, K, dev):
    c = MATRIX[(S, K)]
    seed = 540 + PAIRS.index((S, K))
    rays = _rays(c["kind"], c["n"], seed)
    worst, live = check_seed(_models(c["weights"]), rays, _partial_grid(), S, K, c, seed, f"s{S}_k{K}",
                             frac=(0.05, 0.95), bars="all" if c["weights"] == "random" else "tensor",
                             weights=_positive_weights(c["n"], K, seed))
    print(f"\n[general seed s{S}_k{K}] {c} rows {live}\n  worst: {_fmt(worst)}")


# ------------------------------------------------------------------------------------------ 2. patterned rays
def _pattern_rays(S, seed):
    pats = coarse_patterns(S, seed)
    masks = np.stack(list(pats.values()) * 2)            # each pattern twice: on two rows of cells
    rays, words = pattern_case(masks)
    return pats, masks, torch.from_numpy(rays).cuda(), _grid(words, PAT_M + 1, PAT_RANGES)


PAT_OPTS = dict(kind="pattern", use_disp=False, perturb=0.0, noise_std=1.0, white_back=False, rng="tensors")


@pytest.mark.parametrize("S,K", PAT_PAIRS, ids=[f"s{S}_k{K}" for S, K in PAT_PAIRS])
def test_patterned_rays(S, K, dev):
    seed = 600 + PAT_PAIRS.index((S, K))
    pats, masks, rays, grid = _pattern_rays(S, seed)
    models = ts._models()
    n = rays.shape[0]
    render, got = check_render(models, rays, grid, S, K, False, True, f"pattern s{S}_k{K}")
    assert np.array_equal(sk.mask_bits(got["mask_coarse"].cpu().numpy(), S), masks)      # the designed sets
    rgbs = torch.rand(n, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed))
    train, live = check_train(models, rays, rgbs, grid, S, K, PAT_OPTS, seed, f"pattern s{S}_k{K}", bars="tensor")
    assert live[0] == int(masks.sum())
    gen, _ = check_seed(models, rays, grid, S, K, dict(PAT_OPTS, noise_std=0.0, white_back=True), seed,
                        f"pattern s{S}_k{K}", weights=_positive_weights(n, K, seed), bars="tensor")
    if K:
        P = (S + K) // 32
        ev_f = sk.mask_bits(got["mask_fine"].cpu().numpy(), S + K)
        if P in (3, 5, 6):
            assert straddles(ev_f, P), P
    print(f"\n[patterns s{S}_k{K}] {len(pats)} patterns, rows {live}\n  render {_fmt(render)}\n  train {_fmt(train)}"
          f"\n  general seed {_fmt(gen)}")


# ------------------------------------------------------------------------------------------ 3. row totals
TOTALS = [0, 1, 127, 128, 129, 255]


def _dense_row(model):
    """The cy of the cell row (cy, 64) of the pattern grid where the network's sigma at x = 0.5 (sample 0 of a
    pattern ray) is largest: a lone row there has a weight well above 0."""
    nb = _nb()
    n = PAT_M
    xyz = torch.zeros(n, 3, device="cuda")
    xyz[:, 0], xyz[:, 1], xyz[:, 2] = 0.5, torch.arange(n, device="cuda") + 0.5, 64.5
    d = torch.zeros(n, 3, device="cuda")
    d[:, 0] = 1.0
    with torch.no_grad():
        sigma = model(torch.cat([nb.Embedding(3, 10)(xyz), nb.Embedding(3, 4)(d)], -1))[:, 3]
    assert float(sigma.max()) > 1.0
    return int(sigma.argmax())


@pytest.mark.parametrize("K", [0, 64])
@pytest.mark.parametrize("total", TOTALS)
def test_row_totals_at_tile_edges(total, K, dev):
    """Coarse rows of counted rays (64 samples, eager path); the last row is the first sample of a ray of its own,
    whose target (and upstream gradient) is 40 times the others': counting the 128 - total % 128 padding copies of
    it fails the gradient bars."""
    S, n = 64, 6
    masks = counted_masks(total, n, S)
    last = int(np.nonzero(masks.any(1))[0][-1]) if total else 0
    models = ts._models()
    rows = np.stack([np.arange(n), np.zeros(n, int)], 1)
    rows[last] = (_dense_row(models[0]), 64)
    rays_np, words = pattern_case(masks, rows)
    rays = torch.from_numpy(rays_np).cuda()
    grid = _grid(words, PAT_M + 1, PAT_RANGES)
    check_render(models, rays, grid, S, K, False, False, f"total {total}")
    rgbs = torch.rand(n, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(total))
    rgbs[last] = 40.0
    o = dict(PAT_OPTS, noise_std=0.0)
    padded = total % 128 != 0
    train, live = check_train(models, rays, rgbs, grid, S, K, o, 700 + total, f"total {total}", copies_fail=padded)
    assert live[0] == total
    w = rg._weights(n, K, 710 + total)
    for k in w:
        w[k][last] = w[k][last] * 40.0
    gen, _ = check_seed(models, rays, grid, S, K, o, 720 + total, f"total {total}", copies_fail=padded, weights=w)
    print(f"\n[rows {live}] train {_fmt(train)}\n  general seed {_fmt(gen)}")


def test_coarse_pass_without_rows_fine_pass_with_some(dev):
    """test_gpu_captured_skip's gap at the origin: coarse samples at x = i miss the cell x in [0.3, 0.7], the fine
    sample at depth 0.5 lies in it."""
    from tests import test_gpu_captured_skip as tc
    n, S, K = 40, 64, 64
    rays = torch.zeros(n, 8, device="cuda")
    rays[:, 3], rays[:, 7] = 1.0, 63.0
    grid = tc._box_grid(0.3, 0.7)
    models = ts._models()
    rgbs = torch.rand(n, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    check_render(models, rays, grid, S, K, False, True, "gap")
    train, live = check_train(models, rays, rgbs, grid, S, K, PAT_OPTS, 730, "gap")
    assert live[0] == 0 and live[1] > 0, live
    gen, live2 = check_seed(models, rays, grid, S, K, PAT_OPTS, 731, "gap", weights=_positive_weights(n, K, 731))
    assert live2 == live
    print(f"\n[gap rows {live}] train {_fmt(train)}\n  general seed {_fmt(gen)}")


# ------------------------------------------------------------------------------------------ 4. grid edges
def lattice_case(kind, n, seed, M=64):
    """Rays along +x whose every sample lies on a lattice face ("plane": y on a lattice plane), edge ("line": y and z
    on lattice planes) or corner ("corner": as "line" from x = 0, where the coarse depths are whole numbers), and
    bits in which of the 2 or 4 cells around the ray exactly one column is occupied, at cells no two of which are
    neighbours along x.  Returns (rays, words) for a grid of M + 1 points over [0, M]^3."""
    rng = np.random.default_rng(seed)
    rays = np.zeros((n, 8), F32)
    words = np.zeros((M ** 3 + 31) // 32, np.uint32)
    for j in range(n):
        a, b = 2 + 2 * (j % 30), 2 + 2 * (j // 30)
        y = float(a)
        z = float(b) if kind != "plane" else b + 0.5
        rays[j] = (0.0 if kind == "corner" else 0.5, y, z, 1.0, 0.0, 0.0, 0.0, 31.0)
        cy = a - rng.integers(2)
        cz = (b - rng.integers(2)) if kind != "plane" else b
        xs = np.nonzero(rng.random(M) < 0.5)[0]
        xs = xs[np.concatenate([[True], np.diff(xs) > 1])]
        c = (cz * M + cy) * M + xs
        np.bitwise_or.at(words, c >> 5, np.uint32(1) << (c & 31).astype(np.uint32))
    return rays, words.view(np.int32)


def _render_sets(rays_np, words, N, ranges, S=32, K=64):
    """render_samples' coarse and fine sets and fine depths, with the float64 rule on them."""
    nb = _nb()
    grid = _grid(words, N, ranges)
    rays = torch.from_numpy(np.ascontiguousarray(rays_np, F32)).cuda()
    got = nb.culling.render_samples(ts._models(), rays, grid, S, False, K, False, False, extras=True, per_sample=True)
    ev_c = sk.mask_bits(got["mask_coarse"].cpu().numpy(), S)
    zf = got["z_vals_fine"].cpu().numpy()
    ev_f = sk.mask_bits(got["mask_fine"].cpu().numpy(), S + K)
    return ev_c, ev_f, zf


def _cull_keeps_evaluated(rays_np, words, N, ranges, ev_c, ev_f):
    """nb.cull_rays keeps every ray with an evaluated sample (the cell walk is a superset of the lookup)."""
    flag = _nb().cull_rays(torch.from_numpy(np.ascontiguousarray(rays_np, F32)).cuda(), _grid(words, N, ranges),
                           return_flag=True)[2].cpu().numpy().astype(bool)
    lost = (ev_c.any(1) | ev_f.any(1)) & ~flag
    assert not lost.any(), np.nonzero(lost)[0]


def _rule_sets(rays_np, words, N, ranges, zf, S=32):
    return (sk.evaluated(rays_np, sk.z_base(rays_np, S), words, N, ranges),
            sk.evaluated(rays_np, zf, words, N, ranges))


@pytest.mark.parametrize("kind", ["plane", "line", "corner"])
def test_lattice_faces_edges_and_corners(kind, dev):
    M = 64
    rays, words = lattice_case(kind, 60, 800 + len(kind), M)
    box = (0.0, float(M)) * 3
    ev_c, ev_f, zf = _render_sets(rays, words, M + 1, box)
    want_c, want_f = _rule_sets(rays, words, M + 1, box, zf)
    assert np.array_equal(ev_c, want_c) and np.array_equal(ev_f, want_f), kind
    assert 0.2 < ev_c.mean() < 0.95, ev_c.mean()
    if kind == "corner":      # most coarse samples are at lattice corners, and those are evaluated when one of
        z = sk.z_base(rays, 32)                                        # the two occupied cells along x is
        assert (z == np.round(z)).mean() > 0.8
    # the same rays and bits with every range reversed and the rays mirrored: the float64 rule, and the same sets
    mirror = rays.copy()
    mirror[:, 0:3] = F32(M) - rays[:, 0:3]
    mirror[:, 3:6] = -rays[:, 3:6]
    rev = (float(M), 0.0) * 3
    rc, rf, rzf = _render_sets(mirror, words, M + 1, rev)
    if kind != "corner":    # M - x rounds a corner sample's x = i + ulp onto the corner itself
        assert np.array_equal(rc, ev_c)
    mc, mf = _rule_sets(mirror, words, M + 1, rev, rzf)
    assert np.array_equal(rc, mc) and np.array_equal(rf, mf)
    _cull_keeps_evaluated(rays, words, M + 1, box, ev_c, ev_f)
    _cull_keeps_evaluated(mirror, words, M + 1, rev, rc, rf)
    print(f"\n[{kind}] evaluated coarse {ev_c.mean():.3f} fine {ev_f.mean():.3f}")


def test_box_boundary(dev):
    """Rays along +x with y or z at exactly 0 or M, or one ulp outside; rays along +y with x there: on the box they
    are evaluated at every sample inside the box (every boundary cell is occupied), one ulp outside at none."""
    M = 32
    N = M + 1
    occ = np.zeros((M, M, M), bool)           # [cz, cy, cx]
    occ[0, :, :] = occ[-1, :, :] = occ[:, 0, :] = occ[:, -1, :] = occ[:, :, 0] = occ[:, :, -1] = True
    pad = np.zeros(((M ** 3 + 31) // 32) * 32, bool)
    pad[:M ** 3] = occ.reshape(-1)
    words = np.packbits(pad.reshape(-1, 32)[:, ::-1], axis=1).view(">u4").astype(np.uint32).reshape(-1).view(np.int32)
    below, above = np.nextafter(F32(0), F32(-1)), np.nextafter(F32(M), F32(2 * M))
    edges = [(F32(0), True), (F32(M), True), (below, False), (above, False)]
    rays, want_all = [], []
    for v, on in edges:
        for axis in (1, 2):                    # along x, y or z on the edge value
            r = np.array([0.0, 5.5, 7.5, 1.0, 0.0, 0.0, 0.0, 31.0], F32)
            r[axis] = v
            rays.append(r)
            want_all.append(on)
        r = np.array([5.5, 0.0, 9.5, 0.0, 1.0, 0.0, 0.0, 31.0], F32)    # along y, x on the edge value
        r[0] = v
        rays.append(r)
        want_all.append(on)
    rays = np.stack(rays)
    box = (0.0, float(M)) * 3
    ev_c, ev_f, zf = _render_sets(rays, words, N, box)
    want_c, want_f = _rule_sets(rays, words, N, box, zf)
    assert np.array_equal(ev_c, want_c) and np.array_equal(ev_f, want_f)
    want_all = np.array(want_all)
    assert ev_c[want_all].all() and not ev_c[~want_all].any()
    _cull_keeps_evaluated(rays, words, N, box, ev_c, ev_f)


@pytest.mark.parametrize("N", [2, 33, 34])
def test_grid_sizes(N, dev):
    """(N - 1)^3 = 1, 32768 and 35937 cells; bits past the last cell set."""
    ranges = ((-2.0, 2.0), (2.0, -2.0), (-1.5, 2.5))
    words = cell_words(N, 0.3 if N > 2 else 1.0, 900 + N)
    rays_np = ts._rays("blender", 90, 900 + N).cpu().numpy()
    flat = (-2.0, 2.0, 2.0, -2.0, -1.5, 2.5)
    ev_c, ev_f, zf = _render_sets(rays_np, words, N, ranges)
    want_c, want_f = _rule_sets(rays_np, words, N, flat, zf)
    assert np.array_equal(ev_c, want_c) and np.array_equal(ev_f, want_f), N
    assert ev_c.any() and not ev_c.all()


def test_largest_grid(dev):
    """N = 1625 over (0, 1624)^3 (scale exactly 1): 4.28e9 cells, the occupied ones near the far corner at indices
    above 2^31 (a signed 32-bit cell index would wrap); the expectation is the float64 rule on the set of occupied
    cells."""
    nb = _nb()
    N, M = 1625, 1624
    occupied = np.array([(1620, 1623, 1623), (1622, 1623, 1623), (1623, 1623, 1623), (1610, 1621, 1622),
                         (1611, 1621, 1622), (1623, 1600, 1623)], np.int64)          # (cx, cy, cz)
    cells = (occupied[:, 2] * M + occupied[:, 1]) * M + occupied[:, 0]
    assert (cells >= 1 << 31).all()
    bits = torch.zeros((M ** 3 + 31) // 32, dtype=torch.int32, device="cuda")
    for c in np.unique(cells >> 5):
        word = 0
        for b in cells[(cells >> 5) == c] & 31:
            word |= 1 << int(b)
        bits[int(c)] = torch.tensor(np.uint32(word).view(np.int32))
    grid = nb.OccupancyGrid(bits, N, (0.0, float(M)), (0.0, float(M)), (0.0, float(M)))
    rows = [(1623.5, 1623.5), (1621.5, 1622.5), (1600.5, 1623.5), (1623.0, 1623.5), (1622.5, 1622.5), (1624.0, 1624.0)]
    rays = np.zeros((len(rows), 8), F32)
    for j, (y, z) in enumerate(rows):
        rays[j] = (1600.5, y, z, 1.0, 0.0, 0.0, 0.0, 31.0)
    t = torch.from_numpy(rays).cuda()
    got = nb.culling.render_samples(ts._models(), t, grid, 32, False, 64, False, False, extras=True, per_sample=True)
    occ = set(cells.tolist())
    for name, S, z in (("coarse", 32, sk.z_base(rays, 32)), ("fine", 96, got["z_vals_fine"].cpu().numpy())):
        ev = sk.mask_bits(got["mask_" + name].cpu().numpy(), S)
        touched = sk.touched_cells(sk.sample_points(rays, z), N, (0.0, float(M)) * 3)
        want = np.isin(touched, list(occ)).any(1).reshape(ev.shape)
        assert np.array_equal(ev, want), name
        if name == "coarse":
            assert want.any() and not want.all() and want[:, -8:].sum() == 0        # x > 1624: outside the box
    del got, grid, bits


# ------------------------------------------------------------------------------------------ 5. batch edges
BATCHES = [1, 2, 3, 5, 7, 9, 127, 129]


@pytest.mark.parametrize("n", BATCHES)
def test_batch_edges(n, dev):
    """The MSE seed divides by 3 n; blocks of four rays per launch."""
    S, K = 64, 64
    o = dict(kind="blender", use_disp=False, perturb=1.0, noise_std=1.0, white_back=True, rng="tensors")
    rays = ts._rays("blender", n, 1000 + n)
    rgbs = torch.rand(n, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(n))
    grid = _grid(cell_words(PARTIAL["N"], 0.5, 7), PARTIAL["N"], PARTIAL["ranges"])
    worst, live = check_train(ts._models(), rays, rgbs, grid, S, K, o, 1000 + n, f"n {n}")
    assert live[0] > 0
    print(f"\n[n {n}] rows {live} worst: {_fmt(worst)}")
