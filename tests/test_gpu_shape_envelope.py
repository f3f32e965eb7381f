"""The renderer and the training step over their whole shape envelope (pytest -m gpu).

1. Every (N_samples, N_importance) pair the C ABI accepts (capi.cu check_render_shapes: N_samples in {32, 64, 128},
   N_importance a multiple of 32, at most 192 samples in all), with the other options rotated over the pairs:
   the forward stages of test_gpu_render_stages (bitwise mode invariance and resampling, compositing, encoding,
   the fused loss) and the backward stages of test_gpu_train_stages (every stage and every .grad element), each
   within its existing bars.
2. Training-step batch sizes at the schedules' edges: 1 to 5 rays (a lone ray in the last group of two, head_bwd
   blocks of four rays straddling the pass boundary), 2 rays per SM and one either side (the render kernel's CTA
   ranges), 4 per SM + 3, and 4096 / 8192-ray batches (the chain kernel's probe then sees 1-2 % of the tiles).
3. The render kernel's split of the rays into per-CTA ranges (nerfb200_render_args.max_ctas): inference outputs,
   the training workspace and the 48 gradients are bitwise the same for every CTA count, down to one CTA walking
   all 512 groups of a 1024-ray batch.

The fixture `dev` prints the module's wall time and peak device memory with the card it ran on.
"""
import ctypes
import subprocess
import time

import numpy as np
import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib
from nerf_pl_b200.nerf import packed_weights
from nerf_pl_b200.rendering import _render_args
from nerf_pl_b200.training import TrainWorkspace, _grad_buffers, _params_of
from oracle import nerf_oracle as orc
from tests import cases
from tests import render_tape as rt
from tests import test_gpu_render_stages as rs
from tests import test_gpu_train_stages as ts
from tests import train_tape as tt

# (N_samples, N_importance): batch size and options.  Every value of every option runs with a 96-sample and with a
# 160-sample fine pass (test_matrix_is_the_whole_envelope); "seed" draws the uniforms in the kernel.
MATRIX = {
    (32, 0): dict(n=45, use_disp=True, perturb=1.0, noise_std=1.0, white_back=False, rng="seed", weights="random"),
    (32, 32): dict(n=56, use_disp=False, perturb=1.0, noise_std=0.0, white_back=True, rng="tensors", weights="trained"),
    (32, 64): dict(n=41, use_disp=True, perturb=1.0, noise_std=1.0, white_back=False, rng="seed", weights="trained"),
    (32, 96): dict(n=63, use_disp=True, perturb=0.0, noise_std=0.0, white_back=True, rng="tensors", weights="random"),
    (32, 128): dict(n=77, use_disp=False, perturb=1.0, noise_std=0.0, white_back=True, rng="tensors",
                    weights="trained"),
    (32, 160): dict(n=50, use_disp=False, perturb=1.0, noise_std=1.0, white_back=False, rng="tensors",
                    weights="trained"),
    (64, 0): dict(n=79, use_disp=False, perturb=0.0, noise_std=1.0, white_back=True, rng="tensors", weights="trained"),
    (64, 32): dict(n=64, use_disp=False, perturb=0.0, noise_std=0.0, white_back=True, rng="tensors", weights="random"),
    (64, 64): dict(n=72, use_disp=True, perturb=1.0, noise_std=0.0, white_back=False, rng="seed", weights="random"),
    (64, 96): dict(n=48, use_disp=True, perturb=0.0, noise_std=1.0, white_back=False, rng="tensors", weights="random"),
    (64, 128): dict(n=61, use_disp=False, perturb=1.0, noise_std=0.0, white_back=True, rng="seed", weights="trained"),
    (128, 0): dict(n=40, use_disp=False, perturb=1.0, noise_std=0.0, white_back=False, rng="tensors",
                   weights="random"),
    (128, 32): dict(n=53, use_disp=False, perturb=1.0, noise_std=1.0, white_back=True, rng="seed", weights="random"),
    (128, 64): dict(n=67, use_disp=True, perturb=0.0, noise_std=1.0, white_back=True, rng="tensors",
                    weights="trained"),
}
OPTIONS = {"use_disp": {False, True}, "perturb": {0.0, 1.0}, "noise_std": {0.0, 1.0}, "white_back": {False, True},
           "rng": {"tensors", "seed"}, "weights": {"random", "trained"}}
PAIRS = list(MATRIX)
PAIR_IDS = [f"s{S}_k{K}" for S, K in PAIRS]
# batch sizes of the 64+64 training step, as n = a * SMs + b
EDGES = [(0, 1), (0, 2), (0, 3), (0, 4), (0, 5), (2, -1), (2, 0), (2, 1), (4, 3)]
EDGE_IDS = [f"n{b}" if a == 0 else f"n{a}sm{b:+d}".replace("+0", "") for a, b in EDGES]
LARGE = [(4096, 64, 64), (8192, 64, 128)]
# the per-CTA split at 1024 rays: options per shape; max_ctas 0 is one CTA per SM, "sm-1" leaves 8 or 7 rays per CTA
CTA_SHAPES = {(64, 64): dict(noise_std=0.0, white_back=True, rng="tensors"),
              (32, 160): dict(noise_std=1.0, white_back=False, rng="tensors"),
              (128, 32): dict(noise_std=0.0, white_back=True, rng="seed")}
MAX_CTAS = [0, 1, 2, 3, 7, "sm-1"]


@pytest.fixture(scope="module")
def dev():
    d = torch.device("cuda:0")
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    name = torch.cuda.get_device_name(d)          # initialises CUDA, which resetting the statistics needs
    torch.cuda.reset_peak_memory_stats(d)
    t0 = time.perf_counter()
    yield d
    print(f"\nshape envelope on {name} (power limit {pl}): {time.perf_counter() - t0:.0f} s "
          f"wall, peak device memory {torch.cuda.max_memory_allocated(d) / 2 ** 30:.1f} GiB")


@pytest.fixture(scope="module")
def emb():
    return [nb.Embedding(3, 10), nb.Embedding(3, 4)]


@pytest.fixture(autouse=True)
def _release_workspaces():
    yield
    TrainWorkspace.clear()
    torch.cuda.empty_cache()


def _sm_count(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def test_matrix_is_the_whole_envelope():
    accepted = {(S, K) for S in (32, 64, 128) for K in range(0, 193, 32) if S + K <= 192}
    assert set(MATRIX) == accepted and len(accepted) == 14
    for sf in (96, 160):
        specs = [c for (S, K), c in MATRIX.items() if K and S + K == sf]
        for opt, values in OPTIONS.items():
            assert {c[opt] for c in specs} == values, (sf, opt)
    assert sum(c["n"] % 2 for c in MATRIX.values()) >= len(MATRIX) // 2


# ------------------------------------------------------------------------------------------ 1. the pair matrix
@pytest.mark.gpu
@pytest.mark.parametrize("S,K", PAIRS, ids=PAIR_IDS)
def test_forward_stages(S, K, dev, emb):
    c = dict(rs.DEFAULTS, **MATRIX[(S, K)], S=S, K=K)
    run = rs.run_render(c, 400 + PAIRS.index((S, K)), dev, emb)
    lines, bad = rs.forward_report(run, _sm_count(dev))
    print(f"\n[forward s{S}_k{K}] n {c['n']} " + " ".join(f"{k} {c[k]}" for k in OPTIONS) + "\n" + "\n".join(lines))
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("S,K", PAIRS, ids=PAIR_IDS)
def test_backward_stages(S, K, dev, emb):
    c = dict(ts.DEFAULTS, **MATRIX[(S, K)], S=S, K=K)
    run = ts.run_train(c, 420 + PAIRS.index((S, K)), dev, emb)
    lines, bad = ts.stage_report(run, dev)
    print(f"\n[backward s{S}_k{K}] n {c['n']} " + " ".join(f"{k} {c[k]}" for k in OPTIONS) + "\n" + "\n".join(lines))
    assert not bad, "\n".join(bad)


# ------------------------------------------------------------------------------------------ 2. batch sizes
@pytest.mark.gpu
@pytest.mark.parametrize("a,b", EDGES, ids=EDGE_IDS)
def test_batch_edges(a, b, dev, emb):
    n = a * _sm_count(dev) + b
    run = ts.run_train(dict(ts.DEFAULTS, n=n), 440 + EDGES.index((a, b)), dev, emb)
    lines, bad = ts.stage_report(run, dev)
    print(f"\n[n {n}]\n" + "\n".join(lines))
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("n,S,K", LARGE, ids=[f"n{n}_s{S}_k{K}" for n, S, K in LARGE])
def test_large_batches(n, S, K, dev, emb):
    """Every stage on the float64 references of all samples; the gradient contractions run on the device."""
    torch.cuda.reset_peak_memory_stats(dev)
    t0 = time.perf_counter()
    run = ts.run_train(dict(ts.DEFAULTS, n=n, S=S, K=K, rng="seed"), 460 + LARGE.index((n, S, K)), dev, emb)
    t1 = time.perf_counter()
    peak = torch.cuda.max_memory_allocated(dev) / 2 ** 30
    lines, bad = ts.stage_report(run, dev)
    print(f"\n[n {n} S {S} K {K}] step and host copy {t1 - t0:.0f} s, stage report {time.perf_counter() - t1:.0f} s, "
          f"peak device memory {peak:.1f} GiB (workspace {run['raw'].nbytes / 2 ** 30:.1f} GiB)\n" + "\n".join(lines))
    assert not bad, "\n".join(bad)


# ------------------------------------------------------------------------------------------ 3. the per-CTA split
def _regions(buf, P):
    """The per-sample regions the training forward writes for pass P (train_tape.layout), as byte views of their n
    valid rows (a tiled row's 128-byte pieces in tile order; padding rows are never written)."""
    n, npad = P["n"], P["n_pad"]

    def tiled(key, C, layers=1):
        r = buf[P[key]:P[key] + layers * npad * C * 2].view(layers, npad // 64, C // 64, 64, 128)
        return r.transpose(2, 3).reshape(layers, npad, C * 2)[:, :n]
    return {"enc": tiled("enc", 64), "act": tiled("act", 256, 8),
            "mask": buf[P["mask"]:P["mask"] + 8 * npad * 32].view(8, npad, 32)[:, :n], "d": tiled("d", 128),
            "sigma": buf[P["sigma"]:P["sigma"] + npad * 4][:n * 4], "rgb": buf[P["rgb"]:P["rgb"] + npad * 12][:n * 12],
            "z": buf[P["z"]:P["z"] + n * 4]}


def _differ(a, b):
    return int((a != b).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("S,K", list(CTA_SHAPES), ids=[f"s{S}_k{K}" for S, K in CTA_SHAPES])
def test_cta_split_is_invisible(S, K, dev, emb):
    """The same 1024 rays, random numbers and target rendered with each CTA count: inference outputs and extras
    bitwise equal; in training mode one workspace per CTA count, then nerfb200_render_backward on each with the
    fused-MSE seed: the per-sample workspace regions and the 48 gradients bitwise equal, and the loss within
    loss_report's bar for the capped grid (its per-CTA partial sums change the last bits)."""
    c = CTA_SHAPES[(S, K)]
    n, sm = 1024, _sm_count(dev)
    seed = 480 + list(CTA_SHAPES).index((S, K))
    rs_ = np.random.RandomState(seed)
    rays = torch.from_numpy(orc.make_rays(n, seed)).to(dev)
    target_np = rs_.uniform(0, 1, (n, 3)).astype(np.float32)
    target = torch.from_numpy(target_np).to(dev)
    T = lambda shape: torch.from_numpy(rs_.rand(*shape).astype(np.float32)).to(dev)
    G = lambda shape: torch.from_numpy(rs_.randn(*shape).astype(np.float32)).to(dev)
    randoms = (T((n, S)) if c["rng"] == "tensors" else None,
               G((n, S)) if c["noise_std"] > 0 else None,
               T((n, K)) if c["rng"] == "tensors" else None,
               G((n, S + K)) if c["noise_std"] > 0 else None)
    rng_seed = 1000 + seed if c["rng"] == "seed" else None
    models = ts._models(cases.weights(), dev)
    packed = (packed_weights(models[0]), packed_weights(models[1]))
    params = _params_of(models, K)
    loss_grad = torch.tensor([0.0, 0.0, 1.0, 0.0], device=dev)      # d loss_out / d loss: element 2 is the MSE loss
    f32 = dict(dtype=torch.float32, device=dev)
    keys = ("rgb_coarse", "depth_coarse", "opacity_coarse", "rgb_fine", "depth_fine", "opacity_fine")
    shapes = ((n, 3), (n,), (n,), (n, 3), (n,), (n,))

    def render(max_ctas, ws=None):
        outs = {k: torch.empty(s, **f32) for k, s in zip(keys, shapes)}
        if ws is None:
            outs.update(z_fine=torch.empty(n, S + K, **f32), weights_coarse=torch.empty(n, S, **f32),
                        weights_fine=torch.empty(n, S + K, **f32))
        loss_out = torch.empty(4, **f32) if ws is not None else None
        args = _render_args(rays, S, K, False, 1.0, c["noise_std"], c["white_back"], False, packed, randoms, outs,
                            rng_seed, ws, target if ws is not None else None, loss_out)
        args.max_ctas = max_ctas
        _lib.call("nerfb200_render_rays", dev, ctypes.byref(args))
        if loss_out is not None:
            outs["loss_out"] = loss_out
        return args, outs

    bad, lines, ref_inf, ref_tr = [], [], None, None
    for mc in MAX_CTAS:
        m = sm - 1 if mc == "sm-1" else mc
        grid = min(m if m > 0 else sm, sm, (n + 1) // 2)
        _, inf = render(m)
        ws = TrainWorkspace(dev, n, S, K)
        args, tr = render(m, ws)
        args.target = args.loss_out = None                   # the backward takes the seed from its own arguments
        grads, tables = _grad_buffers(params, dev)
        bargs = _lib.BackwardArgs(render=ctypes.pointer(args), params_coarse=tables[0][0], params_fine=tables[1][0],
                                  target=target.data_ptr(), loss_grad=loss_grad.data_ptr() + 8,
                                  grads_coarse=tables[0][1], grads_fine=tables[1][1])
        _lib.call("nerfb200_render_backward", dev, ctypes.byref(bargs))
        torch.cuda.synchronize()
        assert _lib.load().nerfb200_check_status() == 0
        l4 = tr.pop("loss_out").cpu().numpy()
        lr = rs.loss_report(n, S, K, tr["rgb_coarse"].cpu().numpy(), tr["rgb_fine"].cpu().numpy(), target_np,
                            dict(zip(("mse_coarse", "mse_fine", "loss", "psnr"), l4.astype(np.float64))), grid)
        lines.append(f"max_ctas {m} (grid {grid}, {n // grid}-{-(-n // grid)} rays per CTA): loss " +
                     " ".join(f"{k} {v:.3g}" for k, v in lr.items()))
        bad += [f"max_ctas {m}: loss {k} {v:.3g}" for k, v in lr.items()
                if not v <= rt.BARS["psnr" if k == "psnr" else "loss"]]
        regions = [_regions(ws.buf, P) for P in tt.layout(n, S, K)]
        if ref_inf is None:                 # the views in ref_regions keep the reference's workspace
            ref_inf, ref_tr, ref_regions, ref_grads = inf, tr, regions, grads
            for k in keys:
                if not torch.equal(tr[k], inf[k]):
                    bad.append(f"training {k} differs from inference in {_differ(tr[k], inf[k])} elements")
            continue
        for k, v in inf.items():
            if not torch.equal(v, ref_inf[k]):
                bad.append(f"max_ctas {m}: inference {k} differs in {_differ(v, ref_inf[k])} elements")
        for k, v in tr.items():
            if not torch.equal(v, ref_tr[k]):
                bad.append(f"max_ctas {m}: training {k} differs in {_differ(v, ref_tr[k])} elements")
        for ps, (got, ref) in enumerate(zip(regions, ref_regions)):
            for k in got:
                if not torch.equal(got[k], ref[k]):
                    bad.append(f"max_ctas {m}: {('coarse', 'fine')[ps]} workspace {k} differs in "
                               f"{_differ(got[k], ref[k])} bytes")
        for i, (g, r) in enumerate(zip(grads, ref_grads)):
            if not torch.equal(g, r):
                bad.append(f"max_ctas {m}: gradient {i} ({'coarse' if i < 24 else 'fine'}) differs in "
                           f"{_differ(g, r)} elements")
        del ws, regions, grads              # one workspace besides the reference's at a time
    print(f"\n[1024 rays S {S} K {K}] " + ", ".join(f"{k} {v}" for k, v in c.items()) + "\n" + "\n".join(lines))
    assert not bad, "\n".join(bad)
