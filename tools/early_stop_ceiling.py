"""The most early ray termination could save on the trained test scene, measured before building it (DESIGN.md §10f).

Renders Blender views of the trained test network with skip="samples" and the tests' grid (N = 128 over
[-1.5, 1.5]^3, sigma > 1, dilate 1) through ``culling.render_samples(..., per_sample=True)``, so every sample's
sigma is the device's own.  On the final pass (fine with N_importance > 0, coarse otherwise) it applies the float64
rule of tests/early_stop_ref.py and reports, for each eps:

  - word:   the evaluated final-pass samples in words after the ray's cut (what the word-granular rule drops);
  - sample: the evaluated samples whose transmittance before them is already below eps (what any front-to-back rule
            at that eps could drop, whatever its granularity);
  - the fraction of rays cut, and of live rays cut.

It also times skip="samples" itself (median and range over views x rounds after a warm-up) and, in a separate
profiled render, splits the MLP's kernel time between the two passes, so that a fraction of final-pass rows can be
turned into an upper bound on the time termination could save.  The card's name and power limit are read in the
same run.

    python tools/early_stop_ceiling.py [--sizes 400,800] [--views 3] [--rounds 3] [--shapes 64+128,128+0]
                                       [--eps 1e-4,1e-3,1e-2] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import nerf_pl_b200 as nb  # noqa: E402
from nerf_pl_b200 import culling  # noqa: E402
from tests import cases  # noqa: E402
from tests import early_stop_ref as es  # noqa: E402
from tests import sample_skip_ref as sk  # noqa: E402

CUBE = ((-1.5, 1.5),) * 3
ROWS = 1 << 16          # rays per float64 block on the host


def _gpu():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def ceiling(rays, z, sigma, ev, eps_list):
    """Counts for one pass: rays (n, 8), z / sigma (n, S) float32, ev (n, S) bool evaluated; numpy, in blocks."""
    n = rays.shape[0]
    out = {"evaluated": int(ev.sum()), "rays": n, "live_rays": int(ev.any(1).sum())}
    acc = {e: {"word": 0, "sample": 0, "cut_rays": 0, "cut_live_rays": 0} for e in eps_list}
    for lo in range(0, n, ROWS):
        sl = slice(lo, min(n, lo + ROWS))
        r, zz, sg, e_ = rays[sl], z[sl], sigma[sl], ev[sl]
        plain = sk.plain_pass(r, zz)
        a = es.alphas(r, zz, sg)
        with np.errstate(invalid="ignore", over="ignore"):
            t_before = np.cumprod(np.concatenate([np.ones((a.shape[0], 1)), 1.0 - a[:, :-1] + 1e-10], 1), 1)
        for eps in eps_list:
            cut, _ = es.cut_words(r, zz, sg, eps)
            c = acc[eps]
            c["word"] += int(es.dropped(e_, cut).sum())
            with np.errstate(invalid="ignore"):
                c["sample"] += int((e_ & (t_before < eps) & ~plain[:, None]).sum())
            c["cut_rays"] += int((cut >= 0).sum())
            c["cut_live_rays"] += int(((cut >= 0) & e_.any(1)).sum())
    for eps, c in acc.items():
        out[f"{eps:g}"] = {"word_dropped": c["word"] / max(out["evaluated"], 1),
                           "sample_dropped": c["sample"] / max(out["evaluated"], 1),
                           "cut_rays": c["cut_rays"] / n, "cut_live_rays": c["cut_live_rays"] / max(out["live_rays"], 1)}
    return out


def mlp_split_ms(render, K):
    """(first pass, final pass) MLP kernel time of one render in ms, all kernels' time and the MLP launches, from a
    profiled run: with K > 0 render_samples launches the coarse MLP, then the fine one, per chunk of live rays."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        render()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if "mlp_forward_kernel" in e.name and e.device_type == torch.autograd.DeviceType.CUDA]
    ev.sort(key=lambda e: e.time_range.start)
    ms = [e.time_range.elapsed_us() / 1e3 for e in ev]
    total = sum(e.time_range.elapsed_us() for e in prof.events()
                if e.device_type == torch.autograd.DeviceType.CUDA) / 1e3
    if K == 0:
        return 0.0, sum(ms), total, len(ms)
    return sum(ms[0::2]), sum(ms[1::2]), total, len(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="400,800")
    ap.add_argument("--views", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default="64+128,128+0")
    ap.add_argument("--eps", default="1e-4,1e-3,1e-2")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("early_stop_ceiling needs a CUDA device")
    gpu = _gpu()
    eps_list = [float(e) for e in a.eps.split(",")]
    models = []
    for w in cases.trained_weights():
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        models.append(m.cuda().eval())
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    grid = nb.occupancy_grid(models[1], 128, *CUBE, 1.0, 1)
    report = {"gpu": gpu, "runs": []}
    print(f"on {gpu}")
    for shape in a.shapes.split(","):
        S, K = (int(v) for v in shape.split("+"))
        pre = "fine" if K else "coarse"
        for side in [int(s) for s in a.sizes.split(",")]:
            views = [torch.from_numpy(bench.blender_rays(0, 80 + v, W=side, H=side, pixels="all")).cuda()
                     for v in range(a.views)]
            counts = []
            for rays in views:
                _, _, flag = nb.cull_rays(rays, grid, return_flag=True)
                r = culling.render_samples(models, rays, grid, S, False, K, True, True, live_flag=flag, extras=True,
                                           per_sample=True)
                rn = rays.cpu().numpy()
                z = r["z_vals_fine"].cpu().numpy() if K else sk.z_base(rn, S)
                sigma = r[f"samples_{pre}"][..., 3].cpu().numpy()
                ev = sk.mask_bits(r[f"mask_{pre}"].cpu().numpy(), S + K)
                del r
                torch.cuda.empty_cache()
                counts.append(ceiling(rn, z, sigma, ev, eps_list))

            def render(rays):
                return nb.batched_inference(models, emb, rays, S, K, False, white_back=True, occupancy=grid,
                                            skip="samples")
            for rays in views:
                render(rays)
            times = []
            for _ in range(a.rounds):
                for rays in views:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    render(rays)
                    torch.cuda.synchronize()
                    times.append((time.perf_counter() - t0) * 1e3)
            mc, mf, kern, launches = mlp_split_ms(lambda: render(views[0]), K)
            run = {"S": S, "K": K, "side": side, "views": counts,
                   "ms": (float(np.median(times)), float(np.min(times)), float(np.max(times))),
                   "profiled_view0": {"mlp_first_pass_ms": mc, "mlp_final_pass_ms": mf, "all_kernels_ms": kern,
                                      "mlp_launches": launches}}
            report["runs"].append(run)
            md, lo, hi = run["ms"]
            print(f"{S} + {K} at {side} x {side}: skip='samples' median {md:.2f} ms [{lo:.2f}, {hi:.2f}]; view 80 "
                  f"profiled: MLP first pass {mc:.2f} ms, final pass {mf:.2f} ms of {kern:.2f} ms kernel time "
                  f"({launches} MLP launches)")
            for v, c in enumerate(counts):
                print(f"  view {80 + v}: {json.dumps(c)}")
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
