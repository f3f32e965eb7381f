"""Render time of skip="samples" against the plain render and skip="rays" on the trained test network.

The grid is the tests' (N = 128 over [-1.5, 1.5]^3, sigma > 1, dilate 1); the views are Blender-style views of the
trained scene (radius-4 camera, near 2, far 6) at 400 x 400 and 800 x 800, 64 + 128 samples.  The three modes run
alternately in one process; medians and the spread are over views x rounds.  Also reports the live-ray and
evaluated-sample fractions and the error of "samples" against the plain render (all pixels and the live ones):
mean and max of |d rgb_fine|, |d opacity_fine| and |d depth_fine|.

    python tools/bench_sample_skip.py [--rounds 3] [--views 3] [--out FILE]
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
from tests import cases  # noqa: E402


def _gpu():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--views", type=int, default=3)
    ap.add_argument("--sizes", default="400,800")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = _gpu()
    models = []
    for w in cases.trained_weights():
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        models.append(m.cuda().eval())
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    grid = nb.occupancy_grid(models[1], 128, (-1.5, 1.5), (-1.5, 1.5), (-1.5, 1.5), 1.0, 1)

    def run(mode, rays):
        if mode == "plain":
            return nb.batched_inference(models, emb, rays, 64, 128, False, white_back=True)
        return nb.batched_inference(models, emb, rays, 64, 128, False, white_back=True, occupancy=grid, skip=mode)

    report = {"gpu": gpu, "sizes": {}}
    for side in [int(s) for s in a.sizes.split(",")]:
        views = [torch.from_numpy(bench.blender_rays(0, 80 + v, W=side, H=side, pixels="all")).cuda()
                 for v in range(a.views)]
        for r in views[:1]:
            for mode in ("plain", "rays", "samples"):
                run(mode, r)
        times = {m: [] for m in ("plain", "rays", "samples")}
        errs = []
        for rnd in range(a.rounds):
            for vi, rays in enumerate(views):
                outs = {}
                for mode in ("plain", "rays", "samples"):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    outs[mode] = run(mode, rays)
                    torch.cuda.synchronize()
                    times[mode].append((time.perf_counter() - t0) * 1e3)
                if rnd == 0:
                    p, s = outs["plain"], outs["samples"]
                    n = rays.shape[0]
                    live = s["live_idx"]
                    e = {}
                    for key in ("rgb_fine", "opacity_fine", "depth_fine"):
                        d = (s[key] - p[key]).abs()
                        d = d.amax(1) if d.dim() == 2 else d
                        e[key] = (float(d.mean()), float(d.max()), float(d[live].mean()), float(d[live].max()))
                    e["live_rays"] = s["live"] / n
                    e["live_samples"] = (s["live_samples"][0] / (64 * n), s["live_samples"][1] / (192 * n))
                    errs.append(e)
        med = {m: (float(np.median(v)), float(np.min(v)), float(np.max(v))) for m, v in times.items()}
        report["sizes"][side] = {"ms": med, "errors": errs,
                                 "samples_over_rays": med["samples"][0] / med["rays"][0]}
        print(f"{side}x{side} on {gpu}:")
        for m, (md, lo, hi) in med.items():
            print(f"  {m:8s} median {md:8.2f} ms  [{lo:.2f}, {hi:.2f}]")
        print(f"  samples / rays = {med['samples'][0] / med['rays'][0]:.3f}, samples / plain = "
              f"{med['samples'][0] / med['plain'][0]:.3f}")
        for e in errs:
            print("  " + json.dumps(e))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
