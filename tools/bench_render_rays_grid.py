"""render_rays(..., occupancy=grid) in training and validation, against the plain call and the fused loss.

Set-up of tools/bench_train_skip.py: the trained test scene, the tests' grid (N = 128 over [-1.5, 1.5]^3, sigma > 1,
dilate 1, from the fine network), random pixels of Blender-style views (radius-4 camera, near 2, far 6) with random
targets, perturb 1, noise_std 1, in-kernel random numbers, white_back.

1. Training steps (eager; forward + loss + backward, no optimiser, so that the grid stays the network's):
   (a) plain render_rays + the reference's MSELoss (coarse + fine) + backward;
   (b) render_rays(..., occupancy=grid) + the same MSELoss + backward;
   (c) render_rays_loss(..., occupancy=grid) + loss.backward().
   At 1024 and 4096 rays, 64 + 64 and 64 + 128 samples.
2. Validation: an 800 x 800 render (640,000 rays, 64 + 128 samples, perturb 1, noise_std 1, test_time False) under
   torch.no_grad(), plain and with the grid.

The variants alternate within each round; medians and ranges are over rounds.  The card's name and power limit are
read in the same run.

    python tools/bench_render_rays_grid.py [--rounds 7] [--steps 20] [--val-rounds 5] [--out FILE]
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


def _stats(v):
    return float(np.median(v)), float(np.min(v)), float(np.max(v))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--val-rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_render_rays_grid needs a CUDA device")
    gpu = _gpu()
    models = []
    for w in cases.trained_weights():
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        models.append(m.cuda())
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    with torch.no_grad():
        grid = nb.occupancy_grid(models[1], 128, (-1.5, 1.5), (-1.5, 1.5), (-1.5, 1.5), 1.0, 1)
    mse = torch.nn.MSELoss(reduction="mean")
    report = {"gpu": gpu, "occupied": grid.occupied_fraction(), "train": {}, "validation": {}}
    print(f"{gpu}; occupied cells {report['occupied']:.3f}")
    for n in (1024, 4096):
        rays = torch.from_numpy(bench.blender_rays(n, 7)).cuda()
        rgbs = torch.rand(n, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
        for S, K in ((64, 64), (64, 128)):
            def step(variant):
                for m in models:
                    m.zero_grad(set_to_none=True)
                if variant == "c":
                    res = nb.render_rays_loss(models, emb, rays, rgbs, S, False, 1.0, 1.0, K, 32768, True,
                                              randoms="kernel", occupancy=grid)
                    res["loss"].backward()
                    return
                res = nb.render_rays(models, emb, rays, S, False, 1.0, 1.0, K, 32768, True, randoms="kernel",
                                     occupancy=grid if variant == "b" else None)
                (mse(res["rgb_coarse"], rgbs) + mse(res["rgb_fine"], rgbs)).backward()

            times = {"a": [], "b": [], "c": []}
            for v in times:
                for _ in range(3):
                    step(v)
            for _ in range(a.rounds):
                for v in times:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(a.steps):
                        step(v)
                    torch.cuda.synchronize()
                    times[v].append((time.perf_counter() - t0) * 1e3 / a.steps)
            med = {v: _stats(t) for v, t in times.items()}
            key = f"{n} rays, {S}+{K}"
            report["train"][key] = {"ms": med, "b_over_a": med["b"][0] / med["a"][0]}
            print(f"{key}: " + ", ".join(f"({v}) {m[0]:.3f} ms [{m[1]:.3f}, {m[2]:.3f}]" for v, m in med.items())
                  + f"; (b)/(a) {med['b'][0] / med['a'][0]:.3f}")
    nb.train_skip.SkipTrainWorkspace.clear()
    torch.cuda.empty_cache()
    rays = torch.from_numpy(bench.blender_rays(800 * 800, 80)).cuda()
    times = {"plain": [], "grid": []}

    def render(mode):
        with torch.no_grad():
            return nb.render_rays(models, emb, rays, 64, False, 1.0, 1.0, 128, 32768, True, randoms="kernel",
                                  occupancy=grid if mode == "grid" else None)

    for mode in times:
        render(mode)
    for _ in range(a.val_rounds):
        for mode in times:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            render(mode)
            torch.cuda.synchronize()
            times[mode].append((time.perf_counter() - t0) * 1e3)
    med = {k: _stats(v) for k, v in times.items()}
    report["validation"] = {"ms": med, "grid_over_plain": med["grid"][0] / med["plain"][0]}
    print("validation 800x800, 64+128, perturb 1, noise 1: " +
          ", ".join(f"{k} {m[0]:.1f} ms [{m[1]:.1f}, {m[2]:.1f}]" for k, m in med.items()) +
          f"; grid/plain {med['grid'][0] / med['plain'][0]:.3f}")
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
