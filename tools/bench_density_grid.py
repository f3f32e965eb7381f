"""The density grid (nb.DensityGrid): what an update costs, and whether training with the grid maintained inside the
captured loop beats plain captured training.

1. Update time.  One DensityGrid.update of the trained test network (the fine one) at N in --sizes, against
nb.occupancy_grid at the same N (sigma > 1, dilate 1, over [-1.5, 1.5]^3 for both).  CUDA events around --calls calls,
after a warm-up of each; the two alternate over --rounds rounds and the median and range are over the rounds.

2. From-scratch training (--train) on tools/train_sharp_weights.py's procedural scene and recipe (64 + 64 samples,
perturb 1, noise 1, Adam 5e-4, the same model seed), captured: the 64 training views' rays go into one
DeviceRayBatches, and each run trains with CapturedTrainStep and in-kernel randoms.  "plain" is a plain
CapturedTrainStep for --train-steps steps; "W=.., R=.." is a plain CapturedTrainStep for W steps, then
CapturedTrainStep(occupancy=DensityGrid(128, box, 1.0, decay 0.95, dilate 1), update_every=R) on the same optimizer.
Both batch sizes of --batches.  Every --every steps the held-out view (16384 rays of view 9999, fine pass at test
time) is rendered outside the timed region, plainly and with skip="samples" on the run's grid.  The train time is the
replays' wall-clock (each segment ends in a device synchronise); the construction of each step (warm-up and capture)
is reported apart.  Reported: PSNR at equal steps, and at equal wall-clock (the plain curve interpolated at the
grid run's time).

The card's name and power limit are read in the same run.

    python tools/bench_density_grid.py [--sizes 64,128,256] [--rounds 5] [--calls 10] [--out FILE]
    python tools/bench_density_grid.py --train [--train-steps 3000] [--every 250] [--schedules 500:16,2000:16]
        [--batches 1024,4096] [--out FILE]
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

BOX = ((-1.5, 1.5),) * 3


def _gpu():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def _events_ms(fn, calls):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / calls


def update_times(a, gpu):
    models = []
    for w in cases.trained_weights():
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        models.append(m.cuda().eval())
    fine = models[1]
    report = {"gpu": gpu, "sizes": {}}
    for N in (int(s) for s in a.sizes.split(",")):
        dg = nb.DensityGrid(N, *BOX, sigma_threshold=1.0, decay=0.95, dilate=1, seed=0)
        fns = {"update": lambda: dg.update(fine),
               "occupancy_grid": lambda: nb.occupancy_grid(fine, N, *BOX, 1.0, 1)}
        times = {k: [] for k in fns}
        for f in fns.values():
            f()
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for k, f in fns.items():
                times[k].append(_events_ms(f, a.calls))
        med = {k: (float(np.median(v)), float(np.min(v)), float(np.max(v))) for k, v in times.items()}
        report["sizes"][N] = {"ms": med, "occupied": dg.grid.occupied_fraction()}
        print(f"N = {N} on {gpu}: update {med['update'][0]:.3f} ms [{med['update'][1]:.3f}, {med['update'][2]:.3f}], "
              f"occupancy_grid {med['occupancy_grid'][0]:.3f} ms [{med['occupancy_grid'][1]:.3f}, "
              f"{med['occupancy_grid'][2]:.3f}]; {(N - 1) ** 3} cells")
    return report


def _psnr(models, emb, held, gt, grid):
    with torch.no_grad():
        res = nb.render_rays(models, emb, held, 64, False, 0, 0, 64, 32768, True, test_time=True)
        psnr = -10 * np.log10(float(((res["rgb_fine"] - gt) ** 2).mean()))
        psnr_grid = psnr
        if grid is not None:
            res = nb.render_rays_culled(models, emb, held, grid, 64, False, 64, True, True, skip="samples")
            psnr_grid = -10 * np.log10(float(((res["rgb_fine"] - gt) ** 2).mean()))
    return psnr, psnr_grid


def _train(batches, emb, held, gt, steps, every, schedule):
    """One from-scratch run; schedule None = plain, else (W, R).  -> (curve [(step, train seconds, PSNR, PSNR with
    the grid, evaluated fine fraction)], construction seconds)."""
    torch.manual_seed(1234)
    models = [nb.NeRF().cuda(), nb.NeRF().cuda()]
    opt = nb.FusedAdam([p for m in models for p in m.parameters()], lr=5e-4, eps=1e-8, capturable=True)
    B = batches.batch_size
    build = 0.0

    def make(occ=None, R=None):
        nonlocal build
        torch.cuda.synchronize()
        t = time.perf_counter()
        s = nb.CapturedTrainStep(models, batches, opt, 64, False, 1.0, 1.0, 64, True, randoms="kernel",
                                 occupancy=occ, update_every=R)
        torch.cuda.synchronize()
        build += time.perf_counter() - t
        return s

    step, dg = make(), None
    curve, t_train, frac = [], 0.0, 1.0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for it in range(steps):
        if schedule is not None and it == schedule[0]:
            torch.cuda.synchronize()
            t_train += time.perf_counter() - t0
            dg = nb.DensityGrid(128, *BOX, sigma_threshold=1.0, decay=0.95, dilate=1, seed=5)
            step = make(dg, schedule[1])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        step.step()
        if (it + 1) % every == 0:
            torch.cuda.synchronize()
            t_train += time.perf_counter() - t0
            if dg is not None:
                frac = float(step.live_samples[1]) / (B * 128)
            psnr, psnr_grid = _psnr(models, emb, held, gt, None if dg is None else dg.grid)
            curve.append((it + 1, t_train, psnr, psnr_grid, frac))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
    return curve, build


def train_compare(a, gpu):
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from train_sharp_weights import ground_truth
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    rays = torch.cat([torch.from_numpy(bench.blender_rays(16384, 7000 + v)) for v in range(64)])
    rgbs = torch.cat([ground_truth(r.cuda()) for r in rays.split(16384)])
    held = torch.from_numpy(bench.blender_rays(16384, 9999)).cuda()
    gt = ground_truth(held)
    schedules = [tuple(int(x) for x in s.split(":")) for s in a.schedules.split(",")]
    report = {"gpu": gpu, "steps": a.train_steps, "batches": {}}
    for B in (int(b) for b in a.batches.split(",")):
        batches = nb.DeviceRayBatches(rays, rgbs, batch_size=B, drop_last=True, seed=99)
        runs, builds = {}, {}
        for sch in [None] + schedules:
            name = "plain" if sch is None else f"W={sch[0]} R={sch[1]}"
            runs[name], builds[name] = _train(batches, emb, held, gt, a.train_steps, a.every, sch)
        plain = runs["plain"]
        pt, pp = np.array([c[1] for c in plain]), np.array([c[2] for c in plain])
        rep = {"curves": runs, "construction_seconds": builds, "summary": {}}
        print(f"from-scratch captured training, {B}-ray batches, {a.train_steps} steps, on {gpu}")
        print(f"  plain: {plain[-1][1]:.2f} s, held-out PSNR {plain[-1][2]:.2f} dB (construction {builds['plain']:.2f} s)")
        for name, c in runs.items():
            if name == "plain":
                continue
            T = c[-1][1]
            eq_time = float(np.interp(T, pt, pp))
            rep["summary"][name] = {"seconds": T, "psnr": c[-1][2], "psnr_rendered_with_grid": c[-1][3],
                                    "plain_psnr_equal_steps": plain[-1][2], "plain_psnr_equal_time": eq_time,
                                    "plain_seconds": plain[-1][1], "evaluated_fine_fraction": c[-1][4]}
            print(f"  {name}: {T:.2f} s, held-out PSNR {c[-1][2]:.2f} dB ({c[-1][3]:.2f} dB rendered with its grid); "
                  f"plain at equal steps {plain[-1][2]:.2f} dB, at equal time {eq_time:.2f} dB; evaluated fine "
                  f"fraction {c[-1][4]:.3f} (construction {builds[name]:.2f} s)")
        report["batches"][B] = rep
        del batches
        torch.cuda.empty_cache()
    return report


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="64,128,256")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--train", action="store_true")
    ap.add_argument("--train-steps", type=int, default=3000)
    ap.add_argument("--every", type=int, default=250)
    ap.add_argument("--schedules", default="500:16,2000:16")
    ap.add_argument("--batches", default="1024,4096")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_density_grid.py measures on the GPU; no CUDA device is visible")
    gpu = _gpu()
    report = train_compare(a, gpu) if a.train else update_times(a, gpu)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
