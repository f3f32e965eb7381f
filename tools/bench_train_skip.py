"""Training with empty samples skipped (render_rays_loss(..., occupancy=grid)) against plain training.

1. Step time.  The grid is the tests' (N = 128 over [-1.5, 1.5]^3, sigma > 1, dilate 1, from the fine network); the
rays are random pixels of Blender-style views of the trained scene (radius-4 camera, near 2, far 6) with random targets, perturb 1,
noise_std 1, in-kernel random numbers.  One step is forward + loss.backward() + FusedAdam; the two modes alternate in
one process and the medians and ranges are over rounds.

2. From-scratch training (--train) on tools/train_sharp_weights.py's procedural scene and recipe (64 + 64 samples,
perturb 1, noise 1, 1024-ray batches, Adam 5e-4, the same seeds): plain training, and for each warm-up W and refresh
period R of --schedules, plain steps until W, then a grid from the fine network (N = 128 over [-1.5, 1.5]^3, sigma > 1,
dilate 1) rebuilt every R steps, the grid builds included in the time.  Every --every steps the held-out view's PSNR
(the fine pass at test time, 16384 rays of view 9999) is taken outside the timed region.  Reported: the PSNR at equal
steps, and at equal wall-clock (the plain curve interpolated at the skipped run's total time); the schedule with the
best PSNR at equal wall-clock is the one to use.  The skipped runs' PSNR is also given with the view rendered
with skip="samples" and the run's last grid, as a user of the grid renders it.

The card's name and power limit are read in the same run.

    python tools/bench_train_skip.py [--rounds 5] [--steps 20] [--out FILE]
    python tools/bench_train_skip.py --train [--train-steps 3000] [--every 250] [--schedules 500:100,1000:500]
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


def _train(models, emb, views, targets, held, gt, steps, every, schedule):
    """One from-scratch run; schedule None = plain, else (W, R).  -> [(step, train seconds, held-out PSNR, evaluated
    fraction of the fine samples in the last step, held-out PSNR rendered with the run's grid)]."""
    opt = nb.FusedAdam([p for m in models for p in m.parameters()], lr=5e-4, eps=1e-8)
    gen = torch.Generator(device="cuda").manual_seed(99)
    grid, curve, t_train, frac = None, [], 0.0, 1.0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for it in range(steps):
        if schedule is not None and it >= schedule[0] and (it - schedule[0]) % schedule[1] == 0:
            with torch.no_grad():
                grid = nb.occupancy_grid(models[1], 128, (-1.5, 1.5), (-1.5, 1.5), (-1.5, 1.5), 1.0, 1)
        v = it % len(views)
        idx = torch.randint(0, views[v].shape[0], (1024,), device="cuda", generator=gen)
        out = nb.render_rays_loss(models, emb, views[v][idx], targets[v][idx], 64, False, 1.0, 1.0, 64, 32768, True,
                                  match_reference_rng=False, occupancy=grid)
        opt.zero_grad(set_to_none=True)
        out["loss"].backward()
        opt.step()
        if grid is not None:
            frac = out["live_samples"][1] / (1024 * 128)
        if (it + 1) % every == 0:
            torch.cuda.synchronize()
            t_train += time.perf_counter() - t0
            with torch.no_grad():
                res = nb.render_rays(models, emb, held, 64, False, 0, 0, 64, 32768, True, test_time=True)
                psnr = -10 * np.log10(float(((res["rgb_fine"] - gt) ** 2).mean()))
                psnr_grid = psnr
                if grid is not None:    # rendered as a user of the grid renders: skip="samples" with the same grid
                    res = nb.render_rays_culled(models, emb, held, grid, 64, False, 64, True, True, skip="samples")
                    psnr_grid = -10 * np.log10(float(((res["rgb_fine"] - gt) ** 2).mean()))
            curve.append((it + 1, t_train, psnr, frac, psnr_grid))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
    return curve


def train_compare(a, gpu):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__))))
    from train_sharp_weights import ground_truth
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    views = [torch.from_numpy(bench.blender_rays(16384, 7000 + v)).cuda() for v in range(64)]
    targets = [ground_truth(v) for v in views]
    held = torch.from_numpy(bench.blender_rays(16384, 9999)).cuda()
    gt = ground_truth(held)
    schedules = [tuple(int(x) for x in s.split(":")) for s in a.schedules.split(",")]
    runs = {}
    for sch in [None] + schedules:
        torch.manual_seed(1234)
        models = [nb.NeRF().cuda(), nb.NeRF().cuda()]
        runs["plain" if sch is None else f"W={sch[0]} R={sch[1]}"] = _train(models, emb, views, targets, held, gt,
                                                                            a.train_steps, a.every, sch)
    plain = runs["plain"]
    pt, pp = np.array([c[1] for c in plain]), np.array([c[2] for c in plain])
    report = {"gpu": gpu, "steps": a.train_steps, "curves": runs, "summary": {}}
    print(f"from-scratch training, {a.train_steps} steps, on {gpu}")
    print(f"  plain: {plain[-1][1]:.2f} s, held-out PSNR {plain[-1][2]:.2f} dB")
    best = None
    for name, c in runs.items():
        if name == "plain":
            continue
        T = c[-1][1]
        eq_time = float(np.interp(T, pt, pp))
        report["summary"][name] = {"seconds": T, "psnr": c[-1][2], "plain_psnr_equal_steps": plain[-1][2],
                                   "plain_psnr_equal_time": eq_time, "plain_seconds": plain[-1][1],
                                   "evaluated_fine_fraction": c[-1][3], "psnr_rendered_with_grid": c[-1][4]}
        print(f"  {name}: {T:.2f} s, held-out PSNR {c[-1][2]:.2f} dB ({c[-1][4]:.2f} dB rendered with its grid); plain "
              f"at equal steps {plain[-1][2]:.2f} dB, at equal time {eq_time:.2f} dB; evaluated fine fraction "
              f"{c[-1][3]:.3f}")
        if best is None or c[-1][2] - eq_time > best[1]:
            best = (name, c[-1][2] - eq_time)
    report["best"] = best[0]
    print(f"  best at equal wall-clock: {best[0]} ({best[1]:+.2f} dB against plain)")
    return report


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--train", action="store_true")
    ap.add_argument("--train-steps", type=int, default=3000)
    ap.add_argument("--every", type=int, default=250)
    ap.add_argument("--schedules", default="500:100,1000:500,2000:100,2000:500")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = _gpu()
    if a.train:
        report = train_compare(a, gpu)
        if a.out:
            with open(a.out, "w") as f:
                json.dump(report, f, indent=1)
        return
    models = []
    for w in cases.trained_weights():
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        models.append(m.cuda())
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    with torch.no_grad():
        grid = nb.occupancy_grid(models[1], 128, (-1.5, 1.5), (-1.5, 1.5), (-1.5, 1.5), 1.0, 1)
    init = [{k: v.detach().clone() for k, v in m.state_dict().items()} for m in models]
    report = {"gpu": gpu, "occupied": grid.occupied_fraction(), "cases": {}}
    for n in (1024, 4096):
        rays = torch.from_numpy(bench.blender_rays(n, 7)).cuda()
        rgbs = torch.rand(n, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
        for S, K in ((64, 64), (64, 128)):
            opt = nb.FusedAdam([p for m in models for p in m.parameters()], lr=5e-4)
            live = []

            def step(occ):
                opt.zero_grad(set_to_none=True)
                res = nb.render_rays_loss(models, emb, rays, rgbs, S, False, 1.0, 1.0, K, 32768, True,
                                          randoms="kernel", occupancy=occ)
                res["loss"].backward()
                opt.step()
                if occ is not None:
                    live.append(res["live_samples"])

            times = {"plain": [], "skip": []}
            for mode in times:
                step(grid if mode == "skip" else None)
            for _ in range(a.rounds):
                for mode in times:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(a.steps):
                        step(grid if mode == "skip" else None)
                    torch.cuda.synchronize()
                    times[mode].append((time.perf_counter() - t0) * 1e3 / a.steps)
            for m, s in zip(models, init):
                m.load_state_dict(s)
            med = {k: (float(np.median(v)), float(np.min(v)), float(np.max(v))) for k, v in times.items()}
            frac = (float(np.mean([c for c, _ in live])) / (n * S), float(np.mean([f for _, f in live])) / (n * (S + K)))
            key = f"{n} rays, {S}+{K}"
            report["cases"][key] = {"ms": med, "skip_over_plain": med["skip"][0] / med["plain"][0],
                                    "evaluated_fraction": frac}
            print(f"{key} on {gpu}: plain {med['plain'][0]:.3f} ms [{med['plain'][1]:.3f}, {med['plain'][2]:.3f}], "
                  f"skip {med['skip'][0]:.3f} ms [{med['skip'][1]:.3f}, {med['skip'][2]:.3f}], "
                  f"ratio {med['skip'][0] / med['plain'][0]:.3f}, evaluated coarse {frac[0]:.3f} fine {frac[1]:.3f}")
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
