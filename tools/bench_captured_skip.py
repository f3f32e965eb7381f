"""The training step captured as one CUDA graph, with and without empty samples skipped.

Workloads: eager plain (render_rays_loss + backward + FusedAdam(capturable=True)), captured plain
(CapturedTrainStep), eager skip (the same with occupancy=grid) and captured skip (CapturedTrainStep(occupancy=grid)),
at 1024 and 4096 rays and 64 + 64 and 64 + 128 samples.  The networks are the trained test scene's
(tests/golden/trained_weights), the grid is the tests' (N = 128 over [-1.5, 1.5]^3, sigma > 1, dilate 1, from the
fine network); rays are random pixels of Blender-style views (radius-4 camera, near 2, far 6) with random targets,
perturb 1, noise_std 1, in-kernel random numbers.  The workloads alternate within each round; reported are the median
and range over rounds of the mean step time, and the card's name and power limit read in the same run.

--parent DIR also times the eager skip step of the package under DIR (a build of the tree before the device-planned
pipeline) in a subprocess, between the two halves of each shape's rounds.

    python tools/bench_captured_skip.py [--rounds 5] [--steps 30] [--parent DIR] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(n, S, K) for n in (1024, 4096) for S, K in ((64, 64), (64, 128))]
DATASET = 16                        # batches per epoch of the captured steps' ray set


def _gpu():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def _setup(n, S, K):
    import torch

    import nerf_pl_b200 as nb                        # before bench, which puts this tree first on sys.path
    import bench
    from tests import cases
    models = []
    for w in cases.trained_weights():
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        models.append(m.cuda())
    with torch.no_grad():
        grid = nb.occupancy_grid(models[1], 128, (-1.5, 1.5), (-1.5, 1.5), (-1.5, 1.5), 1.0, 1)
    rays = torch.from_numpy(bench.blender_rays(n * DATASET, 7))
    rgbs = torch.rand(n * DATASET, 3, generator=torch.Generator().manual_seed(0))
    return nb, torch, models, grid, rays, rgbs


def _eager(nb, torch, models, rays, rgbs, S, K, grid):
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    opt = nb.FusedAdam([p for m in models for p in m.parameters()], lr=5e-4, capturable=True)
    n = rays.shape[0] // DATASET
    r, c = rays[:n].cuda(), rgbs[:n].cuda()

    def step():
        opt.zero_grad(set_to_none=True)
        res = nb.render_rays_loss(models, emb, r, c, S, False, 1.0, 1.0, K, 32768, True, randoms="kernel",
                                  occupancy=grid)
        res["loss"].backward()
        opt.step()
    return step


def _captured(nb, torch, models, rays, rgbs, S, K, grid):
    batches = nb.DeviceRayBatches(rays, rgbs, batch_size=rays.shape[0] // DATASET, seed=1)
    opt = nb.FusedAdam([p for m in models for p in m.parameters()], lr=5e-4, capturable=True)
    st = nb.CapturedTrainStep(models, batches, opt, S, False, 1.0, 1.0, K, True, randoms={"seed": 3},
                              occupancy=grid)
    return st.step


def _time(torch, fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def parent_worker(a):
    """Eager skip steps of one shape with the package found first on sys.path (the parent's): one JSON line of
    per-round times."""
    n, S, K = (int(x) for x in a.shape.split(","))
    nb, torch, models, grid, rays, rgbs = _setup(n, S, K)
    if not os.path.abspath(nb.__file__).startswith(os.path.abspath(a.parent) + os.sep):
        raise RuntimeError(f"imported {nb.__file__}, not the package under {a.parent}")
    fn = _eager(nb, torch, models, rays, rgbs, S, K, grid)
    fn()
    print(json.dumps([_time(torch, fn, a.steps) for _ in range(a.rounds)]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--parent", default=None)
    ap.add_argument("--parent-worker", action="store_true")
    ap.add_argument("--shape", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.parent_worker:
        sys.path.insert(0, ROOT)
        sys.path.insert(0, os.path.abspath(a.parent))
        parent_worker(a)
        return
    sys.path.insert(0, ROOT)
    gpu = _gpu()
    report = {"gpu": gpu, "cases": {}}
    for n, S, K in SHAPES:               # one shape at a time: its four workspaces and graphs, then freed
        nb, torch, models, grid, rays, rgbs = _setup(n, S, K)
        fns = {"eager plain": _eager(nb, torch, models, rays, rgbs, S, K, None),
               "captured plain": _captured(nb, torch, models, rays, rgbs, S, K, None),
               "eager skip": _eager(nb, torch, models, rays, rgbs, S, K, grid),
               "captured skip": _captured(nb, torch, models, rays, rgbs, S, K, grid)}
        for f in fns.values():
            f()
        times = {k: [] for k in fns}
        for h, rounds in enumerate(((a.rounds + 1) // 2, a.rounds // 2)):
            for _ in range(rounds):
                for k, f in fns.items():
                    times[k].append(_time(torch, f, a.steps))
            if h == 0 and a.parent:
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--parent-worker", "--parent", a.parent,
                                    "--shape", f"{n},{S},{K}", "--rounds", str(a.rounds), "--steps", str(a.steps)],
                                   capture_output=True, text=True, cwd=ROOT)
                if p.returncode != 0:
                    raise RuntimeError(p.stderr[-3000:])
                times["parent eager skip"] = json.loads(p.stdout.strip().splitlines()[-1])
        del fns
        from nerf_pl_b200.train_skip import SkipTrainWorkspace
        from nerf_pl_b200.training import TrainWorkspace
        SkipTrainWorkspace.clear()
        TrainWorkspace.clear()
        torch.cuda.empty_cache()
        key = f"{n} rays, {S}+{K}"
        med = {k: (float(np.median(v)), float(np.min(v)), float(np.max(v))) for k, v in times.items()}
        report["cases"][key] = med
        print(f"{key} on {gpu}: " + ", ".join(f"{k} {m[0]:.3f} ms [{m[1]:.3f}, {m[2]:.3f}]" for k, m in med.items()),
              flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
