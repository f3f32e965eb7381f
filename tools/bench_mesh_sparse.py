"""Sparse marching cubes through an occupancy grid (nb.sparse_marching_cubes, the route of nb.extract_mesh(...,
occupancy=)) against the dense masked route, marching_cubes(sigma_grid(..., occupancy=)), DESIGN.md §10i.

On the trained test weights with the grid of the trained scene (nb.occupancy_grid of the fine network, N = 128 over
[-1.5, 1.5]^3, sigma > 1, dilate 1), threshold 20:

1. dense against sparse at N_grid in --compare (CUDA events around one call of each; one warm-up each, then the two
   arms alternate over --rounds rounds; median and range over the rounds);
2. the sparse route alone at N_grid in --sparse (one warm-up, --rounds timed calls);
3. per N_grid, the sparse route's time per stage from torch.profiler's kernel times in a run of its own (plan: brick
   selection; sigma: compaction, the point query and the scatter; march: count, key emission and resolution; sort:
   the radix sorts), its peak device memory above the start (torch.cuda.max_memory_allocated: the workspaces are
   torch tensors), the active and march bricks, and the vertex and triangle counts.

The card's name and power limit are read in the same run.

    python tools/bench_mesh_sparse.py [--compare 256,512] [--sparse 1024,1536,2048] [--rounds 5] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nerf_pl_b200 as nb  # noqa: E402
from tests import cases  # noqa: E402

BOX = ((-1.5, 1.5),) * 3
THRESHOLD = 20.0


def _gpu():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def _ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def _stats(v):
    return (float(np.median(v)), float(np.min(v)), float(np.max(v)))


def _fmt(t):
    return f"{t[0]:.1f} ms [{t[1]:.1f}, {t[2]:.1f}]"


def _stage(name):
    if any(s in name for s in ("smc_candidate", "smc_classify", "smc_map", "smc_march_flag", "Select")):
        return "plan"
    if any(s in name for s in ("RadixSort", "Onesweep", "radix")):
        return "sort"
    if any(s in name for s in ("smc_march", "smc_vertices", "smc_triangles", "Scan")):
        return "march"
    return "sigma"


def _stages(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {"plan": 0.0, "sigma": 0.0, "march": 0.0, "sort": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t and e.key and not e.key.startswith("Memcpy") and not e.key.startswith("Memset"):
            out[_stage(e.key)] += t / 1000.0
    return out


def _bricks(fine, grid, N):
    lib = nb._lib.load()
    plan = nb._lib.workspace(lib.nerfb200_sparse_mc_plan_workspace_bytes(N), "cuda")
    bricks = (ctypes.c_int64 * 2)()
    nb._lib.call("nerfb200_sparse_mc_plan", torch.device("cuda"), N, nb._lib.ranges_host(*BOX), grid.bits.data_ptr(),
                 grid.grid_n(), (ctypes.c_double * 6)(*grid.ranges), plan.data_ptr(), plan.numel(), bricks)
    return int(bricks[0]), int(bricks[1]), -(-N // 8) ** 3


def _sparse_row(fine, grid, N, rounds):
    sparse = lambda: nb.sparse_marching_cubes(fine, N, *BOX, THRESHOLD, occupancy=grid)  # noqa: E731
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    v, t = sparse()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    r = {"vertices": int(v.shape[0]), "triangles": int(t.shape[0]), "peak_bytes": int(peak)}
    del v, t
    r["active_bricks"], r["march_bricks"], r["bricks"] = _bricks(fine, grid, N)
    r["stages_ms"] = _stages(sparse)
    return r, sparse


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--compare", default="256,512")
    ap.add_argument("--sparse", default="1024,1536,2048")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh_sparse.py needs a CUDA device")
    gpu = _gpu()
    ws = cases.trained_weights()[1]
    fine = nb.NeRF()
    fine.load_state_dict({k: torch.from_numpy(v) for k, v in ws.items()})
    fine = fine.cuda().eval()
    grid = nb.occupancy_grid(fine, 128, *BOX, 1.0, dilate=1)
    report = {"gpu": gpu, "occupied_cells": grid.occupied_fraction(), "rows": {}}
    print(f"on {gpu}: grid of the trained scene, N = 128, {report['occupied_cells']:.4f} of the cells occupied")
    for N in (int(s) for s in a.compare.split(",") if s):
        r, sparse = _sparse_row(fine, grid, N, a.rounds)
        dense = lambda: nb.marching_cubes(nb.sigma_grid(fine, N, *BOX, occupancy=grid), THRESHOLD)  # noqa: E731
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        dense()
        torch.cuda.synchronize()
        r["dense_peak_bytes"] = int(torch.cuda.max_memory_allocated() - base)
        dense(), sparse()
        times = {"dense": [], "sparse": []}
        for _ in range(a.rounds):
            times["dense"].append(_ms(dense))
            times["sparse"].append(_ms(sparse))
        r["dense_ms"], r["sparse_ms"] = _stats(times["dense"]), _stats(times["sparse"])
        report["rows"][N] = r
        print(f"N_grid {N}: dense {_fmt(r['dense_ms'])} peak {r['dense_peak_bytes'] / 2 ** 30:.2f} GiB; sparse "
              f"{_fmt(r['sparse_ms'])} peak {r['peak_bytes'] / 2 ** 30:.2f} GiB; stages {r['stages_ms']}; "
              f"bricks {r['active_bricks']} active / {r['march_bricks']} march / {r['bricks']}; "
              f"V {r['vertices']} T {r['triangles']}")
    for N in (int(s) for s in a.sparse.split(",") if s):
        r, sparse = _sparse_row(fine, grid, N, a.rounds)
        sparse()
        r["sparse_ms"] = _stats([_ms(sparse) for _ in range(a.rounds)])
        report["rows"][N] = r
        print(f"N_grid {N}: sparse {_fmt(r['sparse_ms'])} peak {r['peak_bytes'] / 2 ** 30:.2f} GiB; stages "
              f"{r['stages_ms']}; bricks {r['active_bricks']} active / {r['march_bricks']} march / {r['bricks']}; "
              f"V {r['vertices']} T {r['triangles']}")
    line = json.dumps(report)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
