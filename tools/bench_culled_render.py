"""Device time of a full-image render with and without empty-space skipping (nerf_pl_b200.culling) on the trained
test weights.

Full 400 x 400 and 800 x 800 Blender-style views of the trained scene (radius-4 camera, near 2, far 6, 64 + 128
samples by default).  In one process, after warm-up, ``batched_inference`` is timed with and without the occupancy
grid in alternation, CUDA events around each call, several rounds; the median of each leg is reported as ms per
image, with the live fraction and the separate cost of cull (classify + compact) and scatter; a third leg uses a
grid with every cell occupied, the view culling cannot help.  The per-ray cost of
the cull is set against the bytes it has to move (32 B read per ray, 1 B flag, and per live ray 8 B index + 32 B
ray written).  Prints the card name and power limit beside the numbers and one JSON line.  Needs a GPU: there is
no CPU fallback.
Run: python tools/bench_culled_render.py [--sides 400 800] [--rounds 7] [--views 3] [--grid 128]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import nerf_pl_b200 as nb  # noqa: E402
from tests import cases  # noqa: E402

RANGE = (-1.5, 1.5)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sides", type=int, nargs="+", default=[400, 800])
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--views", type=int, default=3)
    ap.add_argument("--grid", type=int, default=128)
    ap.add_argument("--sigma-threshold", type=float, default=1.0)
    ap.add_argument("--dilate", type=int, default=1)
    ap.add_argument("--n-importance", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_culled_render.py needs a CUDA device (no CPU fallback)")
    models = []
    for w in cases.trained_weights():
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        models.append(m.cuda().eval())
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    res = {"card": card(), "grid": args.grid, "sigma_threshold": args.sigma_threshold, "dilate": args.dilate,
           "samples": [64, args.n_importance]}
    print("card, power limit:", res["card"])
    ms_grid, grid = event_ms(lambda: nb.occupancy_grid(models[1], args.grid, RANGE, RANGE, RANGE, args.sigma_threshold,
                                                       args.dilate))
    ms_grid, grid = event_ms(lambda: nb.occupancy_grid(models[1], args.grid, RANGE, RANGE, RANGE, args.sigma_threshold,
                                                       args.dilate))
    res["grid_build_ms"] = ms_grid
    res["occupied_fraction"] = grid.occupied_fraction()
    print(f"occupancy grid N {args.grid}, sigma > {args.sigma_threshold}, dilate {args.dilate}: built in {ms_grid:.1f} ms, "
          f"{res['occupied_fraction']:.4f} of the cells occupied")

    # every cell occupied: the rays that meet the box are all live, which prices the cull + scatter on a view it cannot help
    full = nb.occupancy_grid(models[1], args.grid, RANGE, RANGE, RANGE, -1.0, 0)

    def render(rays, occupancy):
        return nb.batched_inference(models, emb, rays, 64, args.n_importance, False, 32768, True, occupancy=occupancy)

    for side in args.sides:
        views = [torch.from_numpy(bench.blender_rays(0, 70 + v, W=side, H=side, pixels="all")).cuda()
                 for v in range(args.views)]
        n = side * side
        for rays in views:                                      # warm every shape both legs will launch
            render(rays, None)
            render(rays, grid)
            render(rays, full)
        torch.cuda.synchronize()
        plain, culled, cull, scatter, live, err, mostly, mostly_live = [], [], [], [], [], 0.0, [], []
        for _ in range(args.rounds):
            for rays in views:
                ms_p, out_p = event_ms(lambda: render(rays, None))
                ms_c, out_c = event_ms(lambda: render(rays, grid))
                ms_f, out_f = event_ms(lambda: render(rays, full))
                mostly.append(ms_f)
                mostly_live.append(out_f["live"] / n)
                plain.append(ms_p)
                culled.append(ms_c)
                live.append(out_c["live"] / n)
                err = max(err, float((out_c["rgb_fine"] - out_p["rgb_fine"]).abs().max()))
                ms_k, (idx, live_rays) = event_ms(lambda: nb.cull_rays(rays, grid))
                compact = {k: v[idx].contiguous() for k, v in out_p.items()}
                ms_s, _ = event_ms(lambda: nb.scatter_results(compact, idx, n, True))
                cull.append(ms_k)
                scatter.append(ms_s)
        med = statistics.median
        cull_bytes = n * 33 + med(live) * n * 40
        r = {"rays": n, "plain_ms": med(plain), "culled_ms": med(culled), "plain_ms_min_max": [min(plain), max(plain)],
             "culled_ms_min_max": [min(culled), max(culled)], "live_fraction": med(live),
             "live_fraction_min_max": [min(live), max(live)], "cull_ms": med(cull), "scatter_ms": med(scatter),
             "cull_GB_per_s": cull_bytes / (med(cull) * 1e-3) / 1e9, "speedup": med(plain) / med(culled),
             "max_abs_rgb_difference": err, "full_grid_ms": med(mostly), "full_grid_live_fraction": med(mostly_live)}
        res[f"{side}x{side}"] = r
        print(f"{side} x {side} ({args.views} views x {args.rounds} rounds, medians): plain {r['plain_ms']:.2f} ms/image, "
              f"culled {r['culled_ms']:.2f} ms/image (x{r['speedup']:.2f}), live fraction {r['live_fraction']:.3f}; "
              f"cull {r['cull_ms']:.3f} ms ({r['cull_GB_per_s']:.0f} GB/s of its minimum traffic), scatter "
              f"{r['scatter_ms']:.3f} ms; max |rgb_fine difference| {err:.2e}; with every cell occupied (live fraction "
              f"{r['full_grid_live_fraction']:.3f}) {r['full_grid_ms']:.2f} ms/image")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
