"""Rendering from a baked volume (nb.bake_volume, nb.render_baked, DESIGN.md §10j) against the MLP renders of the same
views, on the trained test scene: the trained test network (its fine net is baked and makes the grid), the tests' grid
(nb.occupancy_grid, N = 128 over [-1.5, 1.5]^3, sigma > 1, dilate 1), Blender views 80-82 with a white background.

1. per N in --N: the bake's time (CUDA events around one call after one warm-up; median [min, max] over --rounds),
   its stored bricks and bytes;
2. per N, at --side x --side: render_baked eager and replayed from a CUDA graph, and, for comparison on the same
   views, render_image(..., occupancy=grid, skip="samples") at 64 + 128 and at 128 + 0 with early_stop=1e-3.  The
   arms alternate view by view within each round; median [min, max] over views x rounds after one warm-up of each;
3. per N, the PSNR of the baked render against the 64 + 128 MLP render and against the analytic ground truth of
   tools/train_sharp_weights.py (whose colour does not depend on the view, which favours a bake with direction 0).

The card's name and power limit are read in the same run.

    python tools/bench_baked.py [--N 256,512,1024,2048] [--side 800] [--rounds 5] [--out FILE]
"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import nerf_pl_b200 as nb  # noqa: E402
from tests import cases  # noqa: E402

BOX = ((-1.5, 1.5),) * 3


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
    return f"{t[0]:.2f} ms [{t[1]:.2f}, {t[2]:.2f}]"


def _psnr(a, b):
    return float(-10 * torch.log10(((a - b) ** 2).mean()))


def _ground_truth():
    spec = importlib.util.spec_from_file_location("train_sharp_weights", os.path.join(ROOT, "tools",
                                                                                       "train_sharp_weights.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.ground_truth


def _pose(seed, side):
    """bench.blender_rays' camera of view `seed` as a c2w and focal for render_image / generate_rays."""
    rs = np.random.RandomState(seed)
    focal = 0.5 * side / np.tan(0.5 * bench.CAMERA_ANGLE_X)
    th, ph = rs.uniform(0, 2 * np.pi), rs.uniform(np.pi / 6, np.pi / 3)
    cam = 4.0 * np.array([np.cos(th) * np.sin(ph), np.sin(th) * np.sin(ph), np.cos(ph)])
    fwd = -cam / np.linalg.norm(cam)
    right = np.cross(fwd, np.array([0.0, 0.0, 1.0]))
    right /= np.linalg.norm(right)
    up = np.cross(right, fwd)
    return np.stack([right, up, -fwd, cam], 1).astype(np.float32), float(focal)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", default="256,512,1024,2048")
    ap.add_argument("--side", type=int, default=800)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_baked.py needs a CUDA device")
    gpu = _gpu()
    models = []
    for w in cases.trained_weights():
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        models.append(m.cuda().eval())
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    fine = models[1]
    grid = nb.occupancy_grid(fine, 128, *BOX, 1.0, dilate=1)
    side = a.side
    views = [_pose(80 + v, side) for v in range(3)]
    rays = [nb.generate_rays(side, side, f, c2w, 2.0, 6.0) for c2w, f in views]
    gt = _ground_truth()
    truth = [gt(r) for r in rays]
    report = {"gpu": gpu, "side": side, "rounds": a.rounds, "mlp": {}, "baked": {}}
    print(f"on {gpu}: trained scene, grid N = 128 ({grid.occupied_fraction():.4f} occupied), {side} x {side}")

    mlp = {"64+128": lambda v: nb.render_image(models, emb, side, side, views[v][1], views[v][0], 2.0, 6.0, 64, 128,
                                               white_back=True, occupancy=grid, skip="samples"),
           "128+0 eps1e-3": lambda v: nb.render_image(models, emb, side, side, views[v][1], views[v][0], 2.0, 6.0, 128,
                                                      0, white_back=True, occupancy=grid, skip="samples",
                                                      early_stop=1e-3)}
    ref = [mlp["64+128"](v)["rgb"].reshape(-1, 3) for v in range(3)]
    report["mlp_psnr_vs_truth"] = [_psnr(ref[v], truth[v]) for v in range(3)]
    times = {k: [] for k in mlp}
    for k in mlp:
        mlp[k](0)
    for _ in range(a.rounds):
        for v in range(3):
            for k, fn in mlp.items():
                times[k].append(_ms(lambda: fn(v)))
    for k in mlp:
        report["mlp"][k] = _stats(times[k])
        print(f"MLP {k}: {_fmt(report['mlp'][k])}")
    print(f"MLP 64+128 PSNR vs ground truth: {report['mlp_psnr_vs_truth']}")

    for N in (int(s) for s in a.N.split(",") if s):
        torch.cuda.empty_cache()
        try:
            bake = lambda: nb.bake_volume(fine, N, *BOX, occupancy=grid)  # noqa: E731
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            vol = bake()                   # the warm-up, and the call's peak above its start (volume included)
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated() - base
            tb = []
            for _ in range(a.rounds):
                del vol
                held = []
                tb.append(_ms(lambda: held.append(bake())))
                vol = held[0]
        except torch.cuda.OutOfMemoryError:
            print(f"N {N}: the bake does not fit")
            report["baked"][N] = {"fits": False}
            continue
        r = {"bake_ms": _stats(tb), "bricks": vol.bricks, "bytes": vol.nbytes, "bake_peak_bytes": int(peak),
             "map_slots": (-(-N // 8)) ** 3}
        render = lambda v: nb.render_baked(vol, rays[v], white_back=True)  # noqa: E731
        static = rays[0].clone()
        render(0)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            nb.render_baked(vol, static, white_back=True)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            gout = nb.render_baked(vol, static, white_back=True)
        te, tg = [], []
        for _ in range(a.rounds):
            for v in range(3):
                te.append(_ms(lambda: render(v)))
                static.copy_(rays[v])
                tg.append(_ms(g.replay))
        assert torch.equal(gout["rgb"], render(2)["rgb"])
        r["render_ms"], r["graph_ms"] = _stats(te), _stats(tg)
        out = [render(v)["rgb"] for v in range(3)]
        r["psnr_vs_mlp"] = [_psnr(out[v], ref[v]) for v in range(3)]
        r["psnr_vs_truth"] = [_psnr(out[v], truth[v]) for v in range(3)]
        r["speedup_vs_64_128"] = report["mlp"]["64+128"][0] / r["render_ms"][0]
        r["speedup_vs_128_0"] = report["mlp"]["128+0 eps1e-3"][0] / r["render_ms"][0]
        report["baked"][N] = r
        print(f"N {N}: bake {_fmt(r['bake_ms'])}, {r['bricks']} bricks of {r['map_slots']}, "
              f"{r['bytes'] / 2 ** 20:.1f} MiB (bake peak {peak / 2 ** 30:.2f} GiB); render eager {_fmt(r['render_ms'])}, "
              f"graph {_fmt(r['graph_ms'])} ({r['speedup_vs_64_128']:.1f}x / {r['speedup_vs_128_0']:.1f}x the MLP "
              f"64+128 / 128+0); PSNR vs MLP {[round(p, 2) for p in r['psnr_vs_mlp']]}, vs truth "
              f"{[round(p, 2) for p in r['psnr_vs_truth']]}")
        del vol, g, gout
    line = json.dumps(report)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
