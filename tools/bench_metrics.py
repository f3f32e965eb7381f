"""Device time of nb.ssim and nb.visualize_depth at 400 x 400 and 800 x 800, next to the reference's host
visualize_depth (utils/visualization.py) in the same process.

CUDA events around each call, after warm-up; the median over --rounds is reported.  SSIM is timed on a (1, 3, H, W)
image held the way train.py holds it (``rgb.view(H, W, 3).permute(2, 0, 1)[None]``), for 'mean' and 'none'.

The host leg runs the reference's own, unmodified ``utils/visualization.py``, loaded by path (its package's
``__init__`` would pull in the optimisers) from the first of ``--reference``, ``$NERF_PL_REFERENCE`` and
``oracle/_ref`` (the git-ignored directory where reference files are staged) that holds it.  Its time includes the
``depth.cpu()`` device-to-host copy; a separate cProfile pass, outside the timed calls, reports which calls the host
time goes to.  Without the file, or without cv2, PIL or torchvision, the host leg is skipped and says so.  Prints the
card name and power limit beside the numbers and one JSON line.  Needs a GPU: there is no CPU fallback.
Run: python tools/bench_metrics.py [--sides 400 800] [--rounds 50] [--reference /path/to/nerf_pl]
"""
import argparse
import cProfile
import importlib.util
import json
import os
import pstats
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nerf_pl_b200 as nb  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def event_ms(fn, rounds):
    """Median device time of fn over `rounds` calls, each between two events."""
    times = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def reference_visualize_depth(candidates):
    """The reference's visualize_depth from the first candidate checkout holding utils/visualization.py, as
    (function, path), or (None, reason)."""
    for ref in candidates:
        path = os.path.join(ref, "utils", "visualization.py") if ref else ""
        if path and os.path.exists(path):
            try:
                spec = importlib.util.spec_from_file_location("reference_visualization", path)
                mod = importlib.util.module_from_spec(spec)
                spec.loader.exec_module(mod)
            except ImportError as e:
                return None, f"{path} does not import here: {e}"
            return mod.visualize_depth, path
    return None, "no utils/visualization.py in " + ", ".join(c for c in candidates if c)


def host_profile(fn, rounds, top=5):
    """[(call, ms per visualize_depth call)] of the `top` calls with the most own time, over `rounds` calls."""
    prof = cProfile.Profile()
    prof.enable()
    for _ in range(rounds):
        fn()
    prof.disable()
    st = pstats.Stats(prof).stats
    rows = sorted(((v[2], k) for k, v in st.items()), reverse=True)[:top]
    return [(f"{os.path.basename(k[0])}:{k[2]}" if k[0] != "~" else k[2], 1e3 * t / rounds) for t, k in rows]


def host_ms(fn, rounds):
    """Host clock around each call, after a device synchronise: (median, min, max) in ms."""
    times = []
    for _ in range(rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(times), min(times), max(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sides", type=int, nargs="+", default=[400, 800])
    ap.add_argument("--rounds", type=int, default=50)
    ap.add_argument("--reference", default=None, help="a nerf_pl checkout (default: $NERF_PL_REFERENCE, oracle/_ref)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_metrics.py needs a CUDA device (no CPU fallback)")
    res = {"card": card()}
    print("card, power limit:", res["card"])
    host, where = reference_visualize_depth([args.reference, os.environ.get("NERF_PL_REFERENCE"),
                                             os.path.join(ROOT, "oracle", "_ref")])
    res["host_reference"] = where
    print("reference visualize_depth:", where if host is not None else f"not timed ({where})")
    g = torch.Generator(device="cuda").manual_seed(0)
    for side in args.sides:
        n = side * side
        rgb = torch.rand(n, 3, device="cuda", generator=g)
        gt = (rgb + 0.05 * torch.randn(n, 3, device="cuda", generator=g)).clamp(0, 1)
        pred_img, gt_img = (t.view(side, side, 3).permute(2, 0, 1)[None] for t in (rgb, gt))
        depth = (2.0 + 4.0 * torch.rand(n, device="cuda", generator=g)).view(side, side)
        for _ in range(5):                                       # warm-up
            nb.ssim(pred_img, gt_img)
            nb.ssim(pred_img, gt_img, "none")
            nb.visualize_depth(depth)
        torch.cuda.synchronize()
        r = {"ssim_mean_ms": event_ms(lambda: nb.ssim(pred_img, gt_img), args.rounds),
             "ssim_none_ms": event_ms(lambda: nb.ssim(pred_img, gt_img, "none"), args.rounds),
             "visualize_depth_ms": event_ms(lambda: nb.visualize_depth(depth), args.rounds)}
        # bytes each call must move: two fp32 images read (+ the fp32 map written for 'none'); the depth map read and
        # twice (min / max pass, colour pass), the (3, H, W) fp32 image written
        r["ssim_mean_GB_per_s"] = 2 * 3 * n * 4 / (r["ssim_mean_ms"] * 1e-3) / 1e9
        r["visualize_depth_GB_per_s"] = (2 * n * 4 + 3 * n * 4) / (r["visualize_depth_ms"] * 1e-3) / 1e9
        if host is not None:
            for _ in range(3):
                host(depth)
            r["host_visualize_depth_ms"], lo, hi = host_ms(lambda: host(depth), max(10, args.rounds // 2))
            r["host_visualize_depth_ms_min_max"] = [lo, hi]
            same = torch.equal(host(depth), nb.visualize_depth(depth).cpu())
            r["host_equals_device"] = same
            r["host_profile_ms_per_call"] = host_profile(lambda: host(depth), max(5, args.rounds // 5))
        res[f"{side}x{side}"] = r
        line = (f"{side} x {side}: ssim mean {r['ssim_mean_ms']:.4f} ms, ssim none {r['ssim_none_ms']:.4f} ms, "
                f"visualize_depth {r['visualize_depth_ms']:.4f} ms")
        if host is not None:
            line += (f"; reference host visualize_depth {r['host_visualize_depth_ms']:.3f} ms "
                     f"(min {lo:.3f}, max {hi:.3f}; equal: {r['host_equals_device']})")
        print(line)
        if host is not None:
            print("  reference host time by call (own time, ms per visualize_depth call): " +
                  ", ".join(f"{k} {v:.2f}" for k, v in r["host_profile_ms_per_call"]))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
