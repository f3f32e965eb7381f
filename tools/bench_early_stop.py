"""What early ray termination (DESIGN.md §10f, ``early_stop=``) saves on coarse-only renders of the trained test scene.

tools/early_stop_ceiling.py's set-up: the trained test network (its coarse net renders, the fine net makes the
grid), the tests' grid (N = 128 over [-1.5, 1.5]^3, sigma > 1, dilate 1), Blender views 80-82 with a white
background.  For each shape (128 + 0, 64 + 0), size and test_time, ``render_rays_culled(..., skip="samples")`` with
early_stop = 0 and each eps is timed, the arms alternated in one process: CUDA events around each call (the call
ends in a device synchronise), median [min, max] over views x rounds after one warm-up of each arm.  Beside each time:
the evaluated coarse samples as a fraction of all samples, and the fraction eps drops from early_stop = 0 (§10f's
"word" column).  It also times the device-to-host read-back termination adds once per mask word (a one-element
copy and a stream synchronise, median over 200), and ``fuse_vertex_colors`` of bench_mesh_grid.py's N = 256 mesh
over --views views with eps = 0.5 against 0.  The card's name and power limit are read in the same run.

    python tools/bench_early_stop.py [--sizes 400,800] [--shapes 128+0,64+0] [--eps 1e-4,1e-3,1e-2] [--rounds 5]
                                     [--views 100] [--out FILE]
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

CUBE = ((-1.5, 1.5),) * 3


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
    return float(np.median(v)), float(np.min(v)), float(np.max(v))


def _fmt(t):
    return f"{t[0]:.2f} ms [{t[1]:.2f}, {t[2]:.2f}]"


def readback_us(reps=200):
    """Median cost of one sample-count read-back: a one-element device-to-host copy and a stream synchronise."""
    src = torch.zeros(1, dtype=torch.int64, device="cuda")
    dst = torch.zeros(1, dtype=torch.int64).pin_memory()
    t = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        dst.copy_(src, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        t.append((time.perf_counter() - t0) * 1e6)
    return float(np.median(t))


def renders(a, models, emb, grid, eps_list):
    runs = []
    for shape in a.shapes.split(","):
        S, K = (int(v) for v in shape.split("+"))
        for side in [int(s) for s in a.sizes.split(",")]:
            views = [torch.from_numpy(bench.blender_rays(0, 80 + v, W=side, H=side, pixels="all")).cuda()
                     for v in range(3)]
            for test_time in (False, True):
                arms = [0.0] + eps_list

                def render(rays, eps):
                    return nb.render_rays_culled(models[:1], emb, rays, grid, S, False, K, True, test_time,
                                                 skip="samples", early_stop=eps)
                live = {e: [render(r, e)["live_samples"][0] for r in views] for e in arms}      # also the warm-up
                torch.cuda.synchronize()
                times = {e: [] for e in arms}
                for _ in range(a.rounds):
                    for rays in views:
                        for e in arms:
                            times[e].append(_ms(lambda: render(rays, e)))
                n = views[0].shape[0]
                live_chunks = [-(-int(nb.cull_rays(r, grid)[0].numel()) // culling._SAMPLE_CHUNK) for r in views]
                run = {"S": S, "K": K, "side": side, "test_time": test_time, "readbacks_per_render_eps0":
                       [c for c in live_chunks], "readbacks_per_render_eps": [c * (S // 32) for c in live_chunks],
                       "arms": {}}
                for e in arms:
                    run["arms"][f"{e:g}"] = {"ms": _stats(times[e]),
                                             "evaluated": [lv / (n * S) for lv in live[e]],
                                             "dropped": [1 - lv / max(l0, 1) for lv, l0 in zip(live[e], live[0.0])]}
                runs.append(run)
                base = run["arms"]["0"]["ms"]
                print(f"{S} + {K} at {side} x {side}, test_time={int(test_time)}: early_stop=0 {_fmt(base)}, "
                      f"evaluated {' / '.join(f'{x:.3f}' for x in run['arms']['0']['evaluated'])}")
                for e in eps_list:
                    r = run["arms"][f"{e:g}"]
                    print(f"  eps {e:g}: {_fmt(r['ms'])} ({r['ms'][0] / base[0]:.3f} x median, median below the "
                          f"eps=0 minimum: {r['ms'][0] < base[1]}); dropped "
                          f"{' / '.join(f'{100 * x:.1f}' for x in r['dropped'])} % of the evaluated samples")
            del views
            torch.cuda.empty_cache()
    return runs


def fuse(a, fine, grid):
    v, _ = nb.extract_mesh(fine, 256, *CUBE, 20.0)
    rng = np.random.default_rng(0)             # bench_mesh.py's views: radius-4 cameras, focal 1111, near 2
    images = torch.from_numpy(rng.integers(0, 256, (a.views, 800, 800, 3), dtype=np.uint8)).cuda()
    eyes = rng.normal(size=(a.views, 3))
    poses = [_look_at(e) for e in eyes / np.linalg.norm(eyes, axis=1, keepdims=True) * 4.0]
    arms = {e: (lambda e=e: nb.fuse_vertex_colors(fine, v, images, poses, 1111.0, 2.0, occupancy=grid, early_stop=e))
            for e in (0.0, 0.5)}
    same = bool(torch.equal(arms[0.0](), arms[0.5]()))
    times = {e: [] for e in arms}
    for _ in range(max(1, a.rounds // 2)):
        for e, f in arms.items():
            times[e].append(_ms(f))
    out = {"vertices": int(v.shape[0]), "views": a.views, "colours_identical": same,
           "ms": {f"{e:g}": _stats(t) for e, t in times.items()}}
    print(f"fuse_vertex_colors, {a.views} views x {v.shape[0]} vertices: early_stop=0 {_fmt(out['ms']['0'])}, "
          f"0.5 {_fmt(out['ms']['0.5'])}; colours identical: {same}")
    return out


def _look_at(eye):
    eye = np.asarray(eye, np.float64)
    f = -eye / np.linalg.norm(eye)
    r = np.cross(f, [0, 0, 1.0])
    r /= np.linalg.norm(r)
    return np.stack([r, np.cross(r, f), -f, eye], 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="400,800")
    ap.add_argument("--shapes", default="128+0,64+0")
    ap.add_argument("--eps", default="1e-4,1e-3,1e-2")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--views", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_early_stop needs a CUDA device")
    gpu = _gpu()
    models = []
    for w in cases.trained_weights():
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        models.append(m.cuda().eval())
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    grid = nb.occupancy_grid(models[1], 128, *CUBE, 1.0, 1)
    print(f"on {gpu}")
    rb = readback_us()
    print(f"one sample-count read-back (1-element copy + stream synchronise): {rb:.1f} us median")
    report = {"gpu": gpu, "readback_us": rb,
              "renders": renders(a, models, emb, grid, [float(e) for e in a.eps.split(",")])}
    if a.views > 0:
        report["fuse_vertex_colors"] = fuse(a, models[1], grid)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
