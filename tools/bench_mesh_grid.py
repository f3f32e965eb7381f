"""Mesh and Unity-volume grids through an occupancy grid (occupancy= of nb.sigma_grid, nb.rgb_sigma_grid,
nb.fuse_vertex_colors, nb.normal_vertex_colors): what the mask costs or saves, and what it changes for a network
trained with a density grid.

1. Speed, on the trained test weights with the grid of the trained scene (nb.occupancy_grid of the fine network,
N = 128 over [-1.5, 1.5]^3, sigma > 1, dilate 1).  Plain against masked sigma_grid and rgb_sigma_grid at N in --grids;
fuse_vertex_colors of the N = 256 kept mesh over --views views at 800 x 800 (bench_mesh.py's views); and
normal_vertex_colors of the N = 512 kept mesh (64 + 64 samples, near 2, far 6, white background).  CUDA events
around one call; the two arms alternate over --rounds rounds after a warm-up of each, and the median and range are
over the rounds.

2. --train.  From-scratch captured training on bench_density_grid.py's scene and recipe (64 + 64 samples, perturb 1,
noise 1, Adam 5e-4, in-kernel randoms, 1024-ray batches, --train-steps steps): plain, and W = 500 plain steps then
CapturedTrainStep(occupancy=DensityGrid(128, box, 1.0, decay 0.95, dilate 1), update_every=16).  Then the N = 256
mesh at threshold 20 of each network, without a grid and with one: the density grid for the grid-trained network,
nb.occupancy_grid (as above) for the plain one.  Reported per mesh: components before the cluster filter, kept
vertices, the kept mesh's distance to the analytic spheres (median / p99 / max, as tests/test_gpu_mesh_field.py
measures it), and the mean |d| of the vertex-normal colours (uint8 / 255) against train_sharp_weights.ground_truth on
the same rays.  One run per arm.

The card's name and power limit are read in the same run.

    python tools/bench_mesh_grid.py [--grids 256,512] [--views 100] [--rounds 5] [--out FILE]
    python tools/bench_mesh_grid.py --train [--train-steps 3000] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
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


def _alternate(fns, rounds):
    """{name: (median, min, max) ms}: one warm-up call of each, then the arms in turn, `rounds` times."""
    for f in fns.values():
        f()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            times[k].append(_ms(f))
    return {k: (float(np.median(v)), float(np.min(v)), float(np.max(v))) for k, v in times.items()}


def _fmt(t):
    return f"{t[0]:.2f} ms [{t[1]:.2f}, {t[2]:.2f}]"


def _trained_models():
    ms = []
    for w in cases.trained_weights():
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        ms.append(m.cuda().eval())
    return ms


def _look_at(eye):
    eye = np.asarray(eye, np.float64)
    f = -eye / np.linalg.norm(eye)
    r = np.cross(f, [0, 0, 1.0])
    r /= np.linalg.norm(r)
    return np.stack([r, np.cross(r, f), -f, eye], 1)


def speed(a, gpu):
    coarse, fine = _trained_models()
    grid = nb.occupancy_grid(fine, 128, *BOX, 1.0, dilate=1)
    report = {"gpu": gpu, "occupied_cells": grid.occupied_fraction(), "grids": {}}
    print(f"on {gpu}: grid of the trained scene, N = 128, {report['occupied_cells']:.4f} of the cells occupied")
    meshes = {}
    for N in (int(s) for s in a.grids.split(",")):
        _, evaluated = nb.sigma_grid(fine, N, *BOX, occupancy=grid, return_evaluated=True)
        r = {"evaluated": evaluated / N ** 3}
        r["sigma_grid"] = _alternate({"plain": lambda: nb.sigma_grid(fine, N, *BOX),
                                      "masked": lambda: nb.sigma_grid(fine, N, *BOX, occupancy=grid)}, a.rounds)
        torch.cuda.empty_cache()
        r["rgb_sigma_grid"] = _alternate({"plain": lambda: nb.rgb_sigma_grid(fine, N, *BOX),
                                          "masked": lambda: nb.rgb_sigma_grid(fine, N, *BOX, occupancy=grid)},
                                         a.rounds)
        torch.cuda.empty_cache()
        report["grids"][N] = r
        print(f"N = {N}: evaluated {r['evaluated']:.4f} of {N ** 3} points; sigma_grid plain "
              f"{_fmt(r['sigma_grid']['plain'])}, masked {_fmt(r['sigma_grid']['masked'])}; rgb_sigma_grid plain "
              f"{_fmt(r['rgb_sigma_grid']['plain'])}, masked {_fmt(r['rgb_sigma_grid']['masked'])}")
        meshes[N] = nb.extract_mesh(fine, N, *BOX, THRESHOLD)
    N_fuse = 256 if 256 in meshes else min(meshes)
    N_norm = 512 if 512 in meshes else max(meshes)
    # bench_mesh.py's views: random images, cameras on a radius-4 sphere, focal 1111, near 2
    rng = np.random.default_rng(0)
    images = torch.from_numpy(rng.integers(0, 256, (a.views, 800, 800, 3), dtype=np.uint8)).cuda()
    eyes = rng.normal(size=(a.views, 3))
    poses = [_look_at(e) for e in eyes / np.linalg.norm(eyes, axis=1, keepdims=True) * 4.0]
    v = meshes[N_fuse][0]
    fuse = _alternate({"plain": lambda: nb.fuse_vertex_colors(fine, v, images, poses, 1111.0, 2.0),
                       "masked": lambda: nb.fuse_vertex_colors(fine, v, images, poses, 1111.0, 2.0, occupancy=grid)},
                      max(1, a.rounds // 2))
    report["fuse_vertex_colors"] = {"N_grid": N_fuse, "vertices": int(v.shape[0]), "views": a.views, "ms": fuse}
    print(f"fuse_vertex_colors, {a.views} views x {v.shape[0]} vertices (N = {N_fuse} mesh): plain {_fmt(fuse['plain'])},"
          f" masked {_fmt(fuse['masked'])}")
    del images
    v, t = meshes[N_norm]
    norm = _alternate({"plain": lambda: nb.normal_vertex_colors(coarse, fine, v, t, 2.0, 6.0, white_back=True),
                       "masked": lambda: nb.normal_vertex_colors(coarse, fine, v, t, 2.0, 6.0, white_back=True,
                                                                 occupancy=grid)}, a.rounds)
    report["normal_vertex_colors"] = {"N_grid": N_norm, "vertices": int(v.shape[0]), "ms": norm}
    print(f"normal_vertex_colors, {v.shape[0]} vertices (N = {N_norm} mesh): plain {_fmt(norm['plain'])}, masked "
          f"{_fmt(norm['masked'])}")
    return report


def _components(tris):
    """Edge-connected components of a triangle list (the cluster filter's connectivity), on the host."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    t = np.asarray(tris, np.int64)
    if len(t) == 0:
        return 0
    e = np.sort(np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]]), 1)
    tid = np.tile(np.arange(len(t)), 3)
    order = np.lexsort((e[:, 1], e[:, 0]))
    e, tid = e[order], tid[order]
    same = (e[1:] == e[:-1]).all(1)
    g = coo_matrix((np.ones(int(same.sum())), (tid[1:][same], tid[:-1][same])), shape=(len(t), len(t)))
    return int(connected_components(g, directed=False)[0])


def _mesh_report(models, grid, N=256):
    from train_sharp_weights import CENTERS, RADII, ground_truth
    coarse, fine = models
    v, t = nb.extract_mesh(fine, N, *BOX, THRESHOLD, keep_largest=False, occupancy=grid)
    comps = _components(t.cpu().numpy())
    kv, kt = nb.mesh.keep_largest_cluster(v, t)
    # undo the reference's divide-by-N transform (equal cube ranges make its x / y swap moot)
    true = BOX[0][0] + (kv.double().cpu().numpy() - BOX[0][0]) * N / (N - 1)
    d = np.abs((np.linalg.norm(true[:, None, :] - CENTERS.numpy()[None], axis=-1) - RADII.numpy()).min(1))
    cols = nb.normal_vertex_colors(coarse, fine, kv, kt, 2.0, 6.0, white_back=True, occupancy=grid)
    rays = nb.normal_rays(kv, nb.vertex_normals(kv, kt), 2.0, 6.0)
    gt = torch.cat([ground_truth(r) for r in rays.split(8192)])
    err = float((cols.float() / 255 - gt).abs().mean())
    return {"components": comps, "kept_vertices": int(kv.shape[0]), "kept_triangles": int(kt.shape[0]),
            "distance_median": float(np.median(d)), "distance_p99": float(np.quantile(d, 0.99)),
            "distance_max": float(d.max()), "normal_colour_mean_abs_error": err}


def train(a, gpu):
    from train_sharp_weights import ground_truth
    rays = torch.cat([torch.from_numpy(bench.blender_rays(16384, 7000 + v)) for v in range(64)])
    rgbs = torch.cat([ground_truth(r.cuda()) for r in rays.split(16384)])
    batches = nb.DeviceRayBatches(rays, rgbs, batch_size=1024, drop_last=True, seed=99)
    report = {"gpu": gpu, "steps": a.train_steps, "runs": {}}
    for arm in ("plain", "density_grid"):
        torch.manual_seed(1234)
        models = [nb.NeRF().cuda(), nb.NeRF().cuda()]
        opt = nb.FusedAdam([p for m in models for p in m.parameters()], lr=5e-4, eps=1e-8, capturable=True)
        step = nb.CapturedTrainStep(models, batches, opt, 64, False, 1.0, 1.0, 64, True, randoms="kernel")
        dg = None
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for it in range(a.train_steps):
            if arm == "density_grid" and it == 500:
                dg = nb.DensityGrid(128, *BOX, sigma_threshold=1.0, decay=0.95, dilate=1, seed=5)
                step = nb.CapturedTrainStep(models, batches, opt, 64, False, 1.0, 1.0, 64, True, randoms="kernel",
                                            occupancy=dg, update_every=16)
            step.step()
        torch.cuda.synchronize()
        seconds = time.perf_counter() - t0
        for m in models:
            m.eval()
        grid = dg.grid if dg is not None else nb.occupancy_grid(models[1], 128, *BOX, 1.0, dilate=1)
        run = {"train_seconds_with_construction": seconds, "occupied_cells": grid.occupied_fraction(),
               "without_grid": _mesh_report(models, None), "with_grid": _mesh_report(models, grid)}
        report["runs"][arm] = run
        print(f"{arm} training, {a.train_steps} steps of 1024 rays, on {gpu} ({seconds:.1f} s incl. capture; grid "
              f"{'DensityGrid' if dg is not None else 'nb.occupancy_grid'}, {run['occupied_cells']:.4f} occupied):")
        for k in ("without_grid", "with_grid"):
            r = run[k]
            print(f"  N = 256 mesh {k.replace('_', ' ')}: {r['components']} components, {r['kept_vertices']} kept "
                  f"vertices, distance to spheres median {r['distance_median']:.4f} p99 {r['distance_p99']:.4f} max "
                  f"{r['distance_max']:.4f}, normal colours mean |d| {r['normal_colour_mean_abs_error']:.4f}")
        del step, opt, models
        torch.cuda.empty_cache()
    return report


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grids", default="256,512")
    ap.add_argument("--views", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--train", action="store_true")
    ap.add_argument("--train-steps", type=int, default=3000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh_grid.py measures on the GPU; no CUDA device is visible")
    gpu = _gpu()
    report = train(a, gpu) if a.train else speed(a, gpu)
    print(json.dumps(report))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
