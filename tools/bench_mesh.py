"""Device time per stage of the coloured-mesh workflow (nerf_pl_b200.mesh) on the trained test weights.

Stages at N_grid 256 and 512 over [-1.5, 1.5]^3, threshold 20: sigma grid, marching cubes (count + emit),
index -> world, largest cluster; the Unity volume's rgb+sigma grid and its pack (count + emit); the vertex-normal
colours of the kept mesh (normals, rays, the render of one ray per vertex at 64 + 64 samples, and the whole
``normal_vertex_colors`` call); colour fusion over 100 views at 800 x 800.  CUDA events around each stage;
prints the card name and power limit with the numbers, and one JSON line.  The bytes columns are the
minimum traffic of the MC and cluster passes (every array read / written once), as a share of the card's
HBM bandwidth (3.35 TB/s on an H100 SXM).
Run: python tools/bench_mesh.py [--grids 256 512] [--views 100]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nerf_pl_b200 as nb  # noqa: E402
from nerf_pl_b200 import mesh  # noqa: E402
from tests import cases  # noqa: E402

RANGE = (-1.5, 1.5)
HBM = 3.35e12


def timed(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    best = None
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b)
        best = ms if best is None else min(best, ms)
    return best, out


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = torch.cuda.get_device_name()
    return q


def look_at(eye):
    eye = np.asarray(eye, np.float64)
    f = -eye / np.linalg.norm(eye)
    r = np.cross(f, [0, 0, 1.0])
    r /= np.linalg.norm(r)
    return np.stack([r, np.cross(r, f), -f, eye], 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grids", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--views", type=int, default=100)
    args = ap.parse_args()
    model = nb.NeRF()
    model.load_state_dict({k: torch.from_numpy(v) for k, v in cases.trained_weights()[1].items()})
    model = model.cuda().eval()
    coarse = nb.NeRF()
    coarse.load_state_dict({k: torch.from_numpy(v) for k, v in cases.trained_weights()[0].items()})
    coarse = coarse.cuda().eval()
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    res = {"card": card()}
    print("card, power limit:", res["card"])
    for N in args.grids:
        ms_sig, sigma = timed(lambda: nb.sigma_grid(model, N, RANGE, RANGE, RANGE))
        ms_mc, (vi, tri) = timed(lambda: nb.marching_cubes(sigma, 20.0))
        ms_w, vw = timed(lambda: mesh.to_world(vi, N, RANGE, RANGE, RANGE))
        ms_cl, (kv, kt) = timed(lambda: mesh.keep_largest_cluster(vw, tri))
        P, V, T = N ** 3, vi.shape[0], tri.shape[0]
        # classify reads sigma and writes 2 count bytes per point; scans read 1 B, write 4 B; emit re-reads sigma
        mc_bytes = P * 4 + 2 * P + 2 * 5 * P + P * 4 + P + V * 24 + T * 12
        cl_bytes = T * 12 + 3 * T * 12 * 2 + T * 8 * 3 + V * 13 + T * 12 + kv.shape[0] * 12 + kt.shape[0] * 12
        r = {"sigma_grid_ms": ms_sig, "marching_cubes_ms": ms_mc, "to_world_ms": ms_w, "cluster_ms": ms_cl,
             "vertices": V, "triangles": T, "kept_triangles": int(kt.shape[0]),
             "mc_hbm_share": mc_bytes / (ms_mc * 1e-3) / HBM, "cluster_hbm_share": cl_bytes / (ms_cl * 1e-3) / HBM}
        del sigma, vi, tri, vw
        # Unity volume (extract_mesh.ipynb): rgb+sigma grid, then alpha / pack / compaction (count + emit); the pack
        # reads the 16-byte rows twice
        ms_rgb, rgbsigma = timed(lambda: mesh.rgb_sigma_grid(model, N, RANGE, RANGE, RANGE))
        ms_vol, vol = timed(lambda: mesh.pack_volume(rgbsigma, RANGE))
        r.update({"rgb_sigma_grid_ms": ms_rgb, "volume_pack_ms": ms_vol, "volume_voxels": int(vol.shape[0]),
                  "volume_hbm_share": (2 * P * 16 + vol.shape[0] * 8) / (ms_vol * 1e-3) / HBM})
        del rgbsigma, vol
        # vertex-normal colours (--use_vertex_normal) on the kept mesh: normals, rays, one render of V rays at 64 + 64
        ms_nrm, nrm = timed(lambda: nb.vertex_normals(kv, kt))
        ms_rays, rays = timed(lambda: nb.normal_rays(kv, nrm, 2.0, 6.0))
        with torch.no_grad():
            ms_rend, _ = timed(lambda: nb.render_rays([coarse, model], emb, rays, 64, False, 0, 0, 64, 32768, True,
                                                      test_time=True, match_reference_rng=False))
        ms_vn, _ = timed(lambda: nb.normal_vertex_colors(coarse, model, kv, kt, 2.0, 6.0, white_back=True))
        r.update({"normals_ms": ms_nrm, "normal_rays_ms": ms_rays, "normal_render_ms": ms_rend,
                  "normal_colors_total_ms": ms_vn, "normal_rays": int(kv.shape[0]),
                  "normal_render_Msamples_per_s": kv.shape[0] * 128 / (ms_rend * 1e-3) / 1e6})
        del nrm, rays
        res[f"N{N}"] = r
        print(f"N_grid {N}: " + ", ".join(f"{k} {v:.4g}" if isinstance(v, float) else f"{k} {v}" for k, v in r.items()))
        if N == args.grids[0]:
            verts = kv
    H = W = 800
    rng = np.random.default_rng(0)
    images = torch.from_numpy(rng.integers(0, 256, (args.views, H, W, 3), dtype=np.uint8)).cuda()
    eyes = rng.normal(size=(args.views, 3))
    eyes = eyes / np.linalg.norm(eyes, axis=1, keepdims=True) * 4.0
    poses = [look_at(e) for e in eyes]
    ms_col, _ = timed(lambda: nb.fuse_vertex_colors(model, verts, images, poses, 1111.0, 2.0), reps=1)
    res["color_fusion"] = {"views": args.views, "vertices": int(verts.shape[0]), "ms": ms_col}
    print(f"colour fusion: {args.views} views x {verts.shape[0]} vertices: {ms_col:.1f} ms")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
