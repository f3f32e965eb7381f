"""Cascaded occupancy grids on a 360° inward-facing scene (DESIGN.md §10h): does a cascade keep the background that a
grid tight around the object loses, while skipping what a grid over the whole extent cannot?

The scene is analytic (no 360° capture is available offline), in the spirit of tools/train_sharp_weights.py: three
soft spheres with a high-frequency colour pattern inside the level-0 box [-1.2, 1.2]^3, and a textured opaque shell
of radius 6 around everything.  Cameras look at the origin from radius 3 (training: random directions; held out:
the reference's spheric path, create_spheric_poses with phi = -36°, datasets/llff.py:118-156), with the spheric
rule's near = 4/3 and far = 8 near (llff.py:244-245).  Ground truth: a 1024-sample quadrature on [near, far].

Four runs train from scratch with the same seed, recipe (64 + 64 samples, perturb 1, noise 1, Adam 5e-4, batch 1024)
and steps, each captured with in-kernel randoms; runs 2-4 train --warmup steps plainly and then with a DensityGrid
maintained inside the captured loop (update every 16 steps, threshold 1, decay 0.95, dilate 1):
  1. plain;  2. one level over the object box;  3. one level at the same N over the whole extent (the last
  cascade level's box);  4. the cascade (--levels levels over the object box).
Each run reports its training wall time (replays, ending in a synchronise), the evaluated sample fraction over its
last 16 steps, held-out PSNR against the ground truth (all pixels and background pixels only: those whose
ground-truth object opacity is below 0.5), rendered plainly and with skip="samples" through its grid, and the
skip="samples" render time of one held-out view at 504 x 378 and 800 x 800 (CUDA events, median of --reps).  The
runs go in order 1-4 in one process; each is a single run.  The card's name and power limit are read in the same
run.

    python tools/bench_cascade.py [--steps 3000] [--warmup 500] [--N 128] [--levels 4] [--out FILE]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nerf_pl_b200 as nb  # noqa: E402

CENTERS = torch.tensor([[0.0, 0.0, 0.0], [0.7, 0.3, -0.2], [-0.5, -0.6, 0.4]])
RADII = torch.tensor([0.5, 0.35, 0.4])
SHELL = 6.0
BOX = ((-1.2, 1.2),) * 3
CAM_R = 3.0
NEAR = 4.0 / 3.0
FAR = 8.0 * NEAR
FOCAL_FRAC = 0.8            # focal = FOCAL_FRAC * W


def field(x):
    """(sigma, rgb, object sigma) of the scene at points x (..., 3)."""
    dist = (x[..., None, :] - CENTERS.to(x.device)).norm(dim=-1)
    obj = (40.0 / (1.0 + torch.exp((dist - RADII.to(x.device)) * 30.0))).sum(-1)
    r = x.norm(dim=-1)
    shell = 40.0 / (1.0 + torch.exp((SHELL - r) * 20.0))
    col_obj = 0.5 + 0.5 * torch.stack([torch.sin(9.0 * x[..., 0] + 2.0 * x[..., 1]),
                                       torch.sin(7.0 * x[..., 1] - 3.0 * x[..., 2]),
                                       torch.cos(8.0 * x[..., 2] + x[..., 0])], -1)
    u = x / r[..., None].clamp_min(1e-6)
    col_bg = 0.5 + 0.45 * torch.stack([torch.sin(6.0 * u[..., 0]), torch.cos(5.0 * u[..., 1] + u[..., 2]),
                                       torch.sin(7.0 * u[..., 2] - 2.0 * u[..., 0])], -1)
    sig = obj + shell
    w = (obj / sig.clamp_min(1e-12))[..., None]
    return sig, w * col_obj + (1 - w) * col_bg, obj


@torch.no_grad()
def ground_truth(rays, n=1024, chunk=8192):
    """(rgb, object opacity) per ray: quadrature of the analytic field on [near, far], black background."""
    rgb, opac = [], []
    z = torch.linspace(NEAR, FAR, n, device=rays.device)
    dz = z[1] - z[0]
    for i in range(0, rays.shape[0], chunk):
        r = rays[i:i + chunk]
        x = r[:, None, :3] + r[:, None, 3:6] * z[None, :, None]
        sig, col, obj = field(x)
        alpha = 1 - torch.exp(-sig * dz)
        T = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1 - alpha + 1e-10], -1), -1)[:, :-1]
        w = alpha * T
        rgb.append((w[..., None] * col).sum(1))
        opac.append((w * obj / sig.clamp_min(1e-12)).sum(1))
    return torch.cat(rgb), torch.cat(opac)


def look_at(eye):
    """(3, 4) camera-to-world pose at eye looking at the origin (OpenGL axes: the camera looks down -z)."""
    eye = np.asarray(eye, np.float64)
    back = eye / np.linalg.norm(eye)
    up = np.array([0.0, 0.0, 1.0]) if abs(back[2]) < 0.99 else np.array([0.0, 1.0, 0.0])
    right = np.cross(up, back)
    right /= np.linalg.norm(right)
    up = np.cross(back, right)
    return np.stack([right, up, back, eye], 1).astype(np.float32)


def spheric_pose(theta, phi=-math.pi / 5):
    """The reference's spheric path direction (llff.py:127-150) at radius CAM_R, as a look-at pose."""
    return look_at([CAM_R * math.cos(phi) * math.cos(theta), CAM_R * math.cos(phi) * math.sin(theta),
                    -CAM_R * math.sin(phi)])


def rays_of(H, W, c2w):
    return nb.generate_rays(H, W, FOCAL_FRAC * W, torch.from_numpy(c2w), NEAR, FAR)


def training_rays(views, H, W, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(views):
        d = rng.standard_normal(3)
        out.append(rays_of(H, W, look_at(CAM_R * d / np.linalg.norm(d))))
    return torch.cat(out)


def psnr(a, b):
    return float(-10.0 * torch.log10(((a - b) ** 2).mean()))


def _gpu():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def _render(models, H, W, c2w, grid):
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    kw = dict(occupancy=grid, skip="samples") if grid is not None else {}
    return nb.render_image(models, emb, H, W, FOCAL_FRAC * W, torch.from_numpy(c2w), NEAR, FAR, 64, 64, **kw)


def _render_ms(models, H, W, c2w, grid, reps):
    _render(models, H, W, c2w, grid)
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        _render(models, H, W, c2w, grid)
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def run(name, grid_fn, args, batches, evals):
    torch.manual_seed(1234)
    dev = torch.device("cuda")
    models = [nb.NeRF().to(dev), nb.NeRF().to(dev)]
    opt = nb.FusedAdam([p for m in models for p in m.parameters()], lr=5e-4, eps=1e-8, capturable=True)
    cfg = (64, False, 1.0, 1.0, 64, False)
    train_s, fracs = 0.0, []
    plain_steps = args.steps if grid_fn is None else args.warmup
    step = nb.CapturedTrainStep(models, batches, opt, *cfg, randoms={"seed": 99})
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(plain_steps):
        step.step()
    torch.cuda.synchronize()
    train_s += time.perf_counter() - t0
    dg = None
    if grid_fn is not None:
        dg = grid_fn()
        step = nb.CapturedTrainStep(models, batches, opt, *cfg, randoms={"seed": 99 + plain_steps}, occupancy=dg,
                                    update_every=16)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for k in range(args.steps - plain_steps):
            step.step()
            if k >= args.steps - plain_steps - 16:
                fracs.append(step.live_samples.clone())
        torch.cuda.synchronize()
        train_s += time.perf_counter() - t0
        fracs = [float(f.sum()) / (batches.batch_size * (64 + 128)) for f in fracs]
    out = {"run": name, "train_s": round(train_s, 2), "steps": args.steps,
           "evaluated_sample_fraction": round(float(np.mean(fracs)), 4) if fracs else 1.0}
    for tag, grid in (("plain", None), ("grid", None if dg is None else dg.grid)):
        if tag == "grid" and grid is None:
            continue
        all_p, bg_p = [], []
        for c2w, gt, bg in evals:
            img = _render(models, args.eval_h, args.eval_w, c2w, grid)["rgb"].reshape(-1, 3)
            all_p.append(psnr(img, gt))
            bg_p.append(psnr(img[bg], gt[bg]))
        out[f"psnr_{tag}"] = round(float(np.mean(all_p)), 2)
        out[f"psnr_background_{tag}"] = round(float(np.mean(bg_p)), 2)
    if dg is not None:
        out["occupied_fraction"] = round(dg.grid.occupied_fraction(), 4)
        for H, W in ((378, 504), (800, 800)):
            out[f"render_ms_{W}x{H}"] = round(_render_ms(models, H, W, spheric_pose(0.3), dg.grid, args.reps), 1)
    out["render_ms_504x378_plain"] = round(_render_ms(models, 378, 504, spheric_pose(0.3), None, args.reps), 1)
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3000)
    ap.add_argument("--warmup", type=int, default=500)
    ap.add_argument("--N", type=int, default=128)
    ap.add_argument("--levels", type=int, default=4)
    ap.add_argument("--views", type=int, default=48)
    ap.add_argument("--eval-h", type=int, default=94)
    ap.add_argument("--eval-w", type=int, default=126)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rays = training_rays(args.views, 63, 84, seed=5).cuda()
    rgbs, _ = ground_truth(rays)
    batches = nb.DeviceRayBatches(rays, rgbs, batch_size=1024, seed=6)
    evals = []
    for th in np.linspace(0, 2 * math.pi, 5)[:4]:
        c2w = spheric_pose(th)
        r = rays_of(args.eval_h, args.eval_w, c2w).cuda()
        gt, obj = ground_truth(r)
        evals.append((c2w, gt, obj < 0.5))
    whole = nb.level_ranges(*BOX, args.levels - 1)
    dgrid = lambda box, L: lambda: nb.DensityGrid(args.N, *box, sigma_threshold=1.0, decay=0.95, dilate=1,  # noqa
                                                   seed=7, levels=L)
    runs = [("plain", None), ("one level, object box", dgrid(BOX, 1)),
            ("one level, whole extent", dgrid(whole, 1)), (f"cascade, {args.levels} levels", dgrid(BOX, args.levels))]
    res = {"gpu": _gpu(), "N": args.N, "levels": args.levels, "object_box": BOX, "whole_extent": whole,
           "near": NEAR, "far": FAR, "camera_radius": CAM_R, "single_runs": True,
           "runs": [run(name, fn, args, batches, evals) for name, fn in runs]}
    print(json.dumps({k: v for k, v in res.items() if k != "runs"}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
