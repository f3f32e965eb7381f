"""Training from the views against training from stored rays, on a synthetic 100-view 800 x 800 RGBA set
(64 M pixels, the size of a Blender scene):

  (r) DeviceRayBatches: every ray [o, d, near, far] and colour stored on the device, 44 B per pixel;
  (v) DeviceViewBatches: the uint8 images and one pose per view stored, 4 B per pixel; each batch's rays and colours
      are made by one view_batch_kernel launch.

For each: the device bytes of the dataset, the peak of ``torch.cuda.max_memory_allocated`` over building the dataset
and the CapturedTrainStep and its warm-up (above what was allocated before), the ms per CapturedTrainStep replay
(1024 rays, 64 + 64 samples, perturb 1, noise 0, white background, in-kernel random numbers) timed in alternating
rounds, and the gather alone (CUDA events around --gathers gathers of 1024 ids).  Both steps start from the same
weights and seeds, so after the same number of replays their parameters must be equal; that is checked and printed.
Prints the GPU, its power limit and the numbers as JSON lines.

    python tools/bench_view_batches.py [--steps 200] [--warmup 20] [--rounds 5] [--views 100] [--side 800]
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
import nerf_pl_b200 as nb  # noqa: E402


def synthetic_views(views, side, dev, seed=0):
    """RGBA images (random colours, a transparent border) and cameras on a radius-4 sphere looking at the origin."""
    g = torch.Generator(device=dev).manual_seed(seed)
    images = torch.randint(0, 256, (views, side, side, 4), dtype=torch.uint8, device=dev, generator=g)
    images[:, : side // 8, :, 3] = 0
    rng = np.random.default_rng(seed)
    c2w = np.zeros((views, 3, 4))
    for v in range(views):
        z = rng.normal(size=3)
        z[2] = abs(z[2]) + 0.3
        z /= np.linalg.norm(z)
        x = np.cross([0.0, 0.0, 1.0], z)
        x /= np.linalg.norm(x)
        c2w[v] = np.stack([x, np.cross(z, x), z, 4.0 * z], 1)
    return images, c2w, 1.2 * side


def stored_rays(views, c2w, focal, dev):
    """The rays and colours DeviceRayBatches would be given: nb.generate_rays per view, and the colours of
    ``views.view(v)`` (T.ToTensor()'s u8 / 255 blended onto white)."""
    V, H, W, _ = views.shape
    rays = torch.empty(V * H * W, 8, device=dev)
    rgbs = torch.empty(V * H * W, 3, device=dev)
    for v in range(V):
        sl = slice(v * H * W, (v + 1) * H * W)
        rays[sl] = nb.generate_rays(H, W, focal, c2w[v], 2.0, 6.0, device=dev)
        rgbs[sl] = views.view(v)["rgbs"]
    return rays, rgbs


def models(dev):
    torch.manual_seed(1)
    return [nb.NeRF().to(dev), nb.NeRF().to(dev)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--gathers", type=int, default=2000)
    ap.add_argument("--views", type=int, default=100)
    ap.add_argument("--side", type=int, default=800)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_view_batches needs a CUDA device")
    dev = torch.device("cuda:0")
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        smi = "unknown"
    print(json.dumps({"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": smi, "torch": torch.__version__}))
    B, S, K = 1024, 64, 64
    n_pix = args.views * args.side * args.side
    steps, batches, mem = {}, {}, {}
    for kind in ("views", "rays"):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        if kind == "views":
            images, c2w, focal = synthetic_views(args.views, args.side, dev)
            b = nb.DeviceViewBatches(images, c2w, focal, 2.0, 6.0, batch_size=B, seed=2)
            data_bytes = b.images.numel() + b.c2w.numel() * 4
        else:
            rays, rgbs = stored_rays(batches["views"], c2w, focal, dev)
            b = nb.DeviceRayBatches(rays, rgbs, batch_size=B, seed=2)
            del rays, rgbs
            data_bytes = (b.rays.numel() + b.rgbs.numel()) * 4
        ms = models(dev)
        opt = nb.FusedAdam([p for m in ms for p in m.parameters()], lr=5e-4, eps=1e-8, capturable=True)
        st = nb.CapturedTrainStep(ms, b, opt, S, False, 1.0, 0.0, K, True, randoms={"seed": 77})
        for _ in range(args.warmup):
            st.step()
        torch.cuda.synchronize()
        mem[kind] = {"dataset_bytes": data_bytes, "dataset_bytes_per_pixel": data_bytes / n_pix,
                     "peak_bytes_above_before": torch.cuda.max_memory_allocated(dev) - base}
        steps[kind], batches[kind] = st, b
    # the views object reads `images` itself (a device uint8 tensor is not copied); nothing else holds it
    del images
    times = {k: [] for k in steps}
    for _ in range(args.rounds):
        for kind, st in steps.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                st.step()
            torch.cuda.synchronize()
            times[kind].append((time.perf_counter() - t0) * 1e3 / args.steps)
    same = all(torch.equal(p, q) for p, q in zip(steps["views"].params, steps["rays"].params))
    gather = {}
    for kind, b in batches.items():
        perm = b.next_permutation()
        for k in range(20):
            b.gather(perm[k * B:(k + 1) * B])
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for k in range(args.gathers):
            off = (k % (perm.shape[0] // B)) * B
            b.gather(perm[off:off + B])
        e1.record()
        torch.cuda.synchronize()
        gather[kind] = e0.elapsed_time(e1) * 1e3 / args.gathers
    print(json.dumps({"views": args.views, "side": args.side, "pixels": n_pix, "rays_per_step": B, "samples": [S, K],
                      "steps_per_round": args.steps, "rounds": args.rounds, "memory": mem,
                      "ms_per_step_median": {k: sorted(v)[len(v) // 2] for k, v in times.items()},
                      "ms_per_step_rounds": times, "gather_us": gather,
                      "launches_per_step": {k: s.launches_per_step for k, s in steps.items()},
                      "identical_parameters_after_training": same}))


if __name__ == "__main__":
    main()
