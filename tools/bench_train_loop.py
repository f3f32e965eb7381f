"""ms per 1024-ray training step (64 + 64 samples, perturb 1) for three ways of feeding it, on a synthetic 100-view
400x400 set (16 M rays):

  (a) the reference's loop: DataLoader(shuffle=True, num_workers=4, batch_size=1024, pin_memory=True) over host
      rays / rgbs, the batch copied to the device, then the eager step (render_rays_loss, backward, FusedAdam);
  (b) DeviceRayBatches + the same eager step;
  (c) CapturedTrainStep (one CUDA graph replay per step, capturable FusedAdam).

Each loop is warmed up, then timed in alternating rounds (a, b, c, a, b, c, ...) of --steps steps, each round between
device synchronisations; the median round is reported.  noise_std 0 (Blender recipe, white background) and 1 (LLFF
recipe, opt.py's default).  Prints the GPU, its power limit and the host CPU count with the numbers.

    python tools/bench_train_loop.py [--steps 200] [--warmup 20] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nerf_pl_b200 as nb  # noqa: E402


class RayDataset(torch.utils.data.Dataset):
    """The training split as datasets/blender.py serves it: one ray and its colour per item."""

    def __init__(self, rays, rgbs):
        self.rays, self.rgbs = rays, rgbs

    def __len__(self):
        return self.rays.shape[0]

    def __getitem__(self, i):
        return {"rays": self.rays[i], "rgbs": self.rgbs[i]}


def synthetic_set(views=100, H=400, W=400, seed=0):
    """Rays of `views` cameras on a sphere of radius 4 looking at the origin (focal 1.2 W), near 2, far 6."""
    g = torch.Generator().manual_seed(seed)
    n = views * H * W
    rays = torch.empty(n, 8)
    j, i = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    focal = 1.2 * W
    d_cam = torch.stack([(i - W / 2) / focal, -(j - H / 2) / focal, -torch.ones_like(i)], -1).reshape(-1, 3)
    for v in range(views):
        z = torch.nn.functional.normalize(torch.randn(3, generator=g), dim=0)
        x = torch.nn.functional.normalize(torch.linalg.cross(torch.tensor([0.0, 0.0, 1.0]), z), dim=0)
        y = torch.linalg.cross(z, x)
        R = torch.stack([x, y, z], 1)
        sl = slice(v * H * W, (v + 1) * H * W)
        rays[sl, 3:6] = torch.nn.functional.normalize(d_cam @ R.T, dim=-1)
        rays[sl, 0:3] = 4.0 * z
    rays[:, 6], rays[:, 7] = 2.0, 6.0
    rgbs = torch.rand(n, 3, generator=g)
    return rays, rgbs


def make_models(dev, seed):
    torch.manual_seed(seed)
    return [nb.NeRF().to(dev), nb.NeRF().to(dev)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--views", type=int, default=100)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_loop needs a CUDA device")
    dev = torch.device("cuda:0")
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        smi = "unknown"
    print(json.dumps({"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": smi, "host_cpus": os.cpu_count(),
                      "torch": torch.__version__}))
    rays, rgbs = synthetic_set(args.views)
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    B, S, K = 1024, 64, 64
    for noise in (0.0, 1.0):
        white = noise == 0.0

        def eager_step(models, opt, r, c):
            opt.zero_grad(set_to_none=True)
            out = nb.render_rays_loss(models, emb, r, c, S, False, 1.0, noise, K, 32768, white)
            out["loss"].backward()
            opt.step()

        # (a) the reference's DataLoader
        ma = make_models(dev, 1)
        oa = nb.FusedAdam([p for m in ma for p in m.parameters()], lr=5e-4, eps=1e-8)
        loader = torch.utils.data.DataLoader(RayDataset(rays, rgbs), shuffle=True, num_workers=4, batch_size=B,
                                             pin_memory=True, persistent_workers=True)
        it_a = [iter(loader)]

        def run_a(k):
            for _ in range(k):
                b = next(it_a[0], None)
                if b is None:
                    it_a[0] = iter(loader)
                    b = next(it_a[0])
                eager_step(ma, oa, b["rays"].to(dev, non_blocking=True), b["rgbs"].to(dev, non_blocking=True))

        # (b) DeviceRayBatches, eager step
        mb = make_models(dev, 1)
        ob = nb.FusedAdam([p for m in mb for p in m.parameters()], lr=5e-4, eps=1e-8)
        batches = nb.DeviceRayBatches(rays, rgbs, batch_size=B, seed=2, device=dev)
        it_b = [iter(batches)]

        def run_b(k):
            for _ in range(k):
                b = next(it_b[0], None)
                if b is None:
                    it_b[0] = iter(batches)
                    b = next(it_b[0])
                eager_step(mb, ob, b["rays"], b["rgbs"])

        # (c) CapturedTrainStep
        mc = make_models(dev, 1)
        oc = nb.FusedAdam([p for m in mc for p in m.parameters()], lr=5e-4, eps=1e-8, capturable=True)
        cap = nb.CapturedTrainStep(mc, batches, oc, S, False, 1.0, noise, K, white)

        def run_c(k):
            for _ in range(k):
                cap.step()

        loops = {"a_dataloader_eager": run_a, "b_device_batches_eager": run_b, "c_captured_graph": run_c}
        for f in loops.values():
            f(args.warmup)
        torch.cuda.synchronize()
        times = {k: [] for k in loops}
        for _ in range(args.rounds):
            for name, f in loops.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                f(args.steps)
                torch.cuda.synchronize()
                times[name].append((time.perf_counter() - t0) * 1e3 / args.steps)
        loss = float(cap.step()[0])
        print(json.dumps({"noise_std": noise, "white_back": white, "rays_per_step": B, "samples": [S, K],
                          "n_rays": rays.shape[0], "steps_per_round": args.steps, "rounds": args.rounds,
                          "ms_per_step_median": {k: sorted(v)[len(v) // 2] for k, v in times.items()},
                          "ms_per_step_rounds": times, "captured_launches_per_step": cap.launches_per_step,
                          "captured_final_loss": loss}))
        del it_a, loader, cap, batches


if __name__ == "__main__":
    main()
