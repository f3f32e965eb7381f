"""Time forward + backward of one training call of NeRF.forward (models/nerf.py:83-124) over B samples (default
196,608: one training step's samples at 64 + 64 for 1024 rays), on both autograd paths of nerf_pl_b200.NeRF:

  fused   model.autograd_impl = "fused": one save-mode MLP launch + the sm_90a backward kernels
  torch   model.autograd_impl = "torch": torch ops in fp32 with TF32 off, as the reference computes

Both paths run in the same process, alternating, `--rounds` times; each round reports the median of `--steps`
CUDA-event-timed steps after `--warmup` untimed ones.  The card's name and power limit are read in the same run.
Prints one JSON line per round and a summary line.

    python tools/bench_nerf_train.py [--B 196608] [--steps 30] [--warmup 5] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nerf_pl_b200 as nb  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def inputs(B, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    xyz = torch.rand(B, 3, device=dev, generator=g) * 3 - 1.5
    d = torch.nn.functional.normalize(torch.randn(B, 3, device=dev, generator=g), dim=-1)
    x = torch.cat((nb.Embedding(3, 10)(xyz), nb.Embedding(3, 4)(d)), -1)
    return x, torch.randn(B, 4, device=dev, generator=g) * 0.1


def time_impl(m, impl, x, gout, steps, warmup):
    m.autograd_impl = impl
    times = []
    for i in range(warmup + steps):
        m.zero_grad(set_to_none=True)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        m(x).backward(gout)
        e1.record()
        e1.synchronize()
        if i >= warmup:
            times.append(e0.elapsed_time(e1))
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=196608)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_nerf_train.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    m = nb.NeRF().to(dev)
    x, gout = inputs(a.B, dev)
    name, limit = card()
    res = {"fused": [], "torch": []}
    for r in range(a.rounds):
        for impl in ("fused", "torch") if r % 2 == 0 else ("torch", "fused"):
            res[impl].append(time_impl(m, impl, x, gout, a.steps, a.warmup))
        print(json.dumps({"round": r, "fused_ms": round(res["fused"][-1], 3), "torch_fp32_ms": round(res["torch"][-1], 3)}))
    f, t = statistics.median(res["fused"]), statistics.median(res["torch"])
    print(json.dumps({"B": a.B, "card": name, "power_limit": limit, "steps": a.steps, "rounds": a.rounds,
                      "fused_ms_median": round(f, 3), "fused_ms_range": [round(min(res["fused"]), 3), round(max(res["fused"]), 3)],
                      "torch_fp32_ms_median": round(t, 3),
                      "torch_fp32_ms_range": [round(min(res["torch"]), 3), round(max(res["torch"]), 3)],
                      "speedup": round(t / f, 2)}))


if __name__ == "__main__":
    main()
