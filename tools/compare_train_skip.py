"""Dump both paths with empty samples skipped on seeded cases, and compare two dumps bit for bit: the tool that shows
a change to the per-sample skipping kernels computes what the tree before it computed.

Training (the eager step, render_rays_train_skip with extras on): S/K in {(64, 0), (64, 64), (32, 128)} x a full, a
partial and an empty grid x noise 0 / 1 x tensor and in-kernel random numbers.  Per case: the six results, loss4,
the weights, the per-sample values and masks, the per-row d sigma / d rgb_pre (the first live_samples rows) and the
48 gradients (24 without a fine pass).

Rendering (culling.render_samples with extras and per_sample on): S/K in {(64, 0), (64, 128), (32, 64)} x the same
grids x test_time 0 / 1 x without and with a live_flag.  Per case: every returned tensor and the sample counts.

    python tools/compare_train_skip.py --out A.npz [--tree DIR]   # DIR: the tree whose nerf_pl_b200 is imported
    python tools/compare_train_skip.py --compare A.npz B.npz
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

GRIDS = ("full", "partial", "empty")
CASES = [(S, K, grid, noise, rng) for S, K in ((64, 0), (64, 64), (32, 128)) for grid in GRIDS
         for noise in (0.0, 1.0) for rng in ("tensor", "kernel")]
RENDER_CASES = [(S, K, grid, test_time, flag) for S, K in ((64, 0), (64, 128), (32, 64)) for grid in GRIDS
                for test_time in (0, 1) for flag in (False, True)]


def dump(out, tree):
    import torch

    import nerf_pl_b200 as nb                        # before bench, which puts this tree first on sys.path
    from nerf_pl_b200 import culling
    from nerf_pl_b200.train_skip import render_rays_train_skip
    if tree and not os.path.abspath(nb.__file__).startswith(os.path.abspath(tree) + os.sep):
        raise RuntimeError(f"imported {nb.__file__}, not the package under {tree}")
    import bench
    from oracle import nerf_oracle as orc

    n = 700
    rays = torch.from_numpy(bench.blender_rays(n, 31)).cuda()
    rgbs = torch.rand(n, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(32))
    rng = np.random.default_rng(33)
    sig = np.where(rng.random((17, 17, 17)) < 0.3, 5.0, 0.0).astype(np.float32)
    grids = {"full": nb.pack_occupancy(torch.full((3, 3, 3), 5.0, device="cuda"), (-1e4, 1e4), (-1e4, 1e4),
                                       (-1e4, 1e4), 1.0, 0),
             "partial": nb.pack_occupancy(torch.from_numpy(sig).cuda(), (-1.5, 1.5), (-1.5, 1.5), (-1.5, 1.5), 1.0, 0),
             "empty": nb.pack_occupancy(torch.zeros(3, 3, 3, device="cuda"), (-1e4, 1e4), (-1e4, 1e4), (-1e4, 1e4),
                                        1.0, 0)}
    def make_models():
        models = []
        for s in (21, 22):
            m = nb.NeRF()
            m.load_state_dict({k: torch.from_numpy(v) for k, v in orc.make_weights(s).items()})
            models.append(m.cuda())
        return models

    res = {}
    for S, K, grid, noise, rnd in CASES:
        models = make_models()
        g = torch.Generator(device="cuda").manual_seed(S * 1000 + K)
        pr = torch.rand(n, S, device="cuda", generator=g)
        nc = torch.randn(n, S, device="cuda", generator=g) if noise else None
        ur = torch.rand(n, K, device="cuda", generator=g) if K else None
        nf = torch.randn(n, S + K, device="cuda", generator=g) if noise and K else None
        seed = 777 if rnd == "kernel" else None
        if seed is not None:
            pr = ur = None
        out_ = render_rays_train_skip(models, rays, S, False, 1.0, noise, K, True, pr, nc, ur, nf, rgbs, grids[grid],
                                      rng_seed=seed, extras=True)
        out_["loss"].backward()
        torch.cuda.synchronize()
        key = f"S{S}_K{K}_{grid}_noise{int(noise)}_{rnd}"
        live = out_["live_samples"]
        res[f"{key}.live"] = np.array(live, dtype=np.int64)
        for k, v in out_.items():
            if not torch.is_tensor(v):
                continue
            a = v.detach().cpu().numpy()
            if k.startswith(("dsigma", "dprergb")):          # only the first live_samples rows are defined
                a = a[:live[0 if k.endswith("coarse") else 1]]
            res[f"{key}.{k}"] = np.atleast_1d(a)
        for i, m in enumerate(models[:2 if K else 1]):
            for k, p in m.named_parameters():
                res[f"{key}.grad{i}.{k}"] = p.grad.cpu().numpy()
    models = make_models()
    g = torch.Generator(device="cuda").manual_seed(34)
    flag = (torch.rand(n, device="cuda", generator=g) < 0.5).to(torch.uint8)
    for S, K, grid, test_time, with_flag in RENDER_CASES:
        with torch.no_grad():
            out_ = culling.render_samples(models, rays, grids[grid], S, False, K, True, bool(test_time),
                                          live_flag=flag if with_flag else None, extras=True, per_sample=True)
        torch.cuda.synchronize()
        key = f"render_S{S}_K{K}_{grid}_test{test_time}_flag{int(with_flag)}"
        for k, v in out_.items():
            res[f"{key}.{k}"] = np.atleast_1d(v.cpu().numpy() if torch.is_tensor(v) else np.array(v, dtype=np.int64))
    np.savez(out, **res)
    print(f"wrote {len(res)} arrays of {len(CASES)} training and {len(RENDER_CASES)} render cases to {out} "
          f"(package {os.path.dirname(nb.__file__)})")


def compare(a, b):
    A, B = np.load(a), np.load(b)
    bad = sorted(set(A.files) ^ set(B.files))
    diff = [k for k in sorted(set(A.files) & set(B.files))
            if A[k].dtype != B[k].dtype or A[k].shape != B[k].shape
            or not np.array_equal(A[k].view(np.uint8), B[k].view(np.uint8))]
    print(f"{len(A.files)} arrays; missing on one side: {bad}; bitwise different: {diff}")
    return not bad and not diff


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--tree", default=None)
    ap.add_argument("--compare", nargs=2)
    a = ap.parse_args()
    if a.compare:
        sys.exit(0 if compare(*a.compare) else 1)
    sys.path.insert(0, ROOT)
    if a.tree:
        sys.path.insert(0, os.path.abspath(a.tree))
    dump(a.out, a.tree)


if __name__ == "__main__":
    main()
