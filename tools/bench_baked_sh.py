"""View-dependent baked volumes (nb.bake_volume(..., view_dependent=True), DESIGN.md §10k) against the direction-0 bake
of §10j and the MLP renders of the same views.

1. The trained test scene (tools/bench_baked.py's set-up: its fine net is baked and makes the grid, Blender views
   80-82, white background), per N in --N: the SH bake's time (CUDA events around one call after one warm-up; median
   [min, max] over --rounds) and bytes; the SH render eager and replayed from a CUDA graph against the direction-0
   bake's render at the same N (the arms alternate view by view; median [min, max] over views x rounds), and the
   128 + 0 MLP render with early_stop=1e-3; PSNR against the 64 + 128 MLP render and against the analytic ground truth.
2. A view-dependent analytic scene, trained from scratch with CapturedTrainStep as tools/bench_cascade.py trains (its
   scene and helpers are loaded, not copied): that tool's three soft spheres and shell, with a specular lobe
   k max(0, <-d, L>)^p around a fixed light direction L added to the spheres' colour.  Held-out views on the spheric
   path; PSNR against the ground truth of the MLP render (64 + 64), the direction-0 bake and the SH bake (N = --vd-N,
   over the spheres' box), on the pixels the spheres cover (ground-truth object opacity >= 0.5), since the shell
   lies outside the bake box.

The card's name and power limit are read in the same run.

    python tools/bench_baked_sh.py [--N 256,512,1024] [--side 800] [--rounds 5] [--steps 3000] [--out FILE]
"""
import argparse
import importlib.util
import json
import math
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nerf_pl_b200 as nb  # noqa: E402
from tests import cases  # noqa: E402


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tools", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


bb = _load("bench_baked")
bc = _load("bench_cascade")
LIGHT = torch.tensor([0.48, -0.36, 0.8])
LOBE_K, LOBE_P = 0.45, 4.0


def vd_field(x, d):
    """(sigma, rgb, object sigma) of the view-dependent scene at points x (..., 3) seen along unit directions d."""
    sig, col, obj = bc.field(x)
    lobe = LOBE_K * (-(d * LIGHT.to(x.device)).sum(-1)).clamp_min(0) ** LOBE_P
    w = obj / sig.clamp_min(1e-12)
    return sig, (col + (w * lobe)[..., None]).clamp(0, 1), obj


@torch.no_grad()
def vd_truth(rays, n=1024, chunk=8192):
    """(rgb, object opacity) per ray: quadrature of the field on [near, far], black background."""
    rgb, opac = [], []
    z = torch.linspace(bc.NEAR, bc.FAR, n, device=rays.device)
    dz = z[1] - z[0]
    for i in range(0, rays.shape[0], chunk):
        r = rays[i:i + chunk]
        d = r[:, 3:6] / r[:, 3:6].norm(dim=-1, keepdim=True)
        x = r[:, None, :3] + r[:, None, 3:6] * z[None, :, None]
        sig, col, obj = vd_field(x, d[:, None, :].expand_as(x))
        alpha = 1 - torch.exp(-sig * dz)
        T = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1 - alpha + 1e-10], -1), -1)[:, :-1]
        rgb.append(((alpha * T)[..., None] * col).sum(1))
        opac.append((alpha * T * obj / sig.clamp_min(1e-12)).sum(1))
    return torch.cat(rgb), torch.cat(opac)


def trained_scene(a, report):
    models = []
    for w in cases.trained_weights():
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        models.append(m.cuda().eval())
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    fine = models[1]
    grid = nb.occupancy_grid(fine, 128, *bb.BOX, 1.0, dilate=1)
    side = a.side
    views = [bb._pose(80 + v, side) for v in range(3)]
    rays = [nb.generate_rays(side, side, f, c2w, 2.0, 6.0) for c2w, f in views]
    gt = bb._ground_truth()
    truth = [gt(r) for r in rays]
    ref = [nb.render_image(models, emb, side, side, views[v][1], views[v][0], 2.0, 6.0, 64, 128, white_back=True,
                           occupancy=grid, skip="samples")["rgb"].reshape(-1, 3) for v in range(3)]
    mlp = lambda v: nb.render_image(models, emb, side, side, views[v][1], views[v][0], 2.0, 6.0, 128, 0,  # noqa: E731
                                    white_back=True, occupancy=grid, skip="samples", early_stop=1e-3)
    mlp(0)
    tm = [bb._ms(lambda: mlp(v)) for _ in range(a.rounds) for v in range(3)]
    report["mlp_128_0_eps1e-3_ms"] = bb._stats(tm)
    print(f"MLP 128+0 eps 1e-3: {bb._fmt(report['mlp_128_0_eps1e-3_ms'])}")
    report["trained"] = {}
    for N in (int(s) for s in a.N.split(",") if s):
        torch.cuda.empty_cache()
        try:
            bake = lambda: nb.bake_volume(fine, N, *bb.BOX, occupancy=grid, view_dependent=True)  # noqa: E731
            vol = bake()
            tb = []
            for _ in range(a.rounds):
                del vol
                held = []
                tb.append(bb._ms(lambda: held.append(bake())))
                vol = held[0]
            plain = nb.bake_volume(fine, N, *bb.BOX, occupancy=grid)
        except torch.cuda.OutOfMemoryError:
            print(f"N {N}: the bake does not fit")
            report["trained"][N] = {"fits": False}
            continue
        r = {"bake_ms": bb._stats(tb), "bricks": vol.bricks, "bytes": vol.nbytes, "plain_bytes": plain.nbytes}
        static = rays[0].clone()
        nb.render_baked(vol, static, white_back=True)
        nb.render_baked(plain, static, white_back=True)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            nb.render_baked(vol, static, white_back=True)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            gout = nb.render_baked(vol, static, white_back=True)
        te, tg, tp = [], [], []
        for _ in range(a.rounds):
            for v in range(3):
                te.append(bb._ms(lambda: nb.render_baked(vol, rays[v], white_back=True)))
                tp.append(bb._ms(lambda: nb.render_baked(plain, rays[v], white_back=True)))
                static.copy_(rays[v])
                tg.append(bb._ms(g.replay))
        assert torch.equal(gout["rgb"], nb.render_baked(vol, rays[2], white_back=True)["rgb"])
        r["render_ms"], r["graph_ms"], r["plain_render_ms"] = bb._stats(te), bb._stats(tg), bb._stats(tp)
        out = [nb.render_baked(vol, rays[v], white_back=True)["rgb"] for v in range(3)]
        po = [nb.render_baked(plain, rays[v], white_back=True)["rgb"] for v in range(3)]
        r["psnr_vs_mlp"] = [bb._psnr(out[v], ref[v]) for v in range(3)]
        r["psnr_vs_truth"] = [bb._psnr(out[v], truth[v]) for v in range(3)]
        r["plain_psnr_vs_mlp"] = [bb._psnr(po[v], ref[v]) for v in range(3)]
        r["plain_psnr_vs_truth"] = [bb._psnr(po[v], truth[v]) for v in range(3)]
        report["trained"][N] = r
        print(f"N {N}: SH bake {bb._fmt(r['bake_ms'])}, {r['bricks']} bricks, {r['bytes'] / 2 ** 30:.2f} GiB "
              f"(direction 0: {r['plain_bytes'] / 2 ** 30:.2f} GiB); render eager {bb._fmt(r['render_ms'])}, graph "
              f"{bb._fmt(r['graph_ms'])}, direction-0 render {bb._fmt(r['plain_render_ms'])}; PSNR vs MLP "
              f"{[round(p, 2) for p in r['psnr_vs_mlp']]} (direction 0 {[round(p, 2) for p in r['plain_psnr_vs_mlp']]}),"
              f" vs truth {[round(p, 2) for p in r['psnr_vs_truth']]} (direction 0 "
              f"{[round(p, 2) for p in r['plain_psnr_vs_truth']]})", flush=True)
        del vol, plain, g, gout


def vd_scene(a, report):
    torch.manual_seed(1234)
    rays = bc.training_rays(48, 63, 84, seed=5).cuda()
    batches = nb.DeviceRayBatches(rays, vd_truth(rays)[0], batch_size=1024, seed=6)
    models = [nb.NeRF().cuda(), nb.NeRF().cuda()]
    opt = nb.FusedAdam([p for m in models for p in m.parameters()], lr=5e-4, eps=1e-8, capturable=True)
    step = nb.CapturedTrainStep(models, batches, opt, 64, False, 1.0, 1.0, 64, False, randoms={"seed": 99})
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.steps):
        step.step()
    torch.cuda.synchronize()
    res = {"steps": a.steps, "train_s": round(time.perf_counter() - t0, 2), "N": a.vd_N}
    for m in models:
        m.eval()
    grid = nb.occupancy_grid(models[1], 128, *bc.BOX, 1.0, dilate=1)
    vols = {"direction 0": nb.bake_volume(models[1], a.vd_N, *bc.BOX, occupancy=grid),
            "SH": nb.bake_volume(models[1], a.vd_N, *bc.BOX, occupancy=grid, view_dependent=True)}
    psnr = {"MLP 64+64": [], "direction 0": [], "SH": []}
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    H, W = 200, 200
    for th in np.linspace(0, 2 * math.pi, 9)[:8]:
        c2w = bc.spheric_pose(th)
        r = bc.rays_of(H, W, c2w).cuda()
        gt, obj = vd_truth(r)
        on = obj >= 0.5
        mlp = nb.render_image(models, emb, H, W, bc.FOCAL_FRAC * W, torch.from_numpy(c2w), bc.NEAR, bc.FAR, 64, 64)
        psnr["MLP 64+64"].append(bc.psnr(mlp["rgb"].reshape(-1, 3)[on], gt[on]))
        for k, v in vols.items():
            psnr[k].append(bc.psnr(nb.render_baked(v, r)["rgb"][on], gt[on]))
    res["psnr_vs_truth_mean"] = {k: round(float(np.mean(v)), 2) for k, v in psnr.items()}
    res["psnr_vs_truth"] = {k: [round(p, 2) for p in v] for k, v in psnr.items()}
    report["view_dependent_scene"] = res
    print(f"view-dependent scene ({a.steps} steps, {res['train_s']} s): held-out PSNR vs truth "
          f"{res['psnr_vs_truth_mean']}", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", default="256,512,1024")         # "" runs the view-dependent scene only
    ap.add_argument("--side", type=int, default=800)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3000)
    ap.add_argument("--vd-N", type=int, default=256)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_baked_sh.py needs a CUDA device")
    report = {"gpu": bb._gpu(), "side": a.side, "rounds": a.rounds}
    print(f"on {report['gpu']}")
    if a.N:
        trained_scene(a, report)
    vd_scene(a, report)
    line = json.dumps(report)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
