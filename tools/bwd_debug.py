"""Stage-by-stage check of the training step (run on an H100): the forward tape in the workspace (activations,
sign bits, direction layer, heads), the compositing backward, dd, every step of the dgrad chain and the chain as a
whole in float64 on the device's own masks ("same masks"), and the 48 final gradients against float64 contractions
of the device's own operands.  Every comparison takes the device's stored inputs of that stage, so a wrong kernel
stands out in one call.  The reader and the references are tests/train_tape.py, shared with
tests/test_gpu_train_stages.py.

    python tools/bwd_debug.py [n_rays]
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nerf_pl_b200 as nb  # noqa: E402
from nerf_pl_b200 import _lib  # noqa: E402
from oracle import nerf_oracle as orc  # noqa: E402
from oracle import nerf_oracle_grad as og  # noqa: E402
from tests import train_tape as tt  # noqa: E402


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 64
    dev = torch.device("cuda:0")
    ws = [orc.make_weights(11), orc.make_weights(12)]
    models = []
    for w in ws:
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        models.append(m.to(dev))
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    rays = orc.make_rays(n, 31)
    rs = np.random.RandomState(3)
    target = rs.uniform(0, 1, (n, 3)).astype(np.float32)
    randoms = {"perturb_rand": rs.rand(n, 64).astype(np.float32), "u_rand": rs.rand(n, 64).astype(np.float32)}
    rnd = {k: torch.from_numpy(v).to(dev) for k, v in randoms.items()}
    out = nb.render_rays_loss(models, emb, torch.from_numpy(rays).to(dev), torch.from_numpy(target).to(dev), 64, False,
                              1.0, 0.0, 64, 32768, True, randoms=rnd)
    torch.cuda.synchronize()
    print("forward ok, loss", float(out["loss"].detach()), "psnr", float(out["psnr"]))
    ws_obj = out["rgb_coarse"].grad_fn.keep[-1]
    out["loss"].backward()
    torch.cuda.synchronize()
    print("backward ok; status", _lib.load().nerfb200_check_status())
    raw = ws_obj.buf.cpu().numpy()
    loss, res, ref_grads = og.render_rays_loss_grad(ws, rays, target, 64, False, 1.0, 0.0, 64, True, randoms)
    print("oracle loss", loss)
    dir_emb = orc.embed(rays[:, 3:6], 4)
    grads = {}
    for ps, (tag, P) in enumerate(zip(("coarse", "fine"), tt.layout(n, 64, 64))):
        net = tt.Net(ws[ps])
        tape = tt.WorkspaceTape(raw, P)
        fwd = tt.check_forward(tape, net, dir_emb)
        print(f"[{tag}] forward on the device's inputs:", " ".join(f"{k} {v:.3g}" for k, v in fwd.items()))
        masks = tt.check_masks(tape)
        print(f"[{tag}] sign bits vs h == 0: contradictions {masks['illegal']}, "
              f"agreement {1 - masks['legal_frac']:.6f} (the rest: positive pre-activations that round to 0)")
        g_rgb = (2.0 * (out[f"rgb_{tag}"].detach().cpu().numpy().astype(np.float64) - target) / (3 * n)).astype(np.float32)
        comp = tt.check_composite(tape, rays, g_rgb, None, None, None, 0.0, True)
        print(f"[{tag}] compositing backward:", " ".join(f"{k} {v:.3g}" for k, v in comp.items()))
        chain = tt.check_chain(tape, net)
        print(f"[{tag}] scales log2 {[int(np.log2(s)) for s in chain['scales']]}, saturated {chain['saturated']}")
        for v in range(9):
            name = "dd" if v == 0 else f"dpre{9 - v}"
            line = f"[{tag}] {name:6s} one step {chain[f'step{v}']:.3g} ulp"
            if v:
                line += f"  same masks rel_l2 {chain[f'acc{v}']:.3e} max {chain[f'accmax{v}']:.3e}"
            print(line)
        gref = tt.reference_grads(tape, net, chain["scales"], dir_emb)
        dev_g = {k: p.grad.detach().cpu().numpy() for k, p in models[ps].named_parameters()}
        for k, (r, mx) in tt.check_grads(dev_g, gref).items():
            print(f"[{tag}] grad {k:32s} vs own operands rel {r:.3e} max {mx:.3e}")
        grads.update({f"{tag}.{k}": v for k, v in dev_g.items()})
    rows, (rel, cos) = og.grad_compare(grads, ref_grads)
    for k, (r, c) in rows.items():
        print(f"grad {k:36s} vs oracle rel {r:.3e} cos {c:.6f}")
    print(f"GLOBAL vs oracle rel {rel:.3e} cos {cos:.6f}")


if __name__ == "__main__":
    main()
