"""tests/adam_ref.py against torch.optim.Adam in float64 on the CPU (no GPU needed).

Given the same fp32-rounded hyper-parameters, torch's float64 Adam and the reference differ only in float64
rounding (torch updates m with lerp_ and divides before adding eps in another order), so over 60 steps they agree
to ~1e-15 relative.  This pins the reference the GPU tests hold FusedAdam to.
"""
import numpy as np
import pytest
import torch

from tests import adam_ref


@pytest.mark.parametrize("wd", [0.0, 1e-3])
def test_reference_matches_float64_torch_adam(wd):
    lr0, b1, b2, eps = (adam_ref.f32(x) for x in (5e-4, 0.9, 0.999, 1e-8))
    wd = adam_ref.f32(wd)
    gen = torch.Generator().manual_seed(5)
    shapes = [(256, 63), (256,), (1, 256), (3,), (0,), (1025,)]
    params = [torch.randn(s, generator=gen, dtype=torch.float64) * 0.05 for s in shapes]
    params[3].zero_()                                 # a tensor at exactly 0: p' = -update
    tp = [p.clone().requires_grad_(True) for p in params]
    opt = torch.optim.Adam(tp, lr=lr0, betas=(b1, b2), eps=eps, weight_decay=wd)
    ref = [(p.clone(), torch.zeros_like(p), torch.zeros_like(p)) for p in params]
    worst = {"p": 0.0, "m": 0.0, "v": 0.0}
    for t in range(1, 61):
        lr = adam_ref.f32(lr0 * (0.5 if t > 30 else 1.0) * min(1.0, t / 5))   # warm-up, then a step decay
        for group in opt.param_groups:
            group["lr"] = lr
        grads = [torch.randn(p.shape, generator=gen, dtype=torch.float64) * 10.0 ** (-1 - i) for i, p in enumerate(params)]
        for p, g in zip(tp, grads):
            p.grad = g.clone()
        opt.step()
        for i, (p, g) in enumerate(zip(tp, grads)):
            rp, rm, rv, _ = adam_ref.step(ref[i][0], g, ref[i][1], ref[i][2], t, lr, b1, b2, eps, wd)
            ref[i] = (rp, rm, rv)
            st = opt.state[p]
            for key, a, b in (("p", p.detach(), rp), ("m", st["exp_avg"], rm), ("v", st["exp_avg_sq"], rv)):
                if b.numel():
                    worst[key] = max(worst[key], float((a - b).abs().max() / b.abs().max()))
    print(f"\nworst relative difference over 60 steps: {worst}")
    assert max(worst.values()) < 1e-14, worst


def _kernel_fp32(p, g, m, v, t, lr, b1, b2, eps, wd, fp32_bias):
    """adam_kernel's operations in numpy fp32, in its order (fused multiply-adds rounded once).  fp32_bias: the
    bias corrections as an fp32 host computation would form them, 1 - b^t after rounding b^t to fp32."""
    f = np.float32
    lr, b1, b2, eps, wd = (f(x) for x in (lr, b1, b2, eps, wd))
    if fp32_bias:
        step_size = f(lr / (f(1) - np.power(b1, f(t))))
        bias2_sqrt = np.sqrt(f(1) - np.power(b2, f(t)))
    else:
        step_size = f(float(lr) / (1 - float(b1) ** t))
        bias2_sqrt = f((1 - float(b2) ** t) ** 0.5)
    fma = lambda a, b, c: f(np.float64(a) * np.float64(b) + np.float64(c))
    gg = fma(wd, p, g)
    m = fma(b1, m, (f(1) - b1) * gg)
    v = fma(b2, v, (f(1) - b2) * gg * gg)
    return p - step_size * m / (np.sqrt(v) / bias2_sqrt + eps), m, v


@pytest.mark.parametrize("fp32_bias", [False, True])
def test_errors_of_an_fp32_emulation(fp32_bias):
    """adam_ref.errors on a numpy fp32 emulation of adam_kernel, parameters at 0 (p' = -update, wd = 0): the
    kernel's order of operations stays within adam_ref.BARS; bias corrections formed in fp32 do not at t = 2, 3."""
    rs = np.random.RandomState(9)
    n = 20000
    m = np.zeros(n, np.float32)
    v = np.zeros(n, np.float32)
    worst = {}
    for t in range(1, 11):
        p = np.zeros(n, np.float32)
        g = (rs.randn(n) * 10.0 ** rs.uniform(-6, -1, n)).astype(np.float32)
        p1, m1, v1 = _kernel_fp32(p, g, m, v, t, 5e-4, 0.9, 0.999, 1e-8, 0.0, fp32_bias)
        T = lambda x: torch.from_numpy(np.asarray(x, np.float32))
        worst[t] = adam_ref.errors((T(p), T(g), T(m), T(v)), (T(p1), T(m1), T(v1)), t, 5e-4, 0.9, 0.999, 1e-8, 0.0)
        m, v = m1, v1
    print(f"\nfp32_bias={fp32_bias}: " + " ".join(f"t{t} p {e['p']:.3g}" for t, e in worst.items()))
    assert all(e["m"] <= adam_ref.BARS["m"] and e["v"] <= adam_ref.BARS["v"] for e in worst.values())
    if fp32_bias:
        assert worst[2]["p"] > adam_ref.BARS["p"] or worst[3]["p"] > adam_ref.BARS["p"]
    else:
        assert all(e["p"] <= adam_ref.BARS["p"] for e in worst.values())


def test_ulp32():
    x = torch.tensor([0.0, 1.0, -1.0, 1.5, 2.0 ** -130, 3e38], dtype=torch.float64)
    u = adam_ref.ulp32(x)
    assert u[0] == 2.0 ** -149 and u[1] == 2.0 ** -23 and u[2] == 2.0 ** -23 and u[3] == 2.0 ** -23
    assert u[4] == 2.0 ** -149
    assert u[5] == float(np.spacing(np.float32(3e38)))


def test_fp32_hyper_parameters_matter():
    """The reference rounds beta2 = 0.999 to fp32 (0.99900001287...) as the kernel sees it: its 1 - b2 differs
    from 1e-3 by 1.3e-5 relative, far above the float64 agreement above, so the rounding is not a no-op."""
    p = torch.zeros(1, dtype=torch.float64)
    g = torch.ones(1, dtype=torch.float64)
    _, _, v, _ = adam_ref.step(p, g, p, p, 1, 1e-3, 0.9, 0.999, 1e-8, 0.0)
    assert abs(float(v) / 1e-3 - 1) > 1e-5
