"""Adam in float64, as the reference of FusedAdam (nerf_pl_b200/optim.py, adam_kernel in csrc/bwd_kernels.cuh).

The kernel receives its hyper-parameters as fp32 and keeps p, m and v in fp32.  So ``step`` rounds the
hyper-parameters to fp32 first, then evaluates everything else in float64 from those values: 1 - beta (exact in
the kernel too, by Sterbenz), the bias corrections and lr / (1 - b1^t).  Fed the kernel's own fp32 state of step
t - 1, what remains between the two is the kernel's own rounding of step t.

Works on torch tensors of any device (float64 work stays on that device).
"""
import numpy as np
import torch


# Bars on `errors` for FusedAdam (tests/test_gpu_train_loop.py), worst measured on an H100 80GB HBM3 in brackets.
# The kernel rounds m twice, v four times and p about eight times (tests/test_adam_ref.py emulates its order); a
# relative error of k 2^-23 is k to 2k ulps, depending on where in its binade the value lies.  Bias corrections formed
# in fp32, the defect these bars are set against, are 59 ulps of the update wrong at t = 2.
BARS = {
    "m": 3.0,       # [1.5]
    "v": 4.0,       # [2.7]
    "p": 8.0,       # [4.8, in the training run; 3.9 elsewhere]
}


def f32(x):
    """x rounded to fp32, as a Python float."""
    return float(np.float32(x))


def step(p, g, m, v, t, lr, b1, b2, eps, wd):
    """One Adam step at step number t (1-based).  Returns (p', m', v', update) in float64, p' = p - update:
    g' = g + wd p;  m' = b1 m + (1 - b1) g';  v' = b2 v + (1 - b2) g'^2;
    p' = p - lr / (1 - b1^t) * m' / (sqrt(v') / sqrt(1 - b2^t) + eps)."""
    lr, b1, b2, eps, wd = (f32(x) for x in (lr, b1, b2, eps, wd))
    p, g, m, v = (x.to(torch.float64) for x in (p, g, m, v))
    g = g + wd * p
    m = b1 * m + (1.0 - b1) * g
    v = b2 * v + (1.0 - b2) * g * g
    t = int(t)
    step_size = lr / (1.0 - b1 ** t)
    bias2_sqrt = (1.0 - b2 ** t) ** 0.5
    upd = step_size * m / (v.sqrt() / bias2_sqrt + eps)
    return p - upd, m, v, upd


def errors(before, after, t, lr, b1, b2, eps, wd):
    """Worst errors of one step of an fp32 implementation.  ``before`` = (p, g, m, v) it was given (fp32),
    ``after`` = (p, m, v) it produced.  In fp32 ulps:
      m: |m - m_ref| / ulp(largest of |b1 m|, |(1 - b1) g'|, |m_ref|)  (m is a sum that may cancel: its rounding
         is bounded by its largest term, not by the result);
      v: |v - v_ref| / ulp(v_ref)  (a sum of two non-negative terms);
      p: (|p - p_ref| - 0.5 ulp(p_ref)) / ulp(u), u = the update with m replaced by the largest term above, so
         ulp(u) = ulp(update) where m does not cancel.  0.5 ulp(p_ref) is the final rounding of p - update."""
    p0, g, m0, v0 = before
    p1, m1, v1 = (x.to(torch.float64) for x in after)
    if p1.numel() == 0:
        return {"m": 0.0, "v": 0.0, "p": 0.0}
    pr, mr, vr, _ = step(p0, g, m0, v0, t, lr, b1, b2, eps, wd)
    lr, b1, b2, eps, wd = (f32(x) for x in (lr, b1, b2, eps, wd))
    gd = g.to(torch.float64) + wd * p0.to(torch.float64)
    m_big = torch.maximum(torch.maximum((b1 * m0.to(torch.float64)).abs(), ((1.0 - b1) * gd).abs()), mr.abs())
    u_big = lr / (1.0 - b1 ** int(t)) * m_big / (vr.sqrt() / (1.0 - b2 ** int(t)) ** 0.5 + eps)
    ep = ((p1 - pr).abs() - 0.5 * ulp32(pr)).clamp_min(0) / ulp32(u_big)
    return {"m": float(((m1 - mr).abs() / ulp32(m_big)).max()),
            "v": float(((v1 - vr).abs() / ulp32(vr)).max()),
            "p": float(ep.max())}


def ulp32(x):
    """The spacing of fp32 at |x| (x rounded to fp32 first), as float64; the least subnormal at 0."""
    a = x.to(torch.float32).abs()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).to(torch.float64)
