"""Float64 numpy replica of early ray termination's rule (DESIGN.md §10f) for one pass of a ``skip="samples"``
render, and of what that rule would leave unevaluated.

The S samples of a ray (depth order) are taken in rounds of one mask word, 32 samples.  Sample i has
``composite_ray``'s interval ``delta_i = (z[i+1] - z[i]) |d|`` (float32 steps, ``1e10 |d|`` for the last sample) and
``alpha_i = 1 - exp(-delta_i max(sigma_i, 0))``, where ``max`` is ``fmaxf`` (a NaN sigma counts as 0, as in
``composite_ray``) and the product and the exponential are float64.  A skipped sample has sigma = 0.  After round k
the ray's transmittance is ``T_k = T_{k-1} * prod over word k of (1 - alpha_i + 1e-10)`` (float64, ``T_{-1} = 1``).
The ray is *cut* at the first word k with ``T_k < eps``; every sample of a later word would then be treated as
empty.  A ray whose T is NaN never satisfies ``T < eps``.  A plain ray (a non-finite value or ``far <= near``) and a
pass whose interval lengths are not all finite (``sample_skip_ref.plain_pass``) are never cut.
"""
import numpy as np

from tests import sample_skip_ref as sk

F32 = np.float32
WORD = 32


def alphas(rays, z, sigma):
    """(R, S) float64 alpha of the samples at depths z (R, S) with sigma (R, S) (float32 inputs)."""
    r = np.asarray(rays, F32)
    z = np.asarray(z, F32)
    s = np.fmax(np.asarray(sigma, F32), F32(0))
    d = r[:, 3:6]
    with np.errstate(over="ignore", invalid="ignore"):
        dn = np.sqrt(((d[:, 0] * d[:, 0]).astype(F32) + (d[:, 1] * d[:, 1]).astype(F32)).astype(F32)
                     + (d[:, 2] * d[:, 2]).astype(F32)).astype(F32)
        delta = np.concatenate([(z[:, 1:] - z[:, :-1]).astype(F32), np.full((z.shape[0], 1), 1e10, F32)], 1)
        delta = (delta * dn[:, None]).astype(F32)
        return 1.0 - np.exp(-(delta.astype(np.float64) * s.astype(np.float64)))


def word_transmittance(rays, z, sigma):
    """(R, S / 32) float64: T after each round."""
    a = alphas(rays, z, sigma)
    R, S = a.shape
    if S % WORD:
        raise ValueError("S must be a multiple of 32")
    f = (1.0 - a + 1e-10).reshape(R, S // WORD, WORD)
    with np.errstate(invalid="ignore", over="ignore"):
        return np.cumprod(np.prod(f, axis=2), axis=1)


def cut_words(rays, z, sigma, eps):
    """(cut (R) int64, t_cut (R) float64): the word after which each ray stops (-1: never) and T after that word
    (NaN where the ray is not cut)."""
    eps = float(eps)
    if not 0.0 <= eps <= 1.0:
        raise ValueError("eps must be in [0, 1]")
    T = word_transmittance(rays, z, sigma)
    with np.errstate(invalid="ignore"):
        below = T < eps
    below[sk.plain_pass(rays, z)] = False
    hit = below.any(1)
    cut = np.where(hit, below.argmax(1), -1).astype(np.int64)
    t_cut = np.full(T.shape[0], np.nan)
    t_cut[hit] = T[hit, cut[hit]]
    return cut, t_cut


def dropped(evaluated, cut):
    """(R,) int64: the evaluated samples (evaluated: (R, S) bool) that lie in words after each ray's cut."""
    ev = np.asarray(evaluated, bool)
    R, S = ev.shape
    word = np.arange(S) // WORD
    after = (cut[:, None] >= 0) & (word[None, :] > cut[:, None])
    return (ev & after).sum(1)
