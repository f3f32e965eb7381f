"""CPU checks of the float64 replica of early ray termination (tests/early_stop_ref.py) at its edges: eps = 0 and
eps = 1, NaN sigma and NaN transmittance, a cut in the last word, words with every sample skipped, plain rays, and
the count of evaluated samples a cut would drop."""
import numpy as np
import pytest

from tests import early_stop_ref as es

F32 = np.float32


def _rays(n, near=2.0, far=6.0):
    r = np.zeros((n, 8), F32)
    r[:, 5] = 1.0                       # d = +z, |d| = 1
    r[:, 6], r[:, 7] = near, far
    return r


def _z(n, S, near=2.0, far=6.0):
    return np.tile(np.linspace(near, far, S, dtype=F32), (n, 1))


def test_eps_zero_never_cuts():
    rng = np.random.default_rng(0)
    S = 128
    sigma = rng.uniform(0, 1e4, (50, S)).astype(F32)     # opaque: T underflows towards 0 but never below 0
    cut, t = es.cut_words(_rays(50), _z(50, S), sigma, 0.0)
    assert (cut == -1).all() and np.isnan(t).all()


def test_eps_one_cuts_after_the_first_round_with_any_alpha():
    S = 64
    sigma = np.zeros((3, S), F32)
    sigma[0, 5] = 1e-3                  # alpha ~ 6.3e-5 in word 0
    sigma[1, 40] = 1e-3                 # only in word 1
    cut, t = es.cut_words(_rays(3), _z(3, S), sigma, 1.0)
    assert cut.tolist() == [0, 1, -1]   # the all-empty ray: T = (1 + 1e-10)^64 > 1
    assert 0 < t[0] < 1 and 0 < t[1] < 1


def test_hand_computed_transmittance():
    S = 32
    sigma = np.zeros((1, S), F32)
    sigma[0, 3] = 2.0
    z = _z(1, S)
    delta = float(F32(z[0, 4] - z[0, 3]))
    want = (1.0 - (1.0 - np.exp(-delta * 2.0)) + 1e-10) * (1.0 + 1e-10) ** 31
    T = es.word_transmittance(_rays(1), z, sigma)
    assert T.shape == (1, 1) and abs(T[0, 0] - want) <= 1e-14 * want   # a different product order


def test_nan_sigma_counts_as_zero():
    S = 64
    sigma = np.zeros((2, S), F32)
    sigma[:, 10] = 50.0
    sigma[1, 3] = np.nan
    sigma[1, 50] = -np.inf              # max(sigma, 0) = 0 as well
    T = es.word_transmittance(_rays(2), _z(2, S), sigma)
    assert np.array_equal(T[0], T[1])


def test_nan_transmittance_never_cuts():
    S = 64
    z = _z(2, S)
    z[:, 11] = z[:, 10]                 # a zero interval ...
    sigma = np.zeros((2, S), F32)
    sigma[:, 10] = np.inf               # ... times an infinite sigma: alpha = NaN, so T = NaN from word 0 on
    sigma[1, 10] = 0.0
    sigma[1, 12] = 1e3                  # the finite twin is cut in word 0
    T = es.word_transmittance(_rays(2), z, sigma)
    assert np.isnan(T[0]).all()
    cut, t = es.cut_words(_rays(2), z, sigma, 1e-3)
    assert cut.tolist() == [-1, 0]


def test_cut_in_the_last_word_drops_nothing():
    S = 96
    sigma = np.zeros((1, S), F32)
    sigma[0, 80] = 1e4                  # opaque, in word 2 (the last)
    cut, t = es.cut_words(_rays(1), _z(1, S), sigma, 1e-4)
    assert cut.tolist() == [2] and t[0] < 1e-4
    assert es.dropped(np.ones((1, S), bool), cut).tolist() == [0]


def test_a_word_with_every_sample_skipped_cannot_cut():
    S = 128
    sigma = np.zeros((2, S), F32)
    sigma[:, 20] = 3.0                  # T after word 0 above eps on both rays
    sigma[1, 70] = 1e4                  # ray 1: opaque in word 2; words 1 and 3 all skipped
    eps = 1e-3
    T = es.word_transmittance(_rays(2), _z(2, S), sigma)
    assert (T[:, 0] > eps).all()
    assert T[0, 1] > T[0, 0] and T[0, 3] > T[0, 2]      # an empty word multiplies T by (1 + 1e-10)^32
    cut, _ = es.cut_words(_rays(2), _z(2, S), sigma, eps)
    assert cut.tolist() == [-1, 2]


def test_plain_rays_and_passes_are_never_cut():
    S = 64
    r = _rays(4)
    r[1, 0] = np.nan                    # non-finite origin
    r[2, 6], r[2, 7] = 6.0, 2.0         # far <= near
    r[3, 3:6] = 3e19                    # |d|^2 overflows: delta |d| is not finite
    sigma = np.full((4, S), 1e4, F32)
    cut, _ = es.cut_words(r, _z(4, S), sigma, 0.5)
    assert cut.tolist() == [0, -1, -1, -1]


def test_dropped_counts_evaluated_samples_after_the_cut():
    S = 128
    ev = np.zeros((3, S), bool)
    ev[:, ::3] = True
    cut = np.array([0, 2, -1])
    want = [ev[0, 32:].sum(), ev[1, 96:].sum(), 0]
    assert es.dropped(ev, cut).tolist() == want


@pytest.mark.parametrize("eps", [-1e-9, 1.0 + 1e-9, float("nan")])
def test_eps_outside_zero_one(eps):
    with pytest.raises(ValueError):
        es.cut_words(_rays(1), _z(1, 32), np.zeros((1, 32), F32), eps)
