"""The float64 SSIM restatement (tests/ssim_ref.py) the device kernel is checked against: closed forms where they
exist, the zero-padded edges, batches and channel counts, the clamp kornia 0.2.0 applies, and the float32
composition kornia itself runs."""
import numpy as np
import pytest

from tests import ssim_ref as sr

# float32 torch (kornia 0.2.0's composition) against float64, measured on the cases of
# test_float32_composition_agrees: at most 1.07e-5 per pixel and 1.0e-7 on the mean.  The bars leave about 5x.
F32_PIXEL_BAR, F32_MEAN_BAR = 5e-5, 5e-7


def _images(shape, seed, close=False):
    rng = np.random.default_rng(seed)
    x = rng.random(shape).astype(np.float32)
    y = np.clip(x + rng.normal(0, 0.02, shape), 0, 1).astype(np.float32) if close else \
        rng.random(shape).astype(np.float32)
    return x, y


def _inside_weight(H, W):
    """(H, W): the window weight that falls inside the image at every pixel."""
    return sr._filter(np.ones((1, 1, H, W)))[0, 0]


def test_window_is_the_normalised_gaussian_outer_product():
    w = sr.window()
    g = np.exp(-np.array([1.0, 0.0, 1.0]) / 4.5)
    assert np.allclose(w, np.outer(g, g) / g.sum() ** 2, rtol=0, atol=1e-16)
    assert abs(w.sum() - 1.0) < 1e-15 and np.array_equal(w, w.T)


@pytest.mark.parametrize("shape", [(1, 3, 17, 23), (2, 1, 5, 4), (1, 1, 1, 1), (1, 2, 2, 2)])
def test_identical_images_give_one(shape):
    x, _ = _images(shape, 1)
    assert np.array_equal(sr.ssim(x, x, "none"), np.ones(shape))
    assert sr.ssim(x, x) == 1.0 and sr.ssim(x, x, "sum") == 1.0


@pytest.mark.parametrize("H,W", [(1, 1), (2, 2), (3, 5), (9, 7)])
@pytest.mark.parametrize("a,b", [(0.3, 0.3), (0.2, 0.9), (0.0, 1.0), (0.75, 0.0)])
def test_constant_images_follow_the_closed_form(H, W, a, b):
    """Constant planes a and b: with S the window weight inside the image, mu = a S, sigma^2 = a^2 S (1 - S) and
    sigma_xy = a b S (1 - S), so zero padding shows at every edge pixel (and everywhere for 1 x 1 and 2 x 2)."""
    a, b = float(np.float32(a)), float(np.float32(b))          # the values the float32 images hold
    S = _inside_weight(H, W)
    mu1, mu2 = a * S, b * S
    s11, s22, s12 = a * a * S * (1 - S), b * b * S * (1 - S), a * b * S * (1 - S)
    m = ((2 * mu1 * mu2 + sr.C1) * (2 * s12 + sr.C2)) / ((mu1 ** 2 + mu2 ** 2 + sr.C1) * (s11 + s22 + sr.C2))
    want = 1 - 2 * (np.clip(1 - m, 0, 1) / 2)
    x, y = np.full((1, 1, H, W), a, np.float32), np.full((1, 1, H, W), b, np.float32)
    got = sr.ssim(x, y, "none")[0, 0]
    assert np.allclose(got, want, rtol=0, atol=1e-12)
    if H == W == 1:
        g = np.exp(-1 / 4.5)
        assert np.isclose(S[0, 0], (1 / (1 + 2 * g)) ** 2, rtol=0, atol=1e-15)
    if H == W == 2:
        assert np.allclose(S, ((1 + np.exp(-1 / 4.5)) / (1 + 2 * np.exp(-1 / 4.5))) ** 2, rtol=0, atol=1e-15)


def test_batches_and_channels_are_independent_planes():
    x, y = _images((3, 5, 11, 13), 2)
    full = sr.ssim(x, y, "none")
    for b in range(3):
        for c in range(5):
            one = sr.ssim(x[b:b + 1, c:c + 1], y[b:b + 1, c:c + 1], "none")
            assert np.array_equal(full[b, c], one[0, 0])
    assert sr.ssim(x, y, "mean") == pytest.approx(1 - 2 * np.mean((1 - full) / 2), abs=1e-15)
    assert sr.ssim(x, y, "sum") == pytest.approx(1 - 2 * np.sum((1 - full) / 2), abs=1e-11)


def test_negative_ssim_map_is_clamped_as_kornia_0_2_0_does():
    """Anti-correlated images give ssim_map < 0.  kornia 0.2.0's clamp(1 - s, 0, 1) / 2 stops at 1/2, so metrics.ssim
    is 0 there; later kornia's clamp((1 - s) / 2, 0, 1) goes above 1/2 and would make it negative."""
    rng = np.random.default_rng(3)
    x = (rng.random((1, 1, 24, 24)) > 0.5).astype(np.float32)
    y = 1 - x
    s = sr.ssim_map(x, y)
    neg = s < 0
    assert neg.sum() > 50
    assert np.all(sr.ssim(x, y, "none")[neg] == 0.0)
    later = 1 - 2 * sr.dssim_later_kornia(x, y, "none")
    assert np.all(later[neg] < 0) and np.allclose(later[neg], s[neg], rtol=0, atol=1e-15)
    assert np.array_equal(sr.ssim(x, y, "none")[~neg], later[~neg])
    assert sr.ssim(x, y) > 1 - 2 * sr.dssim_later_kornia(x, y)


def test_nan_propagates():
    x, y = _images((1, 1, 6, 6), 4)
    x[0, 0, 2, 3] = np.nan
    m = sr.ssim(x, y, "none")[0, 0]
    assert np.isnan(m[1:4, 2:5]).all() and np.isfinite(m).sum() == 36 - 9
    assert np.isnan(sr.ssim(x, y))


@pytest.mark.parametrize("shape,close", [((1, 3, 64, 64), False), ((1, 3, 64, 64), True), ((2, 1, 33, 47), False),
                                         ((2, 1, 33, 47), True), ((1, 3, 200, 200), False), ((1, 3, 200, 200), True)])
def test_float32_composition_agrees(shape, close):
    x, y = _images(shape, 5, close)
    got = sr.ssim_torch_f32(x, y, "none").numpy()
    assert got.dtype == np.float32
    assert np.abs(got - sr.ssim(x, y, "none")).max() < F32_PIXEL_BAR
    assert abs(float(sr.ssim_torch_f32(x, y)) - sr.ssim(x, y)) < F32_MEAN_BAR
    assert abs(float(sr.ssim_torch_f32(x, y, "sum")) - sr.ssim(x, y, "sum")) < F32_MEAN_BAR * x.size
