"""The float64 restatement of the density grid update (tests/density_ref.py) at its edges: decay 0 and 1, NaN sigma,
N = 2, a cell count that is not a multiple of 32, reversed and unequal ranges."""
import struct

import numpy as np
import pytest

from . import density_ref as dr
from . import occupancy_ref as oc
from . import philox

UNEQUAL = ((-1.5, 1.5), (1.4, -1.2), (-0.5, 2.25))          # y reversed


def _philox_scalar(seed, ray, i, stream):
    """One uniform with Python integers (the counter and key schedule of csrc/render_kernel.cuh philox_uniform)."""
    c = [ray & 0xFFFFFFFF, i >> 2, stream, 0]
    k0, k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k0, p1 & 0xFFFFFFFF, (p0 >> 32) ^ c[3] ^ k1, p0 & 0xFFFFFFFF]
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return (c[i & 3] >> 8) * 2.0 ** -24


@pytest.mark.parametrize("N, ranges", [(2, ((-1.0, 1.0),) * 3), (5, UNEQUAL), (17, ((3.0, -3.0),) * 3)])
def test_points_restate_the_rule_cell_by_cell(N, ranges):
    """Every point against a scalar evaluation of steps 1-2 with Python floats (IEEE doubles, one rounding per
    operation), and inside its cell's closed box."""
    seed = (1 << 63) + 12345                          # a key with the top bit set (a negative int64 on the device)
    p = dr.points(seed, N, ranges)
    M = N - 1
    assert p.shape == (M ** 3, 3) and p.dtype == np.float32
    for c in list(range(min(M ** 3, 40))) + [M ** 3 - 1]:
        cell = (c % M, (c // M) % M, c // (M * M))
        for a in range(3):
            lo, hi = ranges[a]
            want = lo + (float(cell[a]) + _philox_scalar(seed, c, a, 2)) * ((hi - lo) / M)
            assert p[c, a] == struct.unpack("f", struct.pack("f", want))[0], (c, a)
    lo = np.array([r[0] for r in ranges])
    step = (np.array([r[1] for r in ranges]) - lo) / M
    a_end, b_end = lo + dr.cells(N) * step, lo + (dr.cells(N) + 1) * step
    lower, upper = np.minimum(a_end, b_end).astype(np.float32), np.maximum(a_end, b_end).astype(np.float32)
    assert np.all(p >= lower) and np.all(p <= upper)
    u = philox.uniform(seed, M ** 3, 3, 2)
    if M ** 3 >= 7:
        assert np.array_equal(dr.points(seed, N, ranges, 3, 4), p[3:7])
    assert not np.array_equal(dr.points(seed + 1, N, ranges), p)      # the key moves the jitter
    assert np.all((u >= 0) & (u < 1))


def test_initial_state_has_every_cell_occupied_and_no_bit_past_the_last_cell():
    for N in (2, 4, 5, 33):                           # 1, 27, 64 and 32768 cells
        st = dr.initial(N, 7)
        C = (N - 1) ** 3
        assert st["key"] == 7 and not st["density"].any()
        assert oc.unpack_bits(st["bits"], N).all()
        assert st["bits"].shape == ((C + 31) // 32,)
        assert int(sum(bin(int(w)).count("1") for w in st["bits"])) == C


def test_decay_zero_and_one():
    d = np.array([0.0, 3.0, 5.0, 2.0], np.float32)
    s = np.array([1.0, 1.0, 9.0, -4.0], np.float32)
    assert np.array_equal(dr.decay_max(d, s, 0.0), [1.0, 1.0, 9.0, 0.0])          # decay 0: the new sigma, >= 0
    assert np.array_equal(dr.decay_max(d, s, 1.0), [1.0, 3.0, 9.0, 2.0])          # decay 1: the running maximum
    half = dr.decay_max(d, s, 0.5)
    assert np.array_equal(half, [1.0, 1.5, 9.0, 1.0]) and half.dtype == np.float32
    # decay is a float32: 0.95 * 3 rounds as float32(0.95) * float32(3) does
    assert dr.decay_max([3.0], [0.0], 0.95)[0] == np.float32(np.float32(0.95) * np.float32(3.0))


def test_nan_sigma_counts_as_zero():
    d = np.array([4.0, 0.0], np.float32)
    out = dr.decay_max(d, np.array([np.nan, np.nan], np.float32), 0.5)
    assert np.array_equal(out, [2.0, 0.0]) and np.isfinite(out).all()


def test_threshold_dilation_and_packing():
    N = 6                                             # 125 cells: the last word holds 29 of them
    d = np.zeros(125, np.float32)
    d[(2 * 5 + 3) * 5 + 1] = 2.0                      # cell (1, 3, 2)
    d[0] = 1.0                                        # at the threshold: not occupied
    occ = dr.occupied(d, N, 1.0, 0)
    assert occ.sum() == 1 and occ[1, 3, 2]
    assert dr.occupied(d, N, 1.0, 1).sum() == 27
    assert dr.occupied(d, N, 1.0, 9).all()            # a radius past the grid fills it
    w = dr.bits(d, N, 1.0, 9)
    assert w.shape == (4,) and int(w[-1]) == (1 << 29) - 1
    # the threshold is compared in float64: a density just above a non-float32 threshold counts
    assert dr.occupied(np.full(1, np.float32(0.1), np.float32), 2, 0.1, 0)[0, 0, 0]


def test_update_sequence_advances_the_key_and_decays():
    N, ranges = 4, UNEQUAL
    st = dr.initial(N, 100)
    keys = []
    for k in range(3):
        sigma = (lambda p: np.where(p[:, 0] > 0, 5.0, -1.0).astype(np.float32)) if k == 0 else \
            (lambda p: np.full(len(p), np.nan, np.float32))
        st = dr.update(st, sigma, N, ranges, 1.0, 0.5, 0)
        keys.append(st["key"])
    assert keys == [101, 102, 103]
    occ = oc.unpack_bits(st["bits"], N)
    assert np.array_equal(occ, (st["density"].reshape(3, 3, 3).transpose(2, 1, 0) > 1.0))
    assert set(np.unique(st["density"])) <= {0.0, 1.25}       # 5 decayed twice by 0.5; NaN counted as 0
    assert occ.any() and not occ.all()
