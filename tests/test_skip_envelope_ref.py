"""CPU checks of the fixtures of tests/test_gpu_skip_envelope.py: the pair matrix is the whole envelope with every
option value on a 96- and a 160-sample fine pass, the designed coarse patterns and counted rows are what the float64
rule (tests/sample_skip_ref.py) gives, the vectorised rule equals the loop, and each planted defect of the envelope's
comparisons exceeds its bar."""
import numpy as np
import pytest

from tests import sample_skip_ref as sk
from tests import test_gpu_sample_skip as ss
from tests import test_gpu_skip_envelope as env
from tests import test_gpu_train_skip as ts
from tests import test_sample_skip_ref as hand
from tests import train_skip_ref as tr
from tests import train_skip_seed_ref as seed_ref

F32 = np.float32


def test_matrix_is_the_whole_envelope():
    accepted = {(S, K) for S in (32, 64, 128) for K in range(0, 193, 32) if S + K <= 192}
    assert set(env.MATRIX) == accepted and len(accepted) == 14
    assert set(ts.PAIRS) == accepted and set(ss.SHAPES) == accepted      # "nothing to skip" covers every pair
    for sf in (96, 160):
        specs = [c for (S, K), c in env.MATRIX.items() if K and S + K == sf]
        for opt, values in env.OPTIONS.items():
            assert {c[opt] for c in specs} == values, (sf, opt)
    assert all(not c["use_disp"] or c["kind"] == "blender" for c in env.MATRIX.values())
    assert all(40 <= c["n"] <= 100 for c in env.MATRIX.values())
    # the patterned rays reach fine passes of 3, 5 and 6 samples per lane and coarse passes of 1, 2 and 4 words
    assert {(S + K) // 32 for S, K in env.PAT_PAIRS if K} >= {3, 5, 6}
    assert {S for S, _ in env.PAT_PAIRS} == {32, 64, 128}


# ------------------------------------------------------------------------------------------ the vectorised rule
def _both(points, words, N, ranges):
    a = sk.point_evaluated(points, words, N, ranges)
    b = sk.point_evaluated_vec(points, words, N, ranges)
    assert a.shape == b.shape
    return a, b


def test_vectorised_rule_equals_the_loop_on_the_hand_cases():
    cases = [([[1.5, 2.5, 0.5]], [(1, 2, 0)], hand.BOX), ([[1.5, 2.5, 0.5]], [(2, 2, 0)], hand.BOX),
             ([[2.0, 1.5, 1.5], [1.0, 1.5, 1.5], [2.0, 2.0, 1.5], [1.0, 1.0, 1.0], [2.0, 2.0, 2.0]], [(1, 1, 1)],
              hand.BOX),
             ([[np.nextafter(F32(2.0), F32(3.0)), 1.5, 1.5], [np.nextafter(F32(1.0), F32(0.0)), 1.5, 1.5]],
              [(1, 1, 1)], hand.BOX),
             ([[0.0, 0.0, 0.0], [4.0, 4.0, 4.0], [0.0, 0.5, 1.0], [-1e-6, 0.5, 0.5], [4.0000005, 3.5, 3.5],
               [np.nan, 0.5, 0.5], [np.inf, 3.5, 3.5]], [(0, 0, 0), (3, 3, 3)], hand.BOX),
             ([[0.5, 3.5, 0.5], [0.5, 0.5, 0.5], [0.5, 3.0, 0.5]], [(0, 0, 0), (0, 1, 0)], (0.0, 4.0, 4.0, 0.0, 0.0, 4.0))]
    for c in [(2, 2, 2), (1, 2, 2), (2, 1, 1), (1, 1, 2)]:
        cases.append(([[2.0, 2.0, 2.0]], [c], hand.BOX))
    for pts, cells, ranges in cases:
        a, b = _both(np.asarray(pts, F32), hand._words(cells, hand.M), hand.N, ranges)
        assert np.array_equal(a, b), (pts, cells)


@pytest.mark.parametrize("N", [2, 5, 11, 34])
def test_vectorised_rule_equals_the_loop_on_random_points(N):
    """Random points inside and around the box, a third of them moved onto lattice planes, lines and corners."""
    rng = np.random.default_rng(N)
    M = N - 1
    for ranges in ((0.0, float(M)) * 3, (-2.0, 2.0, 2.0, -2.0, -1.5, 2.5), (float(M), 0.0) * 3):
        lo, hi = np.array(ranges[0::2]), np.array(ranges[1::2])
        g = rng.uniform(-0.3, M + 0.3, (3000, 3))
        g[:1000] = np.round(g[:1000])
        g[1000:1500, :2] = np.round(g[1000:1500, :2])
        x = (lo + g * (hi - lo) / M).astype(F32)
        x[-5:, 1] = np.nan
        words = env.cell_words(N, 0.3, N)
        a, b = _both(x, words, N, ranges)
        assert np.array_equal(a, b), ranges
        assert a.any() and not a.all()


def test_touched_cells_of_a_corner():
    cells = sk.touched_cells(np.array([[2.0, 2.0, 2.0], [2.5, 2.0, 2.5], [9.0, 0.0, 0.0]], F32), 5, hand.BOX)
    assert sorted(set(cells[0])) == sorted((cz * 4 + cy) * 4 + cx for cz in (1, 2) for cy in (1, 2) for cx in (1, 2))
    assert sorted(set(cells[1])) == [(2 * 4 + 1) * 4 + 2, (2 * 4 + 2) * 4 + 2]
    assert (cells[2] == -1).all()


# ------------------------------------------------------------------------------------------ the designed fixtures
@pytest.mark.parametrize("S", [32, 64, 128])
def test_patterns_are_the_float64_rule(S):
    pats = env.coarse_patterns(S)
    assert {"empty", "full", "first", "last", "only31", "even", "odd", "random"} <= set(pats)
    if S > 32:
        assert {"only32", "31and32"} <= set(pats)
    assert sum(k.startswith("word") for k in pats) == S // 32
    masks = np.stack(list(pats.values()) * 2)
    rays, words = env.pattern_case(masks)
    z = sk.z_base(rays, S)
    assert np.array_equal(sk.evaluated(rays, z, words, env.PAT_M + 1, env.PAT_RANGES), masks)
    assert np.array_equal(sk.point_evaluated(sk.sample_points(rays[:3], z[:3]), words, env.PAT_M + 1, env.PAT_RANGES),
                          masks[:3])


@pytest.mark.parametrize("total", env.TOTALS)
def test_counted_rows_are_the_float64_rule(total):
    S, n = 64, 6
    masks = env.counted_masks(total, n, S)
    assert masks.sum() == total
    rows = np.stack([np.arange(n), np.zeros(n, int)], 1)
    if total:
        last = int(np.nonzero(masks.any(1))[0][-1])
        assert masks[last].sum() == 1 and masks[last, 0]          # the last row is alone at transmittance 1
        rows[last] = (77, 64)
    rays, words = env.pattern_case(masks, rows)
    assert np.array_equal(sk.evaluated(rays, sk.z_base(rays, S), words, env.PAT_M + 1, env.PAT_RANGES), masks)


def test_straddle_detection():
    ev = np.zeros((1, 96), bool)
    assert not env.straddles(ev, 3)
    ev[0, [31, 32]] = True                  # lane 10 holds 30, 31, 32: 30 skipped, 31 and 32 across the word
    assert env.straddles(ev, 3)
    assert not env.straddles(np.random.default_rng(0).random((50, 64)) < 0.5, 2)     # P = 2 never straddles


@pytest.mark.parametrize("kind", ["plane", "line", "corner"])
def test_lattice_rays_lie_on_the_lattice(kind):
    M = 64
    rays, words = env.lattice_case(kind, 60, 1, M)
    x = sk.sample_points(rays, sk.z_base(rays, 32)).reshape(-1, 3)
    on = (x == np.round(x))
    want = {"plane": [False, True, False], "line": [False, True, True], "corner": [None, True, True]}[kind]
    for a, w in enumerate(want):
        if w is not None:
            assert on[:, a].all() == w and (w or not on[:, a].any()), (kind, a)
    if kind == "corner":
        assert on[:, 0].mean() > 0.8
    cells = sk.touched_cells(x, M + 1, (0.0, float(M)) * 3)
    occupied = sk.bit(words, np.maximum(cells, 0)) & (cells >= 0)
    # at most one touched cell is occupied: a wrong neighbour changes the answer
    distinct = np.array([len(set(c[o])) for c, o in zip(cells, occupied)])
    assert distinct.max() == 1 and 0.2 < (distinct == 1).mean() < 0.9


# ------------------------------------------------------------------------------------------ planted defects
def _pass(seed, R=60, S=96):
    rng = np.random.default_rng(seed)
    z = np.sort(rng.uniform(2, 6, (R, S)), 1).astype(F32)
    ev = rng.random((R, S)) < 0.4
    sigma = rng.uniform(-1, 20, (R, S)).astype(F32)
    rgb = rng.uniform(0, 1, (R, S, 3)).astype(F32)
    dirs = rng.normal(size=(R, 3)).astype(F32)
    noise = rng.normal(size=(R, S)).astype(F32)
    return z, ev, sigma, rgb, dirs, noise


def test_planted_backward_defects_exceed_the_bar():
    """The per-row comparisons against train_skip_ref.backward and train_skip_seed_ref.backward reject a mask
    shifted by one sample, rows starting one row late and the other pass's seed, on the references' own values."""
    rng = np.random.default_rng(5)
    z, ev, sigma, rgb, dirs, noise = _pass(1)
    R = z.shape[0]
    target = rng.uniform(0, 1, (R, 3))
    out, other = rng.uniform(0, 1, (R, 3)), rng.uniform(0, 1, (R, 3))
    mse = lambda ev_=ev, o=out: tr.backward(z, sigma, rgb, ev_, dirs, noise, 1.0, True, o, target, R)  # noqa: E731
    wr, wd, wo = rng.normal(size=(R, 3)), rng.normal(size=R), rng.normal(size=R)
    gen = lambda ev_=ev, s=1.0: seed_ref.backward(z, sigma, rgb, ev_, dirs, noise, 1.0, False,  # noqa: E731
                                                  wr * s, wd * s, wo * s)
    for name, ref_fn, swapped in (("mse", mse, dict(o=other)), ("seed", gen, dict(s=-0.5))):
        ds_ref, dp_ref = ref_fn()
        assert max(tr.backward_errors(ds_ref[ev], dp_ref[ev], ev, ds_ref, dp_ref)) == 0.0
        bds, bdp = ref_fn(ev_=ev & np.roll(ev, 1, 1))
        assert max(tr.backward_errors(bds[ev], bdp[ev], ev, ds_ref, dp_ref)) > tr.BWD_BAR, name
        assert max(tr.backward_errors(env._shift_rows(ds_ref, ev), env._shift_rows(dp_ref, ev), ev, ds_ref,
                                      dp_ref)) > tr.BWD_BAR, name
        bds, bdp = ref_fn(**swapped)
        assert max(tr.backward_errors(bds[ev], bdp[ev], ev, ds_ref, dp_ref)) > tr.BWD_BAR, name


def test_planted_padding_copies_fail_the_gradient_bars():
    """A weight gradient sum_rows a_r d_r^T whose last row carries the large gradient of the row-total fixture: with
    the 127 (or one) padding copies of the last row counted it fails test_gpu_train_skip._grad_bars."""
    rng = np.random.default_rng(2)
    for rows, copies in ((129, 127), (1, 127), (127, 1), (255, 1)):
        a = rng.normal(size=(rows, 64))
        d = rng.normal(size=(rows, 4)) * 1e-2
        d[-1] *= 40.0 * 100
        ref = {"0.w": a.T @ d, "0.b": d.sum(0)}
        ts._grad_bars(dict(ref), ref)
        bad = {"0.w": ref["0.w"] + copies * np.outer(a[-1], d[-1]), "0.b": ref["0.b"] + copies * d[-1]}
        with pytest.raises(AssertionError):
            ts._grad_bars(bad, ref)
