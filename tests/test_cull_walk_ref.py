"""The cell walk's rule (tests/occupancy_ref.ray_live, DESIGN.md §10 "Live") against a brute-force float64 slab test
of every cell's grown box, and against the lookup: every sample point the renderer can place on a segment that the
lookup (cascade_ref.point_evaluated) evaluates lies on a live ray.  On the designed families of
tests/cull_walk_cases.py and on random sparse cascades."""
import numpy as np
import pytest

from . import cascade_ref as cr
from . import cull_walk_cases as cw
from . import occupancy_ref as oc
from . import sample_skip_ref as ss

F32 = np.float32
CUBE = (-1.0, 1.0, -1.0, 1.0, -1.0, 1.0)
REVERSED = (1.0, -1.0, -0.5, 1.5, 3.0, 2.0)
UNEQUAL = (-1.0, 1.0, 1.25, -0.75, -0.5, 0.5)
RANGES = {"forward": CUBE, "reversed": REVERSED, "unequal": UNEQUAL}


def brute_live(rays, words, N, L, ranges):
    occ = cr.unpack(words, N, L)
    live = np.zeros(len(rays), bool)
    for k in range(L):
        live |= oc.brute_live(rays, occ[k], cr.pairs(cr.level_ranges(ranges, k)))
    return live


def crossing_depths(rays, N, L, ranges):
    """(R, P) float32 depths in [near, far]: 65 evenly spaced ones, and around every time the segment crosses a
    lattice plane of some level, that time rounded to float32 and its float32 neighbour either way."""
    r = np.asarray(rays, F32).astype(np.float64)
    zs = [np.linspace(r[:, 6], r[:, 7], 65, axis=1)]
    for k in range(L):
        lo, hi = cw.level_box(ranges, k)
        planes = lo[:, None] + (hi - lo)[:, None] * (np.arange(N) / (N - 1))[None, :]       # (3, N)
        for a in range(3):
            with np.errstate(divide="ignore", invalid="ignore"):
                t = (planes[a][None, :] - r[:, a:a + 1]) / r[:, 3 + a:4 + a]
            t = np.where(np.isfinite(t), t, r[:, 6:7])
            zs.append(t)
    z = np.concatenate(zs, 1).astype(F32)
    near = r[:, 6:7].astype(F32)
    far = r[:, 7:8].astype(F32)
    z = np.concatenate([z, np.nextafter(z, F32(np.inf)), np.nextafter(z, F32(-np.inf))], 1)
    return np.clip(z, near, far)


def lookup_hits(rays, words, N, L, ranges):
    """(R,) bool: some point the renderer places on the ray is evaluated: z_base at S in {32, 64, 128} with and
    without use_disp (where near > 0), and the dense depths of crossing_depths."""
    r = np.asarray(rays, F32)
    hit = np.zeros(len(r), bool)
    zs = [crossing_depths(r, N, L, ranges)]
    for S in (32, 64, 128):
        zs.append(ss.z_base(r, S))
        pos = r[:, 6] > 0
        if pos.any():
            z = ss.z_base(r, S, use_disp=True)
            zs.append(np.where(pos[:, None], z, r[:, 6:7]))
    for z in zs:
        with np.errstate(invalid="ignore", over="ignore"):
            hit |= cr.point_evaluated(ss.sample_points(r, z), words, N, L, ranges).any(1)
    return hit


CONFIGS = [(9, 1, "forward"), (9, 2, "forward"), (8, 3, "reversed"), (9, 4, "unequal"), (6, 2, "unequal")]


@pytest.mark.parametrize("N, L, rname", CONFIGS)
def test_designed_families_restatement_equals_brute_force_and_covers_the_lookup(N, L, rname):
    ranges = RANGES[rname]
    total = {f: [0, 0] for f in cw.FAMILIES}
    rounded = 0
    for k, cell in cw.target_cells(N, L):
        words = cw.one_cell_words(N, L, k, cell)
        for f in cw.FAMILIES:
            rays = cw.family(f, ranges, N, L, k, cell, seed=N + k)
            if not len(rays):
                continue
            live = cr.ray_live(rays, words, N, L, ranges)
            assert np.array_equal(live, brute_live(rays, words, N, L, ranges)), (f, k, cell)
            hit = lookup_hits(rays, words, N, L, ranges)
            lost = hit & ~live
            assert not lost.any(), (f, k, cell, rays[lost][:3])
            if f == "probes":         # d = 0: every sample is o itself, and the walk's growth is 0
                assert np.array_equal(live, cw.touches_any_level(rays[:, :3], words, N, L, ranges)), (k, cell)
            if f == "misses":
                assert not live.any(), (k, cell)
            if f == "rounding":       # the exact segment stops short of the face its last sample lands on
                assert live.all()
                rounded += int(hit.sum())
            total[f][0] += int(live.sum())
            total[f][1] += len(rays)
    for f in ("probes", "axis"):
        assert 0 < total[f][0] < total[f][1], (f, total[f])
    if N == 9:                # exact lattice points: every one of them touches the cell
        assert total["points"][0] == total["points"][1]
    assert total["rounding"][0] > 0
    if N == 9:                # a power-of-two cell: the face is a float32, so a landed sample is evaluated
        assert rounded > 0
    print(f"\nN {N} L {L} {rname}: live / rays {total}; {rounded} rounding rays with an evaluated sample")


def test_the_issue_examples():
    """A ray along +z on x = y = 0 beside one occupied cell; a diagonal whose sample sits on the cell's corner; a ray
    whose last float32 sample rounds onto the cell's face; a ray in a level-0 face plane past an occupied level-1
    cell.  Each is live, and each has an evaluated sample."""
    N = 9
    M = N - 1
    occ = np.zeros((1, M, M, M), bool)
    occ[0, 3, 3, 4] = True
    words = cr.pack(occ)
    ray = np.array([[0, 0, -1, 0, 0, 1, 0, 2]], F32)
    assert cr.ray_live(ray, words, N, 1, CUBE).all() and lookup_hits(ray, words, N, 1, CUBE).all()
    occ = np.zeros((1, M, M, M), bool)
    occ[0, 4, 3, 3] = True                                    # x [0, .25], y [-.25, 0], z [-.25, 0]: touches (0, 0, 0)
    words = cr.pack(occ)
    ray = np.array([[-1, -1, -1, 1, 1, 1, 0, 2]], F32)
    z = np.linspace(0, 2, 65).astype(F32)[None]
    assert cr.point_evaluated(ss.sample_points(ray, z), words, N, 1, CUBE).any()
    assert cr.ray_live(ray, words, N, 1, CUBE).all()
    occ = np.zeros((1, M, M, M), bool)
    occ[0, 5, 4, 4] = True                                    # x [.25, .5]
    words = cr.pack(occ)
    ray = np.array([[-0.29336423, 0.1, 0.1, 1.4860435, 0, 0, 0, 0.3656449]], F32)
    last = ss.sample_points(ray, ss.z_base(ray, 64))[0, -1]
    assert last[0] == F32(0.25)
    assert cr.point_evaluated(last, words, N, 1, CUBE) and cr.ray_live(ray, words, N, 1, CUBE).all()
    # two levels: level 1 is [-2, 2]^3 in cells of 0.5; the ray runs along +x in the plane y = 1
    occ = np.zeros((2, M, M, M), bool)
    occ[1, 6, 6, 4] = True                                    # x [1, 1.5], y [1, 1.5], z [0, .5]
    words = cr.pack(occ)
    ray = np.array([[-3, 1, 0.25, 1, 0, 0, 0, 6]], F32)
    z = ss.z_base(ray, 64)
    assert cr.point_evaluated(ss.sample_points(ray, z), words, N, 2, CUBE).sum() == 5     # x = 1 is level 0's
    assert cr.ray_live(ray, words, N, 2, CUBE).all()


def _random_rays(rng, n, ranges, L, N):
    """Segments of every kind around the cascade: random, axis-parallel, on lattice planes of a random level,
    reversed directions and a few with negative or zero near."""
    lo, hi = cw.level_box(ranges, L - 1)
    c, ext = 0.5 * (lo + hi), np.abs(hi - lo)
    o = c + (rng.random((n, 3)) - 0.5) * ext * 1.4
    d = rng.standard_normal((n, 3))
    par = rng.random(n) < 0.3
    d[par, rng.integers(0, 3, n)[par]] = 0.0
    snap = rng.random(n) < 0.4
    k = rng.integers(0, L, n)
    for i in np.nonzero(snap)[0]:
        a = rng.integers(0, 3)
        o[i, a] = cw.lattice(ranges, N, k[i], np.full(3, rng.integers(0, N)))[a]
        d[i, a] = 0.0
    near = rng.random(n) * 0.5 - 0.1
    far = near + rng.random(n) * ext.max() * 1.2 + 1e-3
    return np.concatenate([o, d, near[:, None], far[:, None]], 1).astype(F32)


@pytest.mark.parametrize("L", [1, 2, 4, 8])
@pytest.mark.parametrize("M", [1, 4, 5, 7, 8, 16])
def test_random_sparse_cascades(M, L):
    rng = np.random.default_rng(100 * M + L)
    N = M + 1
    for rname, ranges in RANGES.items():
        occ = np.stack([(rng.random((M, M, M)) < (0.3 if M < 4 else 0.05)) & ~cr.inner_mask(N, k) for k in range(L)])
        words = cr.pack(occ)
        rays = _random_rays(rng, 60, ranges, L, N)
        live = cr.ray_live(rays, words, N, L, ranges)
        assert np.array_equal(live, brute_live(rays, words, N, L, ranges)), rname
        lost = lookup_hits(rays, words, N, L, ranges) & ~live
        assert not lost.any(), (rname, rays[lost][:3])


def test_guard_cases_keep_their_flags():
    occ, box, rays, want = oc.guard_cases()
    assert oc.ray_live(rays, occ, box)[0].tolist() == want.tolist()
    assert oc.brute_live(rays, occ, box).tolist() == want.tolist()
    words = cr.pack(occ[None])
    r6 = tuple(v for p in box for v in p)
    assert cr.ray_live(rays, words, 5, 1, r6).tolist() == want.tolist()


def test_a_half_cell_growth_makes_a_meeting_ray_live():
    """delta >= 1/2 cell on some axis: a float32 sample cannot resolve a cell there, and a ray that meets the grown
    box is live even with every cell empty; one that misses it stays culled."""
    occ = np.zeros((4, 4, 4), bool)
    box = ((-2.0, 2.0),) * 3
    far = F32(2.0 ** 22)
    rays = np.array([[-5, 0.5, 0.5, 1, 0, 0, 0, far], [-5, 9.5, 0.5, 1, 0, 0, 0, far],
                     [-5, 0.5, 0.5, 1, 0, 0, 0, 10]], F32)
    flag, _ = oc.ray_live(rays, occ, box)
    assert flag.tolist() == [True, False, False]
    assert oc.brute_live(rays, occ, box).tolist() == [True, False, False]
