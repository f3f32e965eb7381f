"""The cell walk on the device (cull_rays, render_rays_culled) at the lattice, box and cascade-level boundaries where
it used to drop rays with an evaluated sample (pytest -m gpu; DESIGN.md §10 "Live", §10h).

One occupied cell at a time, at the corner of each level's box and beside the box of the level below, with the
designed rays of tests/cull_walk_cases.py: (a) zero-direction probes at lattice corners, edge midpoints and face
centres, one ulp either way; (b) axis-parallel rays in lattice planes and on lattice lines; (c), (d) rays through
corners, edges and faces in all 26 directions, whole, starting there and ending there; (e) rays whose last float32
sample rounds onto a face the exact segment stops short of; and rays that miss the cell by 1e-3 of a cell.

- The flags equal the float64 restatement (tests/occupancy_ref.ray_live through cascade_ref) exactly.
- (a): the per-sample masks equal cascade_ref.point_evaluated, and a probe is live iff it touches an occupied cell.
- Every ray with an evaluated coarse or fine sample (K in {0, 64, 128}) is live, and the near misses are culled.
- render_rays_culled(skip="samples") equals culling.render_samples over all rays bit for bit in every key, with the
  same live_samples: culling is a pure optimisation.
Also: masked grids through a mixed cascade whose lattice lies on the level faces."""
import itertools

import numpy as np
import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import culling
from oracle import nerf_oracle as orc
from tests import cascade_ref as cr
from tests import cull_walk_cases as cw
from tests import occupancy_ref as oc
from tests import sample_skip_ref as ss

pytestmark = pytest.mark.gpu
F32 = np.float32
CUBE = (-1.0, 1.0, -1.0, 1.0, -1.0, 1.0)
REVERSED = (1.0, -1.0, -0.5, 1.5, 3.0, 2.0)
UNEQUAL = (-1.0, 1.0, 1.25, -0.75, -0.5, 0.5)
S = 64

_MODELS = []


def _models():
    if not _MODELS:
        for s in (31, 32):
            m = nb.NeRF()
            m.load_state_dict({k: torch.from_numpy(v) for k, v in orc.make_weights(s).items()})
            _MODELS.append(m.cuda().eval())
    return _MODELS


def _emb():
    return [nb.Embedding(3, 10), nb.Embedding(3, 4)]


def _grid(words, N, L, ranges):
    bits = torch.from_numpy(np.ascontiguousarray(np.asarray(words, np.uint32)).view(np.int32)).cuda()
    return nb.OccupancyGrid(bits, N, *cr.pairs(ranges), levels=L)


def _eq(a, b, tag):
    for k in culling.result_keys(0, False) + ["rgb_fine", "depth_fine", "opacity_fine"]:
        if k in a or k in b:
            assert k in a and k in b, (tag, k)
            assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), (tag, k)
    assert tuple(a["live_samples"]) == tuple(b["live_samples"]), (tag, a["live_samples"], b["live_samples"])


def _check(rays_np, words, N, L, ranges, fam, tag, full=False, exact=True):
    """Every check of the module docstring on one batch; fam (n,) names each ray's family.  ``exact``: the flags
    equal the restatement's on every ray (designed inputs), else away from a rounding margin of 1e-9 cells."""
    rays = torch.from_numpy(np.ascontiguousarray(rays_np, F32)).cuda()
    g = _grid(words, N, L, ranges)
    models = _models()
    flag = nb.cull_rays(rays, g, return_flag=True)[2].cpu().numpy().astype(bool)
    want = cr.ray_live(rays_np, words, N, L, ranges)
    diff = flag != want
    if not exact:
        occ = cr.unpack(words, N, L)
        margin = np.min([oc.ray_live(rays_np, occ[k], cr.pairs(cr.level_ranges(ranges, k)))[1] for k in range(L)], 0)
        diff &= margin > 1e-9
    bad = np.nonzero(diff)[0]
    assert len(bad) == 0, (tag, bad[:5], fam[bad[:5]], rays_np[bad[:5]])
    assert not flag[fam == "misses"].any(), tag
    probe = fam == "probes"
    # (a) every sample of a probe sits at o: the masks are point_occupied of o
    res = culling.render_samples(models, rays[torch.from_numpy(probe).cuda()], g, 32, False, 0, False, False,
                                 per_sample=True)
    m = ss.mask_bits(res["mask_coarse"].cpu().numpy(), 32)
    pe = cr.point_evaluated(rays_np[probe, :3], words, N, L, ranges)
    assert np.array_equal(m, np.repeat(pe[:, None], 32, 1)), tag
    assert np.array_equal(flag[probe], cw.touches_any_level(rays_np[probe, :3], words, N, L, ranges)), tag
    assert not (pe & ~flag[probe]).any(), tag
    # every ray with an evaluated sample is live
    for K in (0, 64, 128):
        res = culling.render_samples(models, rays, g, S, False, K, False, False, per_sample=True, extras=K > 0)
        ev = ss.mask_bits(res["mask_coarse"].cpu().numpy(), S).any(1)
        if K:
            ev |= ss.mask_bits(res["mask_fine"].cpu().numpy(), S + K).any(1)
            assert np.array_equal(ss.mask_bits(res["mask_fine"].cpu().numpy(), S + K),
                                  cr.evaluated(rays_np, res["z_vals_fine"].cpu().numpy(), words, N, L, ranges)), tag
        lost = np.nonzero(ev & ~flag)[0]
        assert len(lost) == 0, (tag, K, lost[:5], fam[lost[:5]], rays_np[lost[:5]])
    # culling under skip="samples" changes no pixel
    combos = itertools.product((0, 64, 128), (False, True), (False, True)) if full else \
        [(0, False, True), (64, True, False), (128, False, False)]
    for K, tt, wb in combos:
        a = nb.render_rays_culled(models, _emb(), rays, g, S, False, K, wb, tt, skip="samples")
        b = culling.render_samples(models, rays, g, S, False, K, wb, tt)
        _eq(a, b, (tag, K, tt, wb))
    for wb in (False, True):
        a = nb.render_rays_culled(models[:1], _emb(), rays, g, S, False, 0, wb, False, skip="samples", early_stop=1e-3)
        b = culling.render_samples(models[:1], rays, g, S, False, 0, wb, False, early_stop=1e-3)
        _eq(a, b, (tag, "early stop", wb))
    return flag


@pytest.mark.parametrize("N, L, rname", [(9, 1, "cube"), (9, 2, "cube"), (8, 3, "reversed"), (9, 8, "unequal"),
                                         (6, 2, "unequal")])
def test_designed_families(N, L, rname):
    ranges = {"cube": CUBE, "reversed": REVERSED, "unequal": UNEQUAL}[rname]
    live = {f: 0 for f in cw.FAMILIES}
    for j, (k, cell) in enumerate(cw.target_cells(N, L)):
        words = cw.one_cell_words(N, L, k, cell)
        parts = [(f, cw.family(f, ranges, N, L, k, cell, seed=N + k)) for f in cw.FAMILIES]
        rays = np.concatenate([r for _, r in parts])
        fam = np.concatenate([np.full(len(r), f) for f, r in parts])
        flag = _check(rays, words, N, L, ranges, fam, (N, L, rname, k, cell), full=(j < 2))
        for f in cw.FAMILIES:
            live[f] += int(flag[fam == f].sum())
    assert live["probes"] > 0 and live["axis"] > 0 and live["points"] > 0 and live["rounding"] > 0
    print(f"\nN {N} L {L} {rname}: live rays per family {live}")


def test_random_cascades_through_lattice_planes():
    """Random sparse cascades and rays snapped to lattice planes of random levels: the same checks."""
    rng = np.random.default_rng(5)
    for N, L, ranges in ((9, 3, CUBE), (8, 4, REVERSED), (17, 2, UNEQUAL)):
        M = N - 1
        words = cr.pack(np.stack([(rng.random((M, M, M)) < 0.05) & ~cr.inner_mask(N, k) for k in range(L)]))
        lo, hi = cw.level_box(ranges, L - 1)
        n = 4096
        o = 0.5 * (lo + hi) + (rng.random((n, 3)) - 0.5) * np.abs(hi - lo) * 1.4
        d = rng.standard_normal((n, 3))
        for i in range(n):
            if rng.random() < 0.6:
                a = rng.integers(0, 3)
                o[i, a] = cw.lattice(ranges, N, rng.integers(0, L), np.full(3, rng.integers(0, N)))[a]
                d[i, a] = 0.0
        near = rng.random(n) * 0.5
        far = near + rng.random(n) * np.abs(hi - lo).max() * 1.2 + 1e-3
        rays = np.concatenate([o, d, near[:, None], far[:, None]], 1).astype(F32)
        _check(rays, words, N, L, ranges, np.full(n, "random"), (N, L), exact=False)


@pytest.mark.parametrize("ch", [1, 4])
def test_masked_grids_through_a_mixed_cascade_on_the_level_faces(ch):
    """sigma_grid / rgb_sigma_grid(occupancy=cascade) on [-4, 4]^3 at N = 17 over a 3-level cascade on [-1, 1]^3 with
    M = 8: the lattice lies on every level's faces.  The evaluated set equals cascade_ref.point_evaluated of the
    lattice positions, and the evaluated values equal the unmasked grid's bit for bit."""
    rng = np.random.default_rng(17 + ch)
    N, L, M = 9, 3, 8
    words = cr.pack(np.stack([(rng.random((M, M, M)) < 0.2) & ~cr.inner_mask(N, k) for k in range(L)]))
    g = _grid(words, N, L, CUBE)
    model = _models()[1]
    rng_ = ((-4.0, 4.0),) * 3
    fn = nb.sigma_grid if ch == 1 else nb.rgb_sigma_grid
    out, n_ev = fn(model, 17, *rng_, occupancy=g, return_evaluated=True)
    full = fn(model, 17, *rng_)
    x = np.linspace(-4.0, 4.0, 17)
    Y, X, Z = np.meshgrid(x, x, x, indexing="ij")                 # out[i, j, k] is (x_j, y_i, z_k)
    want = cr.point_evaluated(np.stack([X, Y, Z], -1).astype(F32), words, N, L, CUBE)
    assert n_ev == int(want.sum()) and 0 < n_ev < 17 ** 3
    o, f = out.cpu().numpy(), full.cpu().numpy()
    if ch == 4:
        assert np.array_equal((o[..., :3] != 0).any(-1), want)    # sigmoid rgb is never 0 where evaluated
        w = want[..., None]
    else:
        w = want
    assert np.array_equal(np.where(w, f, F32(0)).view(np.uint32), o.view(np.uint32))
