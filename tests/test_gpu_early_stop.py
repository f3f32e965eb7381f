"""Early ray termination on the device (culling.render_samples(..., early_stop=), csrc/early_stop_kernels.cuh): the
cut word is the float64 rule of tests/early_stop_ref.py on the device's own sigma; every weight up to the end of the
cut word is the render's without termination bit for bit and later ones are 0; a ray never cut is bit-identical in
every output; the cut rays are within DESIGN.md §10f's bound; the evaluated-sample count drops by exactly the
dropped samples.  Edges (eps = 1, NaN sigma, plain rays, non-finite intervals, dead rays, a cut in the last word,
n in {0, 1, 75}, chunking and one CTA), the public entries and mesh colour fusion."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import bench
from nerf_pl_b200 import culling
from oracle import nerf_oracle as orc
from tests import cases
from tests import early_stop_ref as es
from tests import mesh_grid_ref as mg
from tests import occupancy_ref as oc
from tests import sample_skip_ref as sk

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUBE = ((-1.5, 1.5),) * 3


def _nb():
    import nerf_pl_b200 as nb
    return nb


def _emb():
    return [_nb().Embedding(3, 10), _nb().Embedding(3, 4)]


_M = {}


def _models(kind="random"):
    """[coarse, fine] of seeded random weights or of the trained test weights; "nan": random with a NaN sigma head."""
    if kind not in _M:
        ws = cases.trained_weights() if kind == "trained" else [orc.make_weights(21), orc.make_weights(22)]
        ms = []
        for w in ws:
            w = dict(w)
            if kind == "nan":
                w["sigma.bias"] = np.full_like(w["sigma.bias"], np.nan)
            m = _nb().NeRF()
            m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
            ms.append(m.cuda().eval())
        _M[kind] = ms
    return _M[kind]


_G = {}


def _grid(kind):
    if kind not in _G:
        if kind == "trained":       # the tests' grid: N = 128 over the box, sigma > 1, dilate 1
            _G[kind] = _nb().occupancy_grid(_models("trained")[1], 128, *CUBE, 1.0, 1)
        else:
            words = mg.random_words(17, 0.3, 4)
            _G[kind] = _nb().OccupancyGrid(torch.from_numpy(words.view(np.int32)).cuda(), 17, *CUBE)
    return _G[kind]


def _rays(kind, n=600, seed=7):
    if kind == "trained":
        return torch.from_numpy(bench.blender_rays(0, 80 + seed % 3, W=64, H=64, pixels="all")).cuda()
    return torch.from_numpy(bench.blender_rays(n, seed)).cuda()


def _render(models, rays, grid, S, use_disp, white_back, test_time, eps=0.0, **kw):
    return culling.render_samples(models, rays, grid, S, use_disp, 0, white_back, test_time, extras=True,
                                  per_sample=True, early_stop=eps, **kw)


def _i32(t):
    return t.detach().cpu().numpy().view(np.int32)


def _check(models, rays, grid, S, use_disp, white_back, test_time, eps, **kw):
    """Every property of one render with termination against the same render without; returns the cut words."""
    ref = _render(models, rays, grid, S, use_disp, white_back, test_time, **kw)
    got = _render(models, rays, grid, S, use_disp, white_back, test_time, eps, **kw)
    keys = culling.result_keys(0, test_time)
    n = rays.shape[0]
    cut = got["cut_coarse"].cpu().numpy().astype(np.int64)
    assert cut.shape == (n,)
    if n == 0:
        assert got["live_samples"] == (0, 0)
        return cut
    rn = rays.cpu().numpy()
    z = sk.z_base(rn, S, use_disp)
    sigma = ref["samples_coarse"][..., 3].cpu().numpy()
    ev = sk.mask_bits(ref["mask_coarse"].cpu().numpy(), S)
    T = es.word_transmittance(rn, z, sigma)
    if S == 32:                 # one word: nothing to drop, the path without termination
        want = np.full(n, -1)
    else:
        want, _ = es.cut_words(rn, z, sigma, eps)
    with np.errstate(invalid="ignore", divide="ignore"):
        tie = (np.abs(T / eps - 1.0) < 1e-9).any(1)
    assert np.all((cut == want) | tie), np.nonzero((cut != want) & ~tie)[0][:10]
    assert not tie.all() and (cut < S // 32).all() and (cut >= -1).all()
    word = np.arange(S) // 32
    keep = (cut[:, None] < 0) | (word[None, :] <= cut[:, None])
    # weights, samples and masks: the render's up to the end of the cut word, nothing after it
    for k in ("weights_coarse", "samples_coarse"):
        a, b = _i32(got[k]), _i32(ref[k])
        assert np.array_equal(a[keep], b[keep]), k
        assert not a[~keep].any(), k
    assert np.array_equal(sk.mask_bits(got["mask_coarse"].cpu().numpy(), S), ev & keep)
    assert got["live_samples"] == (ref["live_samples"][0] - int(es.dropped(ev, cut).sum()), 0)
    # a ray never cut, or cut in its last word, is the render's in every output
    same = (cut < 0) | (cut == S // 32 - 1)
    for k in keys:
        assert np.array_equal(_i32(got[k])[same], _i32(ref[k])[same]), k
    # the cut rays: within T_cut (1 + S 1e-10) + 4e-6, depth times the ray's largest z
    cr = np.nonzero(cut >= 0)[0]
    bound = T[cr, cut[cr]] * (1 + S * 1e-10) + 4e-6
    d = {k: np.abs(got[k].cpu().numpy().astype(np.float64) - ref[k].cpu().numpy())[cr] for k in keys}
    assert np.all(d["opacity_coarse"] <= bound)
    if not test_time:
        assert np.all(d["rgb_coarse"] <= bound[:, None])
        assert np.all(d["depth_coarse"] <= bound * z[cr].max(1))
    return cut


COMBOS = [(True, False, True), (False, True, False), (False, False, True)]     # (test_time, use_disp, white_back)


@pytest.mark.parametrize("S", [32, 64, 128])
@pytest.mark.parametrize("test_time,use_disp,white_back", COMBOS)
def test_random_weights(S, test_time, use_disp, white_back):
    for eps in (0.5, 1.0):
        cut = _check(_models(), _rays("random"), _grid("random"), S, use_disp, white_back, test_time, eps)
        if S > 32 and eps == 1.0:
            assert (cut >= 0).any()


@pytest.mark.parametrize("S", [32, 64, 128])
@pytest.mark.parametrize("test_time,use_disp,white_back", COMBOS)
def test_trained_scene(S, test_time, use_disp, white_back):
    if not cases.have_trained():
        pytest.skip("no trained weights")
    for i, eps in enumerate((1e-4, 1e-3, 1e-2)):
        cut = _check(_models("trained"), _rays("trained", seed=i), _grid("trained"), S, use_disp, white_back,
                     test_time, eps)
        if S > 32:
            assert (cut >= 0).mean() > 0.02


@pytest.mark.parametrize("S", [32, 64, 128])
def test_zero_is_the_skipped_render_bit_for_bit(S):
    nb = _nb()
    lib = nb._lib.load()
    rays, grid = _rays("random", 500, 3), _grid("random")
    for test_time, use_disp, white_back in COMBOS:
        a = culling.render_samples(_models(), rays, grid, S, use_disp, 0, white_back, test_time, extras=True)
        before = lib.nerfb200_launch_count()
        b = culling.render_samples(_models(), rays, grid, S, use_disp, 0, white_back, test_time, extras=True,
                                   early_stop=0.0)
        launches = lib.nerfb200_launch_count() - before
        before = lib.nerfb200_launch_count()
        culling.render_samples(_models(), rays, grid, S, use_disp, 0, white_back, test_time, extras=True)
        assert launches == lib.nerfb200_launch_count() - before        # not one new launch
        assert a.keys() == b.keys() and a["live_samples"] == b["live_samples"]
        for k, v in a.items():
            if k != "live_samples":
                assert np.array_equal(_i32(v), _i32(b[k])), k


def test_nan_sigma_is_never_cut():
    cut = _check(_models("nan"), _rays("random"), _grid("random"), 128, False, True, False, 1.0)
    assert (cut == -1).all()


def _bad_rays():
    rays = bench.blender_rays(64, 10)
    bad = rays[:10].copy()
    bad[0, 0] = np.nan
    bad[1, 4] = np.inf
    bad[2, 7] = np.inf
    bad[3, 6] = np.nan
    bad[4, 6], bad[4, 7] = 6.0, 2.0                   # far <= near
    bad[5, 6] = bad[5, 7] = 4.0
    bad[6, 3:6] = 3e19                                # |d|^2 overflows
    bad[7, 3:6] = np.array([1e30, 0, 0], np.float32)  # 1e10 |d| overflows: the intervals are not finite
    bad[8, 5] = -np.inf
    bad[9, 1] = np.inf
    return torch.from_numpy(np.concatenate([rays, bad])).cuda()


@pytest.mark.parametrize("S", [64, 128])
def test_plain_rays_and_non_finite_intervals_are_never_cut(S):
    rays = _bad_rays()
    full = _nb().OccupancyGrid(torch.tensor([1], dtype=torch.int32).cuda(), 2, *(((-1e4, 1e4),) * 3))
    for grid in (_grid("random"), full):
        for test_time in (True, False):
            cut = _check(_models(), rays, grid, S, False, True, test_time, 1.0)
            assert (cut[64:] == -1).all() and (cut[:64] >= 0).any()


def test_dead_rays_and_culled_rays():
    nb = _nb()
    rays, grid = _rays("random", 400, 9), _grid("random")
    flag = torch.zeros(400, dtype=torch.uint8, device="cuda")
    flag[::3] = 1
    cut = _check(_models(), rays, grid, 128, False, True, False, 1.0, live_flag=flag)
    assert (cut[flag.cpu().numpy() == 0] == -1).all()
    # render_rays_culled: a culled ray still gets the vacuum value
    sparse = nb.OccupancyGrid(torch.from_numpy(mg.random_words(17, 0.02, 6).view(np.int32)).cuda(), 17, *CUBE)
    for test_time in (True, False):
        out = nb.render_rays_culled(_models()[:1], _emb(), rays, sparse, 128, False, 0, True, test_time,
                                    skip="samples", early_stop=0.5, extras=True)
        want = nb.render_rays_culled(_models()[:1], _emb(), rays, sparse, 128, False, 0, True, test_time,
                                     skip="samples", extras=True)
        dead = torch.ones(400, dtype=torch.bool, device="cuda")
        dead[out["live_idx"]] = False
        assert 0 < int(dead.sum()) < 400 and out["live"] == want["live"]
        keys = culling.result_keys(0, test_time)
        vac = oc.vacuum_results(int(dead.sum()), keys, True)
        for k in keys:
            assert np.array_equal(out[k][dead].cpu().numpy(), vac[k]), k
        assert out["live_samples"][0] <= want["live_samples"][0]
        compact = nb.render_rays_culled(_models()[:1], _emb(), rays, sparse, 128, False, 0, True, test_time,
                                        skip="samples", early_stop=0.5)
        for k in keys:
            assert np.array_equal(_i32(compact[k]), _i32(out[k])), k
        assert compact["live_samples"] == out["live_samples"]


def test_cut_in_the_last_word():
    """Rays along +x through a box occupied only at their far end: every evaluated sample is in the last word, so
    with eps = 1 a ray is cut there or never, and nothing is dropped."""
    n = 256
    rng = np.random.default_rng(3)
    rays = np.zeros((n, 8), np.float32)
    rays[:, 0] = -3.0
    rays[:, 1:3] = rng.uniform(-1.2, 1.2, (n, 2))
    rays[:, 3] = 1.0
    rays[:, 7] = 4.0
    box = ((0.2, 1.5), (-1.5, 1.5), (-1.5, 1.5))
    grid = _nb().OccupancyGrid(torch.tensor([1], dtype=torch.int32).cuda(), 2, *box)
    for S in (64, 128):
        cut = _check(_models(), torch.from_numpy(rays).cuda(), grid, S, False, True, False, 1.0)
        assert set(np.unique(cut)) <= {-1, S // 32 - 1} and (cut == S // 32 - 1).any()


@pytest.mark.parametrize("n", [0, 1, 75])
def test_small_batches(n):
    rays = _rays("random", 600, 11)[:n].contiguous()
    for S in (64, 128):
        _check(_models(), rays, _grid("random"), S, False, True, False, 1.0)
        _check(_models(), rays, _grid("random"), S, False, False, True, 0.5)


_SUBPROCESS = r"""
import sys
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
import nerf_pl_b200 as nb
from nerf_pl_b200 import culling
from oracle import nerf_oracle as orc
ms = []
for s in (21, 22):
    m = nb.NeRF()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in orc.make_weights(s).items()})
    ms.append(m.cuda().eval())
words = np.load(sys.argv[2])
grid = nb.OccupancyGrid(torch.from_numpy(words.view(np.int32)).cuda(), 17, *(((-1.5, 1.5),) * 3))
rays = torch.from_numpy(np.load(sys.argv[3])).cuda()
r = culling.render_samples(ms, rays, grid, 128, False, 0, True, False, extras=True, per_sample=True, early_stop=0.5)
np.savez(sys.argv[4], live=np.array(r.pop("live_samples")), **{k: v.cpu().numpy() for k, v in r.items()})
"""


def test_independent_of_chunk_and_cta_count(monkeypatch, tmp_path):
    rays, grid = _rays("random", 900, 12), _grid("random")
    base = _render(_models(), rays, grid, 128, False, True, False, 0.5)
    assert (base["cut_coarse"] >= 0).any()
    np.save(tmp_path / "w.npy", mg.random_words(17, 0.3, 4))
    np.save(tmp_path / "r.npy", rays.cpu().numpy())
    env = dict(os.environ, NERFB200_MAX_CTAS="1")
    subprocess.run([sys.executable, "-c", _SUBPROCESS, ROOT, str(tmp_path / "w.npy"), str(tmp_path / "r.npy"),
                    str(tmp_path / "o.npz")], check=True, env=env, cwd=ROOT)
    one = np.load(tmp_path / "o.npz")
    monkeypatch.setattr(culling, "_SAMPLE_CHUNK", 257)
    chunked = _render(_models(), rays, grid, 128, False, True, False, 0.5)
    assert chunked["live_samples"] == base["live_samples"] == tuple(one["live"])
    for k, v in base.items():
        if k == "live_samples":
            continue
        a, b, c = _i32(chunked[k]), one[k].view(np.int32), _i32(v)
        if k == "mask_coarse":          # the words of a 128-sample pass; the last two are not written
            a, b, c = a[:, :4], b[:, :4], c[:, :4]
        assert np.array_equal(a, c) and np.array_equal(b, c), k


def test_public_entries_pass_it_through():
    nb = _nb()
    kind = "trained" if cases.have_trained() else "random"
    models, grid = _models(kind), _grid(kind)
    rays = torch.from_numpy(bench.blender_rays(0, 70, W=48, H=48, pixels="all")).cuda()
    for eps in (0.0, 1e-3):
        a = nb.batched_inference(models[:1], _emb(), rays, 128, 0, False, white_back=True, occupancy=grid,
                                 skip="samples", early_stop=eps)
        b = nb.render_rays_culled(models[:1], _emb(), rays, grid, 128, False, 0, True, True, skip="samples",
                                  early_stop=eps)
        assert torch.equal(a["opacity_coarse"], b["opacity_coarse"]) and a["live_samples"] == b["live_samples"]
        img = nb.render_image(models[:1], _emb(), 48, 48, float(bench.IMG_W), np.eye(3, 4), 2.0, 6.0, 128, 0,
                              white_back=True, occupancy=grid, skip="samples", early_stop=eps)
        c = nb.batched_inference(models[:1], _emb(), img["rays"], 128, 0, False, white_back=True, occupancy=grid,
                                 skip="samples", early_stop=eps)
        assert torch.equal(img["opacity"].reshape(-1), c["opacity_coarse"]) and img["live_samples"] == c["live_samples"]
        if eps == 0.0:
            full = a["live_samples"]
    assert a["live_samples"][0] < full[0]


def _look_at(eye):
    eye = np.asarray(eye, np.float64)
    f = -eye / np.linalg.norm(eye)
    r = np.cross(f, [0, 0, 1.0])
    r /= np.linalg.norm(r)
    return np.stack([r, np.cross(r, f), -f, eye], 1)


def test_fused_vertex_colours():
    """eps <= 1 - occ_threshold - 1e-5: the colours of early_stop = 0 bit for bit, the opacities within the bound."""
    if not cases.have_trained():
        pytest.skip("no trained weights")
    nb = _nb()
    fine, grid = _models("trained")[1], _grid("trained")
    v, _ = nb.extract_mesh(fine, 64, *CUBE, 20.0)
    poses = [_look_at(e) for e in ([3.5, 0.4, 0.8], [-1.2, 3.1, -0.6], [0.3, -2.6, 2.4], [0.2, 0.3, -3.9])]
    H, W = 60, 80
    yy, xx = np.mgrid[0:H, 0:W]
    images = torch.from_numpy(np.stack([np.stack([(xx * 3 + k * 40) % 256, (yy * 4 + k * 17) % 256,
                                                  (xx + yy + 60 * k) % 256], -1)
                                        for k in range(len(poses))]).astype(np.uint8)).cuda()
    c0, o0 = nb.fuse_vertex_colors(fine, v, images, poses, 70.0, 1.0, return_opacities=True, occupancy=grid)
    for eps in (1e-3, 0.5):
        c1, o1 = nb.fuse_vertex_colors(fine, v, images, poses, 70.0, 1.0, return_opacities=True, occupancy=grid,
                                       early_stop=eps)
        assert torch.equal(c0, c1), eps
        moved = (o1 != o0)
        assert eps < 0.5 or moved.any()
        assert float((o1.double() - o0.double()).abs().max()) <= eps * (1 + 64 * 1e-10) + 4e-6
        # what moved is a cut ray: opaque either way
        assert bool((o1[moved] > 1 - eps - 4e-6).all() and (o0[moved] > 1 - eps - 4e-6).all())
