"""View-dependent baked volumes (nb.query_rgb_sh, nb.bake_volume(..., view_dependent=True), nb.render_baked;
DESIGN.md §10k).

- query_rgb_sh meets the float64 fit of tests/baked_sh_ref.py, random and trained weights; its sigma is
  query_rgb_sigma's bit for bit; with the direction weights zeroed every coefficient but c0 vanishes;
- the bake's sigma, bricks and map are the direction-0 bake's bit for bit, and its points are query_rgb_sh's;
- a bake and its dense twin render the same bits; the render meets the float64 restatement;
- rays are isolated, a graph replay equals the eager call, early stop keeps uncut rays bit for bit;
- on the trained scene the SH render is close to the MLP render."""
import numpy as np
import pytest
import torch

import bench
from tests import baked_sh_ref as sr
from tests import cases
from tests import test_gpu_baked as tb

pytestmark = pytest.mark.gpu
CUBE = tb.CUBE
UNEQUAL = tb.UNEQUAL


def _nb():
    import nerf_pl_b200 as nb
    return nb


def _u32(a):
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.uint32)


def _weights(kind):
    from oracle import nerf_oracle as orc
    return cases.trained_weights()[1] if kind == "trained" else orc.make_weights(21)


def _model_of(w):
    m = _nb().NeRF()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
    return m.cuda().eval()


# ---- the query ------------------------------------------------------------------------------------------------------
# The bar.  A coefficient is sum_j P[m, j] f_j, so its error is at most ||P|| = max_m sum_j |P[m, j]| (3.545,
# tests/test_baked_sh_ref.py) times the worst per-direction colour error, plus the float32 accumulation (below 2e-5).
# The per-direction colour error is that of the rgb head on the fp16 trunk: the north-star rgb bar, 1e-3 abs
# (tests/test_gpu_parity.py), or, where the fp16 trunk itself exceeds it at these points, twice the error of
# query_rgb_sigma's colour (the same trunk and head at the direction 0) against the same float64 forward.  Twice,
# because each direction moves the head's operating point; query_rgb_sigma's error is measured in the same test.
P_NORM = 3.545


def _query_bar(w, xyz, rgb0):
    f0, _ = sr.direction_colours(w, xyz, np.zeros((1, 3), np.float32))
    e0 = float(np.abs(rgb0 - f0[:, 0]).max())
    return P_NORM * max(1e-3, 2 * e0) + 2e-5, e0


@pytest.mark.parametrize("kind", ["random", "trained"])
def test_query_rgb_sh_against_float64(kind):
    if kind == "trained" and not cases.have_trained():
        pytest.skip("no trained weights")
    nb = _nb()
    w = _weights(kind)
    model = _model_of(w)
    xyz = np.random.default_rng(3).uniform(-1.5, 1.5, (3000, 3)).astype(np.float32)
    got = nb.query_rgb_sh(model, torch.from_numpy(xyz).cuda()).cpu().numpy().astype(np.float64)
    assert got.shape == (3000, 28)
    want = sr.query(w, xyz, sr.projection().astype(np.float32))
    rs = nb.query_rgb_sigma(model, torch.from_numpy(xyz).cuda()).cpu().numpy()
    bar, e0 = _query_bar(w, xyz, rs[:, :3].astype(np.float64))
    coef = np.delete(np.arange(28), 3)
    err = np.abs(got[:, coef] - want[:, coef]).max()
    print(f"\nquery_rgb_sh {kind}: worst coefficient error {err:.3e} (bar {bar:.3e}; query_rgb_sigma's colour error "
          f"{e0:.3e})")
    assert err <= bar
    # sigma is the rgb + sigma query's, bit for bit
    assert np.array_equal(_u32(got[:, 3]), _u32(rs[:, 3]))


def test_direction_free_weights():
    nb = _nb()
    w = {k: v.copy() for k, v in _weights("random").items()}
    w["dir_encoding.0.weight"][:, 256:] = 0
    model = _model_of(w)
    xyz = torch.from_numpy(np.random.default_rng(4).uniform(-1.5, 1.5, (5000, 3)).astype(np.float32)).cuda()
    got = nb.query_rgb_sh(model, xyz).double().cpu().numpy()
    f = nb.query_rgb_sigma(model, xyz).double().cpu().numpy()[:, :3]       # the colour of every direction
    P = sr.projection().astype(np.float32).astype(np.float64)
    # float32 accumulation of 64 terms: |fl(sum) - sum| <= 64 u sum_j |P[m, j] f|, u = 2^-24; plus the rounding of P
    coef, _ = sr.unpack_points(got)
    bound = 64 * 2.0 ** -24 * np.abs(P).sum(1)[None, :, None] * np.abs(f)[:, None, :] + 1e-12
    exact = P.sum(1)[None, :, None] * f[:, None, :]
    assert (np.abs(coef - exact) <= bound).all()
    assert np.abs(coef[:, 1:]).max() < 1e-5
    assert np.abs(coef[:, 0] * sr.C0 - f).max() < 1e-5


# ---- the bake ---------------------------------------------------------------------------------------------------------
def _check_bake(model, N, grid, full_points):
    nb = _nb()
    vd = nb.bake_volume(model, N, *CUBE, occupancy=grid, view_dependent=True)
    plain = nb.bake_volume(model, N, *CUBE, occupancy=grid)
    assert vd.view_dependent and not plain.view_dependent
    assert vd.bricks == plain.bricks
    nbk = (-(-N // 8)) ** 3
    assert vd.nbytes == 81648 * vd.bricks + 4 * nbk
    assert torch.equal(vd.data[-4 * nbk:], plain.data[-4 * nbk:])                     # the map
    d7, d1 = vd.to_dense(), plain.to_dense()
    assert d7.shape == (N, N, N, 28)
    assert torch.equal(d7[..., 3].contiguous().view(torch.int32), d1[..., 3].contiguous().view(torch.int32))
    off = (d1 == 0).all(-1)                                    # not evaluated (sigmoid rgb is never 0 where evaluated)
    assert bool((d7[off] == 0).all())
    if full_points:
        pts = nb.query_rgb_sh(model, nb.mesh.grid_positions(N, *CUBE)).reshape(N, N, N, 28)
        on = ~off
        assert torch.equal(d7[on].view(torch.int32), pts[on].view(torch.int32))
    st = nb.BakedVolume.from_state_dict(vd.state_dict())
    assert st.view_dependent and st.bricks == vd.bricks and torch.equal(st.data, vd.data)
    assert "view_dependent" not in plain.state_dict()
    return vd


@pytest.mark.parametrize("N", [9, 17, 64])
@pytest.mark.parametrize("gi", range(4))
def test_bake_against_the_plain_bake(N, gi):
    _, words, occ_N, box, levels = tb._grids()[gi]
    _check_bake(tb._model(), N, tb._grid(words, occ_N, box, levels), True)


def test_bake_against_the_plain_bake_trained_512():
    if not cases.have_trained():
        pytest.skip("no trained weights")
    nb = _nb()
    fine = tb._model("trained")
    grid = nb.occupancy_grid(fine, 128, *CUBE, 1.0, dilate=1)
    vd = _check_bake(fine, 512, grid, False)
    with pytest.raises(ValueError):
        nb.pack_volume(vd.to_dense()[:64, :64, :64].contiguous(), CUBE[0])


@pytest.mark.parametrize("gi", range(4))
def test_bake_and_its_dense_twin_render_the_same_bits(gi):
    nb = _nb()
    _, words, occ_N, box, levels = tb._grids()[gi]
    vol = nb.bake_volume(tb._model(), 33, *CUBE, occupancy=tb._grid(words, occ_N, box, levels), view_dependent=True)
    twin = nb.BakedVolume.from_grid(vol.to_dense(), *CUBE)
    assert twin.view_dependent and twin.bricks <= vol.bricks
    rays = tb._rays(3000, 7 + gi)
    s = nb.baked.default_step(vol)
    for kw in (dict(), dict(white_back=True), dict(step=s / 7), dict(step=2.5 * s), dict(early_stop=1e-2)):
        tb._same(nb.render_baked(vol, rays, **kw), nb.render_baked(twin, rays, **kw), (gi, kw))


# ---- against float64 --------------------------------------------------------------------------------------------------
def _field(N, seed):
    """Random coefficients (c0 giving a colour in [0, 1], the others in [-0.3, 0.3], so that colours leave [0, 1] and
    the clamp acts) and tests/test_gpu_baked._field's sigma."""
    rng = np.random.default_rng(seed)
    coef = rng.uniform(-0.3, 0.3, (N ** 3, 9, 3))
    coef[:, 0] = rng.uniform(0, 1, (N ** 3, 3)) / sr.C0
    sig = tb._field(N, seed)[..., 3].reshape(-1)
    return sr.pack_points(coef, sig).reshape(N, N, N, 28).astype(np.float32)


# Bars on |err| (rgb and opacity absolute, depth over max(t_max, 1)): the direction-0 render's 5e-6, and for rgb
# 2e-5, since a colour is a sum of nine float32 products of up to 3.5 in size before the clamp.
BARS = {"rgb": 2e-5, "opacity": 5e-6, "depth": 5e-6}


@pytest.mark.parametrize("N,ranges,scale,step_mul,wb", [
    (9, CUBE, 1.0, 1.0, False), (17, UNEQUAL, 1.0, 1.0, True), (33, CUBE, 2.5, 1.0, False),
    (33, tb.INSIDE, 0.4, 0.3, True)])
def test_render_against_float64(N, ranges, scale, step_mul, wb):
    nb = _nb()
    g = _field(N, N)
    vol = nb.BakedVolume.from_grid(torch.from_numpy(g).cuda(), *ranges)
    rays = tb._rays(1500, N + 1, box=[(min(r), max(r)) for r in ranges], scale=scale)
    step = nb.baked.default_step(vol) * step_mul
    got = nb.render_baked(vol, rays, step=step, white_back=wb)
    want = sr.render(g, vol.ranges, rays.cpu().numpy(), step=step, white_back=wb)
    tmax = np.maximum(np.abs(want["t_max"]), 1.0)
    err = {"rgb": np.abs(got["rgb"].cpu().numpy() - want["rgb"]).max(),
           "opacity": np.abs(got["opacity"].cpu().numpy() - want["opacity"]).max(),
           "depth": (np.abs(got["depth"].cpu().numpy() - want["depth"]) / tmax).max()}
    print(f"\nSH baked vs float64 N={N} scale={scale} step x{step_mul} wb={wb}: " +
          ", ".join(f"{k} {v:.2e} (bar {BARS[k]:.0e})" for k, v in err.items()))
    for k, v in err.items():
        assert v <= BARS[k], (k, v)
    assert want["opacity"].max() > 0.5


# ---- isolation, graphs, early stop ----------------------------------------------------------------------------------
def _volume():
    return _nb().BakedVolume.from_grid(torch.from_numpy(_field(33, 3)).cuda(), *UNEQUAL)


def test_rays_are_isolated():
    nb = _nb()
    vol = _volume()
    rays = tb._rays(2000, 11, box=UNEQUAL)
    full = nb.render_baked(vol, rays, white_back=True, early_stop=1e-3)
    perm = torch.randperm(rays.shape[0], generator=torch.Generator().manual_seed(0)).cuda()
    tb._same({k: v[perm] for k, v in full.items()}, nb.render_baked(vol, rays[perm], white_back=True, early_stop=1e-3),
             "permuted")
    for r in (0, 777, rays.shape[0] - 6):
        one = nb.render_baked(vol, rays[r:r + 1], white_back=True, early_stop=1e-3)
        tb._same({k: v[r:r + 1] for k, v in full.items()}, one, r)


def test_graph_replay_equals_eager():
    nb = _nb()
    vol = _volume()
    a, b = tb._rays(4096, 21, box=UNEQUAL)[:4096], tb._rays(4096, 22, box=UNEQUAL)[:4096]
    static = a.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        nb.render_baked(vol, static, white_back=True)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = nb.render_baked(vol, static, white_back=True)
    for rays in (a, b, a):
        static.copy_(rays)
        g.replay()
        torch.cuda.synchronize()
        tb._same(out, nb.render_baked(vol, rays, white_back=True), "replay")


@pytest.mark.parametrize("eps", [1e-3, 0.1])
def test_early_stop(eps):
    nb = _nb()
    vol = _volume()
    rays = tb._rays(3000, 31, box=UNEQUAL)
    full = nb.render_baked(vol, rays, white_back=True)
    cut = nb.render_baked(vol, rays, white_back=True, early_stop=eps)
    never = (1 - full["opacity"].double()) >= eps + 1e-5
    assert never.any()
    for k in ("rgb", "depth", "opacity"):
        assert torch.equal(tb._bits(full[k][never]), tb._bits(cut[k][never])), k
    diff = cut["opacity"] != full["opacity"]
    assert diff.any()
    T_cut = 1 - cut["opacity"].double()
    assert bool((T_cut[diff] < eps + 1e-5).all())
    assert bool(((cut["rgb"].double() - full["rgb"].double()).abs().max(1).values <= T_cut + 1e-5).all())
    assert bool(((cut["depth"].double() - full["depth"].double()).abs() <= T_cut * 9.0 + 1e-4).all())


# ---- trained scene ----------------------------------------------------------------------------------------------------
# PSNR of the SH render (N = 256) against the MLP render (64 + 128, skip="samples") on three 200 x 200 Blender views.
# Measured on an H100 80GB HBM3: 45.52, 45.69 and 45.05 dB (the direction-0 bake of test_gpu_baked.py: 44.06, 43.73,
# 43.07).  The bar leaves 3 dB below the worst view.
PSNR_BAR = 42.0


def test_trained_scene_psnr_against_the_mlp():
    if not cases.have_trained():
        pytest.skip("no trained weights")
    nb = _nb()
    models = [_model_of(w) for w in cases.trained_weights()]
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    grid = nb.occupancy_grid(models[1], 128, *CUBE, 1.0, dilate=1)
    vol = nb.bake_volume(models[1], 256, *CUBE, occupancy=grid, view_dependent=True)
    psnr = []
    for v in range(3):
        rays = torch.from_numpy(bench.blender_rays(0, 80 + v, W=200, H=200, pixels="all")).cuda()
        mlp = nb.batched_inference(models, emb, rays, 64, 128, False, white_back=True, occupancy=grid, skip="samples")
        out = nb.render_baked(vol, rays, white_back=True)
        psnr.append(-10 * np.log10(float(((out["rgb"] - mlp["rgb_fine"]) ** 2).mean())))
    print(f"\nSH baked vs MLP PSNR on the trained scene: {psnr}")
    assert min(psnr) > PSNR_BAR, psnr
