"""Empty-space skipping on the device (nerf_pl_b200.culling) against the float64 reference (tests/occupancy_ref.py):
the bit field exactly, the ray flags away from grazing rays, the compaction, the scatter, and on the trained network
the two things culling promises: live rays bit-identical to the plain render, culled rays within a measured bound of
the vacuum value."""
import numpy as np
import pytest
import torch

import bench
from tests import cases
from tests import occupancy_ref as oc

pytestmark = pytest.mark.gpu
CUBE = ((-1.5, 1.5),) * 3
UNEQUAL = ((-1.5, 1.5), (1.4, -1.2), (-1.5, 1.3))            # y reversed
THR = 2.0


def _nb():
    import nerf_pl_b200 as nb
    return nb


_MODELS = []


def _models():
    if not _MODELS:
        for w in cases.trained_weights():
            m = _nb().NeRF()
            m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
            _MODELS.append(m.cuda().eval())
    return _MODELS


def _emb():
    return [_nb().Embedding(3, 10), _nb().Embedding(3, 4)]


def _sigma(kind, N, seed=0):
    """Synthetic sigma grids: values below, at and above the threshold, and a few NaN (never above)."""
    rng = np.random.default_rng(1000 * N + seed)
    if kind == "full":
        return np.full((N, N, N), THR + 1.0, np.float32)
    if kind == "empty":
        s = np.full((N, N, N), THR, np.float32)              # exactly the threshold: not occupied
        s[rng.random(s.shape) < 0.01] = np.nan
        return s
    s = rng.uniform(0.0, THR, (N, N, N)).astype(np.float32)
    s[rng.random(s.shape) < (0.4 if N == 2 else 0.003)] = THR + 0.5
    s[rng.random(s.shape) < 0.01] = np.nan
    s[rng.random(s.shape) < 0.01] = THR
    return s


def _grid(sigma, ranges, dilate):
    return _nb().pack_occupancy(torch.from_numpy(sigma).cuda(), *ranges, THR, dilate)


def _words(grid):
    return grid.bits.cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("dilate", [0, 1, 3])
@pytest.mark.parametrize("N", [2, 33, 64, 100])
@pytest.mark.parametrize("kind", ["sparse", "full", "empty"])
def test_bit_field_equals_the_reference_exactly(kind, N, dilate):
    sigma = _sigma(kind, N)
    want = oc.occupancy(sigma, THR, dilate)
    grid = _grid(sigma, UNEQUAL, dilate)
    assert grid.N == N and grid.dilate == dilate and grid.bits.numel() == ((N - 1) ** 3 + 31) // 32
    assert np.array_equal(_words(grid), oc.pack_bits(want))
    assert np.array_equal(grid.to_dense().cpu().numpy(), want)
    assert grid.occupied_fraction() == want.sum() / want.size
    if kind == "sparse" and N > 2:
        assert 0 < want.sum() < want.size


def test_state_dict_round_trip():
    nb = _nb()
    grid = _grid(_sigma("sparse", 33), UNEQUAL, 1)
    state = grid.state_dict()
    assert not state["bits"].is_cuda
    again = nb.OccupancyGrid.from_state_dict(state)
    other = _grid(_sigma("empty", 5), CUBE, 0).load_state_dict(state)
    for g in (again, other):
        assert torch.equal(g.bits, grid.bits) and g.bits.is_cuda
        assert (g.N, g.ranges, g.dilate) == (grid.N, grid.ranges, grid.dilate)


def _random_rays(n, ranges, seed):
    """Rays around and inside the box: most aimed at it from outside, some starting inside, with random segments
    and some axis-parallel directions."""
    rng = np.random.default_rng(seed)
    lo = np.array([min(r) for r in ranges])
    hi = np.array([max(r) for r in ranges])
    mid, half = (lo + hi) / 2, (hi - lo) / 2
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    o = mid + 4.0 * u
    inside = rng.random(n) < 0.2
    o[inside] = (mid + half * rng.uniform(-1, 1, (n, 3)))[inside]
    target = mid + 1.3 * half * rng.uniform(-1, 1, (n, 3))
    d = target - o
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    axis_par = rng.random(n) < 0.1
    d[axis_par, rng.integers(0, 3, n)[axis_par]] = 0.0
    d *= rng.uniform(0.5, 2.0, (n, 1))                        # culling takes d as given, unit or not
    near = rng.uniform(0.0, 3.0, n)
    far = near + rng.uniform(0.01, 6.0, n)
    return np.concatenate([o, d, near[:, None], far[:, None]], 1).astype(np.float32)


@pytest.mark.parametrize("N,ranges", [(33, CUBE), (64, UNEQUAL), (100, UNEQUAL)])
def test_ray_flags_match_the_float64_walk(N, ranges):
    nb = _nb()
    sigma = _sigma("sparse", N, seed=1)
    occ = oc.occupancy(sigma, THR, 1)
    grid = _grid(sigma, ranges, 1)
    rays = _random_rays(50000, ranges, N)
    _, _, flag = nb.cull_rays(torch.from_numpy(rays).cuda(), grid, return_flag=True)
    flag = flag.cpu().numpy().astype(bool)
    want, margin = oc.ray_live(rays, occ, ranges)
    clear = margin > 1e-4
    print(f"N {N}: {int((~clear).sum())} of {len(rays)} rays graze a cell boundary within 1e-4 of a cell and are "
          f"excluded; {int((flag != want)[~clear].sum())} of those differ; live fraction {want.mean():.3f}")
    assert clear.mean() > 0.8
    assert want[clear].any() and not want[clear].all()
    assert np.array_equal(flag[clear], want[clear])


def test_ray_guards_one_by_one():
    nb = _nb()
    occ, box, rays, want = oc.guard_cases()
    for cells, ranges in ((occ, box), (occ[::-1], ((2.0, -2.0), (-2.0, 2.0), (-2.0, 2.0)))):
        bits = torch.from_numpy(oc.pack_bits(cells).view(np.int32)).cuda()
        grid = nb.OccupancyGrid(bits, 5, *ranges)
        assert np.array_equal(grid.to_dense().cpu().numpy(), cells)
        live_idx, live_rays, flag = nb.cull_rays(torch.from_numpy(rays).cuda(), grid, return_flag=True)
        assert flag.cpu().numpy().astype(bool).tolist() == want.tolist()
        assert live_idx.cpu().numpy().tolist() == np.nonzero(want)[0].tolist()
        assert np.array_equal(live_rays.cpu().numpy(), rays[want], equal_nan=True)


@pytest.mark.parametrize("mode", ["mixed", "all", "none"])
@pytest.mark.parametrize("n", [1, 31, 1024, 160000])
def test_compaction_is_stable_and_complete(n, mode):
    nb = _nb()
    N = 33
    grid = _grid(_sigma({"mixed": "sparse", "all": "full", "none": "empty"}[mode], N, seed=2), CUBE, 1)
    rays = _random_rays(n, CUBE, n)
    if mode == "all":                                          # every segment inside the box crosses an occupied cell
        rays[:, :3] = np.clip(rays[:, :3], -1.4, 1.4)
        rays[:, 6] = 0.0
    r = torch.from_numpy(rays).cuda()
    live_idx, live_rays, flag = nb.cull_rays(r, grid, return_flag=True)
    assert live_idx.dtype == torch.int64 and live_rays.dtype == torch.float32 and flag.dtype == torch.uint8
    assert live_rays.shape == (live_idx.shape[0], 8) and flag.shape == (n,)
    assert torch.equal(live_idx, flag.nonzero().reshape(-1))
    if live_idx.numel() > 1:
        assert bool((live_idx[1:] > live_idx[:-1]).all())
    assert torch.equal(live_rays, r[live_idx])
    if mode == "all":
        assert live_idx.numel() == n
    if mode == "none":
        assert live_idx.numel() == 0
    if mode == "mixed" and n >= 1024:
        assert 0 < live_idx.numel() < n
    a, b = nb.cull_rays(r, grid)
    assert torch.equal(a, live_idx) and torch.equal(b, live_rays)


def test_no_rays():
    nb = _nb()
    grid = _grid(_sigma("sparse", 33), CUBE, 1)
    live_idx, live_rays = nb.cull_rays(torch.empty(0, 8, device="cuda"), grid)
    assert live_idx.shape == (0,) and live_rays.shape == (0, 8)


@pytest.mark.parametrize("white_back", [False, True])
@pytest.mark.parametrize("K,test_time", [(64, True), (64, False), (0, True), (0, False)])
@pytest.mark.parametrize("n,frac", [(1, 1.0), (1000, 0.0), (1000, 1.0), (70001, 0.37)])
def test_scatter_equals_full_plus_index_copy(n, frac, K, test_time, white_back):
    nb = _nb()
    keys = oc.result_keys(K, test_time)
    g = torch.Generator(device="cuda").manual_seed(n + K)
    live_idx = (torch.rand(n, device="cuda", generator=g) < frac).nonzero().reshape(-1)
    n_live = live_idx.numel()
    compact = {k: torch.rand((n_live, 3) if k.startswith("rgb") else (n_live,), device="cuda", generator=g) for k in keys}
    out = nb.scatter_results(compact if n_live else None, live_idx, n, white_back, keys)
    assert list(out) == keys
    for k in keys:
        want = torch.full((n, 3) if k.startswith("rgb") else (n,), 1.0 if (white_back and k.startswith("rgb")) else 0.0,
                          device="cuda")
        want.index_copy_(0, live_idx, compact[k])
        assert out[k].dtype == torch.float32 and torch.equal(out[k], want), k


# ---- the trained network ----------------------------------------------------------------------------------------
# The grid the end-to-end tests use: N = 128 over the box the scene was trained in, cells occupied above sigma 1
# (the surfaces of tests/test_gpu_mesh_field.py are extracted at 20), dilated by one cell.
GRID_N, GRID_THR, GRID_DILATE = 128, 1.0, 1
_GRID = []


def _trained_grid():
    if not _GRID:
        _GRID.append(_nb().occupancy_grid(_models()[1], GRID_N, *CUBE, GRID_THR, GRID_DILATE))
    return _GRID[0]


def _view(side, seed):
    """Every pixel of a side x side Blender-style view of the trained scene (radius-4 camera, near 2, far 6)."""
    return torch.from_numpy(bench.blender_rays(0, seed, W=side, H=side, pixels="all")).cuda()


def test_trained_grid_is_the_dilated_cell_max_of_its_sigma_grid():
    nb = _nb()
    grid = _trained_grid()
    sigma = nb.sigma_grid(_models()[1], GRID_N, *CUBE).cpu().numpy()
    want = oc.occupancy(sigma, GRID_THR, GRID_DILATE)
    assert np.array_equal(grid.to_dense().cpu().numpy(), want)
    frac = grid.occupied_fraction()
    print(f"trained grid: {frac:.4f} of {GRID_N - 1}^3 cells occupied")
    assert 0.01 < frac < 0.5


# What the plain render gives on the culled rays of the three views below, minus the vacuum value.  Measured on an
# NVIDIA H100 80GB HBM3 at 64 + 128 samples: mean |rgb_fine - 1| 4.9e-4, 1.1e-5 and 1.1e-5, mean opacity_fine 2.4e-2,
# 3.1e-4 and 7.5e-4.  The MAXIMUM is not small and no grid setting makes it so: this network was trained on 64 views
# and holds opaque density outside the box (for a few rays even non-white: max |rgb_fine - 1| 0.35, 5.5e-3 and 1.4e-2,
# max opacity_fine 1.0), and space outside the box counts as empty.  A box of [-2.6, 2.6]^3 at sigma > 0.05 brings two
# of the views to max |rgb_fine - 1| 0 and 1.6e-4 and leaves the first at 0.35 (DESIGN.md has the table).  So the
# means are pinned, at about three times the worst measured value.
CULLED_MEAN_RGB = 1.5e-3
CULLED_MEAN_OPACITY = 8e-2


@pytest.mark.parametrize("seed", [61, 62, 63])
@pytest.mark.parametrize("K", [64, 128])
def test_culled_render_of_the_trained_scene(K, seed):
    nb = _nb()
    grid = _trained_grid()
    rays = _view(200, seed)
    n = rays.shape[0]
    with torch.no_grad():
        plain = nb.render_rays(_models(), _emb(), rays, 64, False, 0, 0, K, 32768, True, test_time=True,
                               match_reference_rng=False)
    culled = nb.render_rays_culled(_models(), _emb(), rays, grid, 64, False, K, True, test_time=True)
    live_idx = culled["live_idx"]
    assert culled["live"] == live_idx.numel() and live_idx.dtype == torch.int64
    assert set(culled) == set(plain) | {"live", "live_idx"}
    dead = torch.ones(n, dtype=torch.bool, device="cuda")
    dead[live_idx] = False
    for k, v in plain.items():
        assert culled[k].shape == v.shape and culled[k].dtype == v.dtype
        assert torch.equal(culled[k][live_idx], v[live_idx]), k            # live rays: bit for bit
    want = oc.vacuum_results(int(dead.sum()), list(plain), True)
    for k in plain:
        assert np.array_equal(culled[k][dead].cpu().numpy(), want[k]), k
    opac, err = plain["opacity_fine"][dead], (plain["rgb_fine"][dead] - 1.0).abs().amax(1)
    print(f"view {seed}, 64 + {K}: {culled['live']} of {n} rays live ({culled['live'] / n:.3f}); on the culled rays the "
          f"plain render has opacity_fine mean {float(opac.mean()):.3e} max {float(opac.max()):.3e}, |rgb_fine - 1| mean "
          f"{float(err.mean()):.3e} max {float(err.max()):.3e}, {int((err > 1e-2).sum())} rays above 1e-2")
    assert dead.float().mean() >= 1 / 3                                    # the grid does something
    assert float(err.mean()) < CULLED_MEAN_RGB and float(opac.mean()) < CULLED_MEAN_OPACITY


def test_culled_render_with_the_coarse_results_and_a_black_background():
    nb = _nb()
    grid = _trained_grid()
    rays = _view(96, 64)
    for white_back, K in ((False, 64), (True, 0)):
        with torch.no_grad():
            plain = nb.render_rays(_models(), _emb(), rays, 64, False, 0, 0, K, 32768, white_back, test_time=False,
                                   match_reference_rng=False)
        culled = nb.render_rays_culled(_models(), _emb(), rays, grid, 64, False, K, white_back, test_time=False)
        assert list(plain) == oc.result_keys(K, False)
        live_idx = culled["live_idx"]
        want = oc.scatter({k: v[live_idx].cpu().numpy() for k, v in plain.items()}, live_idx.cpu().numpy(),
                          rays.shape[0], white_back)
        for k in plain:
            assert np.array_equal(culled[k].cpu().numpy(), want[k]), k


def test_no_live_ray_means_no_render_launch():
    nb = _nb()
    lib = nb._lib.load()
    grid = _grid(_sigma("empty", 33), CUBE, 1)
    rays = _view(64, 65)
    before = lib.nerfb200_launch_count()
    out = nb.render_rays_culled(_models(), _emb(), rays, grid, 64, False, 64, True)
    assert lib.nerfb200_launch_count() - before == 3                       # classify, scan, scatter
    assert out["live"] == 0 and out["live_idx"].numel() == 0
    assert bool((out["rgb_fine"] == 1).all()) and bool((out["opacity_fine"] == 0).all())
    assert bool((out["depth_fine"] == 0).all()) and bool((out["opacity_coarse"] == 0).all())


def test_inference_entries_take_the_grid_and_default_to_the_plain_path():
    nb = _nb()
    grid = _trained_grid()
    rays = _view(96, 66)
    args = (_models(), _emb(), rays, 64, 64, False, 32768, True)
    plain = nb.batched_inference(*args)
    same = nb.batched_inference(*args, occupancy=None)
    assert list(plain) == list(same) and all(torch.equal(plain[k], same[k]) for k in plain)
    culled = nb.batched_inference(*args, occupancy=grid)
    direct = nb.render_rays_culled(_models(), _emb(), rays, grid, 64, False, 64, True)
    assert culled["live"] == direct["live"] and 0 < culled["live"] < rays.shape[0]
    for k in plain:
        assert torch.equal(culled[k], direct[k]), k
    # sharded without a process group is one rank: the same result
    one_rank = nb.batched_inference(*args, sharded=True, occupancy=grid)
    assert all(torch.equal(one_rank[k], culled[k]) for k in plain)

    c2w = np.array([[1, 0, 0, 0.1], [0, 0, -1, -4.0], [0, 1, 0, 0.2]], np.float32)
    cam = (_models(), _emb(), 80, 80, 110.0, c2w, 2.0, 6.0)
    img = nb.render_image(*cam, white_back=True)
    img_none = nb.render_image(*cam, white_back=True, occupancy=None)
    assert list(img) == list(img_none) and all(torch.equal(img[k], img_none[k]) for k in img)
    img_c = nb.render_image(*cam, white_back=True, occupancy=grid)
    assert 0 < img_c["live"] < 80 * 80 and img_c["rgb_uint8"].shape == (80, 80, 3)
    live = nb.cull_rays(img["rays"], grid)[0]
    assert torch.equal(img_c["rgb"].view(-1, 3)[live], img["rgb"].view(-1, 3)[live])
    assert float((img_c["rgb"] - img["rgb"]).abs().mean()) < CULLED_MEAN_RGB


def test_culling_is_inference_only():
    nb = _nb()
    grid = _trained_grid()
    rays = _view(16, 67)
    with pytest.raises(ValueError, match="inference only"):
        nb.render_rays_culled(_models(), _emb(), rays, grid, 64, False, 64, True, perturb=1.0)
    with pytest.raises(ValueError, match="inference only"):
        nb.render_rays_culled(_models(), _emb(), rays, grid, 64, False, 64, True, noise_std=1.0)
    with pytest.raises(ValueError):
        nb.render_rays_culled(_models(), _emb(), rays[:, :6], grid, 64, False, 64, True)
    with torch.enable_grad():
        out = nb.render_rays_culled(_models(), _emb(), rays, grid, 64, False, 64, True)
    assert not out["rgb_fine"].requires_grad
