"""Mesh and Unity-volume grids through an occupancy grid on the device (nb.sigma_grid / nb.rgb_sigma_grid /
nb.extract_mesh / nb.fuse_vertex_colors / nb.normal_vertex_colors with occupancy=; csrc/masked_grid_kernels.cuh).

An evaluated lattice point (tests/mesh_grid_ref.py: the float64 rule of skip="samples" on the fp32 lattice
positions) gets the plain grid's value bit for bit, every other point exactly zero; the evaluated count is the
replica's; nothing depends on the chunk or the CTA count; the trained network's mesh is the plain mesh; the colour
paths are render_rays_culled(..., skip="samples") bit for bit, and the plain calls when nothing is skipped."""
import copy
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as mo
from oracle import nerf_oracle as orc
from tests import cases
from tests import mesh_grid_ref as mg

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUBE = ((-1.5, 1.5),) * 3
UNEQUAL = ((-1.5, 1.5), (-1.2, 1.4), (-1.5, 1.3))
REVERSED = ((1.5, -1.5), (-1.2, 1.4), (1.3, -1.5))
INSIDE = ((-0.9, 1.1), (-1.0, 0.8), (-1.1, 0.7))       # strictly inside CUBE
# (mesh box, occupancy box)
BOXES = {"cube": (CUBE, CUBE), "unequal_reversed": (UNEQUAL, REVERSED), "reversed_unequal": (REVERSED, UNEQUAL),
         "grid_inside": (CUBE, INSIDE)}


def _nb():
    import nerf_pl_b200 as nb
    return nb


_M = {}


def _model(kind="random"):
    """The fine network of seeded random weights ("random") or of the trained test weights ("trained")."""
    if kind not in _M:
        ws = cases.trained_weights() if kind.startswith("trained") else [orc.make_weights(22), orc.make_weights(21)]
        ms = []
        for w in ws:
            m = _nb().NeRF()
            m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
            ms.append(m.cuda().eval())
        _M[kind] = ms
    return _M[kind][1]


def _coarse(kind):
    _model(kind)
    return _M[kind][0]


def _grid(words, occ_N, ranges):
    return _nb().OccupancyGrid(torch.from_numpy(np.asarray(words, np.uint32).view(np.int32)).cuda(), occ_N, *ranges)


def _i32(t):
    return t.detach().cpu().numpy().view(np.int32)


def _check(model, N, mesh, grid, words, channels=1, chunk=1 << 21):
    """The masked grid against the plain one and the replica; returns (masked, plain, evaluated mask) on the host."""
    nb = _nb()
    fn = nb.sigma_grid if channels == 1 else nb.rgb_sigma_grid
    plain = fn(model, N, *mesh).cpu().numpy().reshape(N ** 3, -1)
    out, evaluated = fn(model, N, *mesh, chunk=chunk, occupancy=grid, return_evaluated=True)
    assert out.shape == ((N,) * 3 if channels == 1 else (N,) * 3 + (4,)) and out.dtype == torch.float32
    got = out.cpu().numpy().reshape(N ** 3, -1)
    ev = mg.evaluated_points(N, *mesh, words, grid.N, grid.ranges)
    assert evaluated == int(ev.sum())
    assert np.array_equal(got[ev].view(np.int32), plain[ev].view(np.int32))
    assert not got[~ev].view(np.int32).any()                     # +0.0, every channel
    return got, plain, ev


@pytest.mark.parametrize("N, occ_N, box", list(itertools.product((2, 17, 33, 128), (2, 17, 65), BOXES)))
def test_masked_sigma_grid(N, occ_N, box):
    mesh, occ = BOXES[box]
    words = mg.random_words(occ_N, 0.3 if occ_N > 2 else 1.0, seed=N * 1000 + occ_N)
    _, _, ev = _check(_model(), N, mesh, _grid(words, occ_N, occ), words)
    if N >= 33 and occ_N > 2:
        assert 0 < ev.sum() < N ** 3                              # a partial grid: both kinds of point occur


@pytest.mark.parametrize("ranges", [CUBE, UNEQUAL])
def test_every_lattice_point_a_cell_corner(ranges):
    """Mesh N = occupancy N on the same box: every lattice point is a corner, evaluated iff one of the up to 8 cells
    around it is occupied."""
    for fill, seed in ((0.02, 1), (0.3, 2), (0.7, 3)):
        words = mg.random_words(33, fill, seed)
        _check(_model(), 33, ranges, _grid(words, 33, ranges), words)


def test_empty_grid_is_zero_without_an_mlp_launch():
    nb = _nb()
    lib = nb._lib.load()
    model = _model()
    before = lib.nerfb200_launch_count()
    nb.nerf.packed_weights(model)                                 # the weight image each call takes
    packs = lib.nerfb200_launch_count() - before
    for channels, fn in ((1, nb.sigma_grid), (4, nb.rgb_sigma_grid)):
        grid = _grid(mg.random_words(17, 0.0, 0), 17, CUBE)
        for chunk in (33 ** 3, 5000):
            before = lib.nerfb200_launch_count()
            out, evaluated = fn(model, 33, *CUBE, chunk=chunk, occupancy=grid, return_evaluated=True)
            # classify and scan per chunk, nothing else
            assert lib.nerfb200_launch_count() - before == 2 * -(-33 ** 3 // chunk) + packs
            assert evaluated == 0 and not _i32(out).any()


@pytest.mark.parametrize("N", [17, 64])
def test_full_grid_is_the_plain_grid(N):
    words = mg.random_words(9, 1.0, 0)
    for channels in (1, 4):
        got, plain, ev = _check(_model(), N, CUBE, _grid(words, 9, CUBE), words, channels)
        assert ev.all() and np.array_equal(got.view(np.int32), plain.view(np.int32))


def test_independent_of_chunk():
    N = 17
    words = mg.random_words(9, 0.3, 4)
    grid = _grid(words, 9, UNEQUAL)
    for channels in (1, 4):
        fn = _nb().sigma_grid if channels == 1 else _nb().rgb_sigma_grid
        base, n0 = fn(_model(), N, *CUBE, occupancy=grid, return_evaluated=True)
        for chunk in (1, 127, 4096, 4097, N ** 3 - 1, N ** 3):
            out, n = fn(_model(), N, *CUBE, chunk=chunk, occupancy=grid, return_evaluated=True)
            assert n == n0 and np.array_equal(_i32(out), _i32(base)), (channels, chunk)


_SUBPROCESS = r"""
import sys
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
import nerf_pl_b200 as nb
from oracle import nerf_oracle as orc
m = nb.NeRF()
m.load_state_dict({k: torch.from_numpy(v) for k, v in orc.make_weights(21).items()})
m = m.cuda().eval()
words = np.load(sys.argv[2])
grid = nb.OccupancyGrid(torch.from_numpy(words.view(np.int32)).cuda(), 17, (1.5, -1.5), (-1.2, 1.4), (1.3, -1.5))
box = ((-1.5, 1.5),) * 3
s, ns = nb.sigma_grid(m, 45, *box, chunk=20000, occupancy=grid, return_evaluated=True)
r, nr = nb.rgb_sigma_grid(m, 45, *box, chunk=20000, occupancy=grid, return_evaluated=True)
np.savez(sys.argv[3], s=s.cpu().numpy(), r=r.cpu().numpy(), n=np.array([ns, nr]))
"""


def test_independent_of_the_cta_count(tmp_path):
    words = mg.random_words(17, 0.3, 5)
    np.save(tmp_path / "w.npy", words)
    env = dict(os.environ, NERFB200_MAX_CTAS="1")
    subprocess.run([sys.executable, "-c", _SUBPROCESS, ROOT, str(tmp_path / "w.npy"), str(tmp_path / "o.npz")],
                   check=True, env=env, cwd=ROOT)
    z = np.load(tmp_path / "o.npz")
    grid = _grid(words, 17, REVERSED)
    s, ns = _nb().sigma_grid(_model(), 45, *CUBE, occupancy=grid, return_evaluated=True)
    r, nr = _nb().rgb_sigma_grid(_model(), 45, *CUBE, occupancy=grid, return_evaluated=True)
    assert list(z["n"]) == [ns, nr] and 0 < ns < 45 ** 3
    assert np.array_equal(z["s"].view(np.int32), _i32(s)) and np.array_equal(z["r"].view(np.int32), _i32(r))


@pytest.mark.parametrize("N, occ_N, box", [(17, 17, "cube"), (33, 65, "unequal_reversed"), (128, 17, "grid_inside"),
                                           (33, 2, "reversed_unequal"), (64, 65, "cube")])
def test_masked_rgb_sigma_grid_and_its_volume(N, occ_N, box):
    nb = _nb()
    mesh, occ = BOXES[box]
    model = _model("trained") if cases.have_trained() else _model()
    words = mg.random_words(occ_N, 0.3 if occ_N > 2 else 1.0, seed=N + occ_N)
    got, plain, ev = _check(model, N, mesh, _grid(words, occ_N, occ), words, channels=4)
    zeroed = plain.copy()
    zeroed[~ev] = 0.0
    a = nb.pack_volume(torch.from_numpy(got.reshape(N, N, N, 4)).cuda(), mesh[0]).view(torch.int32).cpu().numpy()
    b = nb.pack_volume(torch.from_numpy(zeroed.reshape(N, N, N, 4)).cuda(), mesh[0]).view(torch.int32).cpu().numpy()
    assert np.array_equal(a, b)
    assert np.all(ev[a[:, 0].view(np.uint32).astype(np.int64)])                   # every packed point was evaluated


# ---- the trained test weights, with the grid of the trained scene (sigma > 1 on 128 points, dilate 1) ------------
_GRID = []


def _trained_grid():
    if not _GRID:
        _GRID.append(_nb().occupancy_grid(_model("trained"), 128, *CUBE, 1.0, dilate=1))
    return _GRID[0]


def _trained():
    if not cases.have_trained():
        pytest.skip("no trained weights")


@pytest.mark.parametrize("N", [128, 256])
def test_trained_mesh_is_the_plain_mesh(N):
    """A lattice point with sigma > 20 lies in an occupied cell, and the dilation occupies its neighbours, so every
    edge marching cubes crosses has both ends evaluated: the same vertices and triangles, before and after the
    cluster filter."""
    _trained()
    nb = _nb()
    fine, grid = _model("trained"), _trained_grid()
    sigma, evaluated = nb.sigma_grid(fine, N, *CUBE, occupancy=grid, return_evaluated=True)
    print(f"N_grid {N}: {evaluated / N ** 3:.4f} of the lattice points evaluated, occupied cells "
          f"{grid.occupied_fraction():.4f}")
    for keep in (False, True):
        v0, t0 = nb.extract_mesh(fine, N, *CUBE, 20.0, keep_largest=keep)
        v1, t1 = nb.extract_mesh(fine, N, *CUBE, 20.0, keep_largest=keep, occupancy=grid)
        assert len(t0) > 1000
        assert torch.equal(v0.view(torch.int32), v1.view(torch.int32)) and torch.equal(t0, t1), keep


def _look_at(eye):
    eye = np.asarray(eye, np.float64)
    f = -eye / np.linalg.norm(eye)
    r = np.cross(f, [0, 0, 1.0])
    r /= np.linalg.norm(r)
    return np.stack([r, np.cross(r, f), -f, eye], 1)


def _views():
    poses = [_look_at(e) for e in ([3.5, 0.4, 0.8], [-1.2, 3.1, -0.6], [0.3, -2.6, 2.4], [0.2, 0.3, -3.9])]
    H, W = 60, 80
    yy, xx = np.mgrid[0:H, 0:W]
    images = np.stack([np.stack([(xx * 3 + k * 40) % 256, (yy * 4 + k * 17) % 256, (xx + yy + 60 * k) % 256], -1)
                       for k in range(len(poses))]).astype(np.uint8)
    return torch.from_numpy(images).cuda(), poses, 70.0, 1.0


def _full_grid_around(rays):
    """A one-cell grid, occupied, over a box holding every point between near and far of every ray."""
    r = rays.double()
    ends = torch.cat([r[:, :3] + r[:, 3:6] * r[:, 6:7], r[:, :3] + r[:, 3:6] * r[:, 7:8]])
    lo, hi = ends.amin(0).cpu().numpy(), ends.amax(0).cpu().numpy()
    pad = 0.01 * (hi - lo).max() + 0.01
    return _grid(np.array([1], np.uint32), 2, [(lo[a] - pad, hi[a] + pad) for a in range(3)])


def test_fused_colours_through_the_grid():
    _trained()
    nb = _nb()
    fine, grid = _model("trained"), _trained_grid()
    v, _ = nb.extract_mesh(fine, 64, *CUBE, 20.0)
    images, poses, focal, near = _views()
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    cols, opac = nb.fuse_vertex_colors(fine, v, images, poses, focal, near, return_opacities=True, occupancy=grid)
    all_rays = []
    for k in range(len(poses)):
        _, _, rays = nb.mesh.project_view(v, images[k], poses[k], focal, near)
        all_rays.append(rays)
        want = nb.render_rays_culled([fine], emb, rays, grid, 64, False, 0, False, True, skip="samples")
        assert torch.equal(want["opacity_coarse"].view(torch.int32), opac[k].view(torch.int32)), k
    ref = mo.fuse_colors(v.cpu().numpy(), images.cpu().numpy(), poses, focal, opac.cpu().numpy(), 0.2)
    assert np.array_equal(cols.cpu().numpy(), ref)
    # nothing to skip: the plain call bit for bit
    full = _full_grid_around(torch.cat(all_rays))
    c0, o0 = nb.fuse_vertex_colors(fine, v, images, poses, focal, near, return_opacities=True)
    c1, o1 = nb.fuse_vertex_colors(fine, v, images, poses, focal, near, return_opacities=True, occupancy=full)
    assert torch.equal(c0, c1) and torch.equal(o0.view(torch.int32), o1.view(torch.int32))


def test_normal_colours_through_the_grid():
    _trained()
    nb = _nb()
    coarse, fine, grid = _coarse("trained"), _model("trained"), _trained_grid()
    v, t = nb.extract_mesh(fine, 64, *CUBE, 20.0)
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    for white_back in (False, True):
        got = nb.normal_vertex_colors(coarse, fine, v, t, 2.0, 6.0, white_back=white_back, occupancy=grid)
        rays = nb.normal_rays(v, nb.vertex_normals(v, t), 2.0, 6.0)
        want = nb.render_rays_culled([coarse, fine], emb, rays, grid, 64, False, 64, white_back, True, skip="samples")
        assert got.dtype == torch.uint8 and torch.equal(got, nb.to_uint8(want["rgb_fine"]))
        full = _full_grid_around(rays)
        plain = nb.normal_vertex_colors(coarse, fine, v, t, 2.0, 6.0, white_back=white_back)
        assert torch.equal(nb.normal_vertex_colors(coarse, fine, v, t, 2.0, 6.0, white_back=white_back,
                                                   occupancy=full), plain)


def test_argument_errors():
    nb = _nb()
    model = _model()
    grid = _grid(mg.random_words(9, 0.5, 0), 9, CUBE)
    v = torch.rand(10, 3, device="cuda")
    t = torch.tensor([[0, 1, 2]], dtype=torch.int32, device="cuda")
    images = torch.zeros(1, 8, 8, 3, dtype=torch.uint8, device="cuda")
    pose = [_look_at([3.0, 0.0, 0.0])]
    dg = nb.DensityGrid(9, *CUBE)
    calls = {
        "sigma_grid": lambda occ: nb.sigma_grid(model, 9, *CUBE, occupancy=occ),
        "rgb_sigma_grid": lambda occ: nb.rgb_sigma_grid(model, 9, *CUBE, occupancy=occ),
        "extract_mesh": lambda occ: nb.extract_mesh(model, 9, *CUBE, 20.0, occupancy=occ),
        "fuse_vertex_colors": lambda occ: nb.fuse_vertex_colors(model, v, images, pose, 10.0, 1.0, occupancy=occ),
        "normal_vertex_colors": lambda occ: nb.normal_vertex_colors(model, model, v, t, 2.0, 6.0, occupancy=occ),
    }
    elsewhere = copy.copy(grid)
    elsewhere.bits = grid.bits.to("meta")                        # a grid whose bits live on another device
    for name, fn in calls.items():
        for bad in (grid.bits, dg, "grid", 1):
            with pytest.raises(ValueError, match="OccupancyGrid"):
                fn(bad)
        with pytest.raises(RuntimeError, match="occupancy grid is on"):
            fn(elsewhere)
        fn(dg.grid)                                               # a DensityGrid's grid is an OccupancyGrid
    with pytest.raises(ValueError, match="1625"):
        nb.rgb_sigma_grid(model, 1626, *CUBE, occupancy=grid)
    with pytest.raises(ValueError, match="N < 2"):
        nb.sigma_grid(model, 1, *CUBE, occupancy=grid)
    with pytest.raises(ValueError, match="chunk"):
        nb.sigma_grid(model, 9, *CUBE, chunk=0, occupancy=grid)
    with pytest.raises(ValueError, match="min, max"):
        nb.sigma_grid(model, 9, (-1.0, 1.0), (-1.0,), (-1.0, 1.0), occupancy=grid)
    cpu = nb.NeRF()
    with pytest.raises(RuntimeError, match="CUDA"):
        nb.sigma_grid(cpu, 9, *CUBE, occupancy=grid)
    # without a grid nothing changes, and return_evaluated counts every point
    s, n = nb.sigma_grid(model, 9, *CUBE, return_evaluated=True)
    assert n == 9 ** 3 and torch.equal(s, nb.sigma_grid(model, 9, *CUBE))
