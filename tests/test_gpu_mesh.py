"""Coloured-mesh extraction on the device (nerf_pl_b200.mesh) against the numpy restatement
(oracle/mesh_oracle.py): grid, marching cubes, cluster filter, bilinear sampling and colour fusion."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as mo
from oracle import nerf_oracle as orc
from tests import cases

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CENTERS = np.array([[0.0, 0.0, 0.0], [0.9, 0.3, -0.2], [-0.6, -0.7, 0.4]])
RADII = np.array([0.8, 0.45, 0.55])
RANGE = (-1.5, 1.5)


def _nb():
    import nerf_pl_b200 as nb
    return nb


def _fine_model():
    nb = _nb()
    m = nb.NeRF()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in cases.trained_weights()[1].items()})
    return m.cuda().eval()


def _sphere(n, r, c):
    g = np.stack(np.meshgrid(*(np.arange(n),) * 3, indexing="ij"), -1).astype(np.float64)
    return (r - np.linalg.norm(g - np.asarray(c), axis=-1)).astype(np.float32)


def _torus(n, R, r):
    g = np.stack(np.meshgrid(*(np.arange(n),) * 3, indexing="ij"), -1).astype(np.float64) - (n - 1) / 2 - 0.17
    q = np.hypot(g[..., 0], g[..., 1]) - R
    return (r - np.hypot(q, g[..., 2])).astype(np.float32)


def _grids():
    rng = np.random.default_rng(3)
    return {
        "random32": (rng.normal(0, 1, (32, 32, 32)).astype(np.float32), 0.2),
        "random_shape": (rng.uniform(0, 40, (33, 40, 36)).astype(np.float32), 20.0),
        "sphere48": (_sphere(48, 17.3, (23.2, 24.7, 22.9)), 0.0),
        "torus64": (_torus(64, 18.0, 7.5), 0.0),
        "all_cases": (rng.uniform(0, 1, (24, 25, 26)).astype(np.float32), 0.5),
        "all_inside": (np.full((5, 6, 7), 3.0, np.float32), 2.0),
        "all_outside": (np.full((5, 6, 7), 1.0, np.float32), 2.0),
        # values exactly at the threshold count as outside
        "at_threshold": (rng.choice(np.float32([19.0, 20.0, 21.0]), (17, 18, 19)), 20.0),
        "threshold_pinf": (rng.normal(0, 1, (9, 10, 11)).astype(np.float32), np.inf),
        "threshold_minf": (rng.normal(0, 1, (9, 10, 11)).astype(np.float32), -np.inf),
        "thin_2_2_2": (rng.normal(0, 1, (2, 2, 2)).astype(np.float32), 0.0),
        "thin_2_2_300": (rng.normal(0, 1, (2, 2, 300)).astype(np.float32), 0.0),
        "thin_300_2_2": (rng.normal(0, 1, (300, 2, 2)).astype(np.float32), 0.0),
        "odd_3_50_7": (rng.normal(0, 1, (3, 50, 7)).astype(np.float32), 0.1),
    }


def _cube_cases(sigma, thr):
    s = sigma.astype(np.float64) > thr
    n0, n1, n2 = s.shape
    cube = np.zeros((n0 - 1, n1 - 1, n2 - 1), np.int64)
    for c in range(8):
        cube |= s[c & 1:n0 - 1 + (c & 1), (c >> 1) & 1:n1 - 1 + ((c >> 1) & 1),
                  (c >> 2) & 1:n2 - 1 + ((c >> 2) & 1)].astype(np.int64) << c
    return set(np.unique(cube).tolist())


def _mc(sigma, thr):
    v, t = _nb().marching_cubes(torch.from_numpy(sigma).cuda(), thr)
    torch.cuda.synchronize()
    return v.cpu().numpy(), t.cpu().numpy()


@pytest.mark.parametrize("name", list(_grids()))
def test_marching_cubes_equals_oracle_and_is_repeatable(name):
    sigma, thr = _grids()[name]
    if name == "all_cases":
        assert _cube_cases(sigma, thr) == set(range(256))
    v, t = _mc(sigma, thr)
    rv, rt = mo.marching_cubes(sigma, thr)
    assert v.dtype == np.float64 and t.dtype == np.int32
    if name in ("all_inside", "all_outside", "threshold_pinf"):
        assert v.shape == (0, 3) and t.shape == (0, 3)
    assert np.array_equal(v, rv)
    assert np.array_equal(t, rt)
    v2, t2 = _mc(sigma, thr)
    assert np.array_equal(v, v2) and np.array_equal(t, t2)


def test_marching_cubes_independent_of_launch_shape(tmp_path):
    sigma, thr = _grids()["torus64"]
    np.save(tmp_path / "s.npy", sigma)
    script = ("import sys, numpy as np, torch; sys.path.insert(0, %r); import nerf_pl_b200 as nb;"
              "s = torch.from_numpy(np.load(%r)).cuda(); v, t = nb.marching_cubes(s, %r);"
              "np.savez(%r, v=v.cpu().numpy(), t=t.cpu().numpy())") % (ROOT, str(tmp_path / "s.npy"), thr,
                                                                      str(tmp_path / "o.npz"))
    env = dict(os.environ, NERFB200_MAX_CTAS="3")
    subprocess.run([sys.executable, "-c", script], check=True, env=env, cwd=ROOT)
    z = np.load(tmp_path / "o.npz")
    v, t = _mc(sigma, thr)
    assert np.array_equal(z["v"], v) and np.array_equal(z["t"], t)


def _closed_manifold(v, t):
    e = np.sort(np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]]), 1)
    _, cnt = np.unique(e, axis=0, return_counts=True)
    assert (cnt == 2).all()
    # each directed edge once: consistent orientation
    d = np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])
    assert len(np.unique(d, axis=0)) == len(d)
    return len(v) - len(cnt) + len(t)


def test_padded_sphere_and_torus_are_closed_with_outward_normals():
    s = _sphere(40, 12.4, (19.3, 20.1, 18.8))
    v, t = _mc(s, 0.0)
    assert _closed_manifold(v, t) == 2
    n = np.cross(v[t[:, 1]] - v[t[:, 0]], v[t[:, 2]] - v[t[:, 0]])
    assert (np.einsum("ij,ij->i", n, v[t].mean(1) - [19.3, 20.1, 18.8]) > 0).all()
    tv, tt = _mc(_torus(64, 18.0, 7.5), 0.0)
    assert _closed_manifold(tv, tt) == 0
    # outward: the normal points away from the tube's core circle
    c = tv[tt].mean(1) - (63 / 2 + 0.17)
    rho = np.hypot(c[:, 0], c[:, 1])
    core = np.stack([c[:, 0] / rho * 18.0, c[:, 1] / rho * 18.0, np.zeros_like(rho)], 1)
    n = np.cross(tv[tt[:, 1]] - tv[tt[:, 0]], tv[tt[:, 2]] - tv[tt[:, 0]])
    assert (np.einsum("ij,ij->i", n, c - core) > 0).all()


def test_largest_cluster_keeps_the_big_sphere():
    n = 48
    s = np.maximum.reduce([_sphere(n, 6.2, (12.3, 12.1, 30.4)), _sphere(n, 10.1, (30.2, 28.7, 22.3)),
                           _sphere(n, 2.3, (8.5, 38.2, 9.1)), _sphere(n, 1.6, (40.4, 8.3, 40.2))])
    v, t = _mc(s, 0.0)
    vw = mo.to_world(v, n, RANGE, RANGE, RANGE)
    kv, kt = _nb().mesh.keep_largest_cluster(torch.from_numpy(vw).cuda(), torch.from_numpy(t).cuda())
    rv, rt = mo.keep_largest_cluster(vw, t)
    assert np.array_equal(kv.cpu().numpy(), rv) and np.array_equal(kt.cpu().numpy(), rt)
    assert _closed_manifold(rv, rt) == 2
    assert len(rt) < len(t)
    # the kept vertices are those of the radius-10.1 sphere (world column 0 holds index axis 1, and back)
    idx = (rv[:, [1, 0, 2]].astype(np.float64) - RANGE[0]) * n / (RANGE[1] - RANGE[0])
    assert np.allclose(np.linalg.norm(idx - [30.2, 28.7, 22.3], axis=1), 10.1, atol=0.5)


def test_grid_positions_and_sigma_grid_bit_exact():
    nb = _nb()
    N, xr, yr, zr = 33, (-1.5, 1.5), (-1.2, 1.4), (-1.5, 1.3)
    pts = nb.mesh.grid_positions(N, xr, yr, zr).cpu().numpy()
    ref = mo.grid_positions(N, xr, yr, zr)
    assert np.array_equal(pts, ref)
    model = _fine_model()
    sig = nb.sigma_grid(model, N, xr, yr, zr, chunk=5000).cpu().numpy()
    q = nb.query_sigma(model, torch.from_numpy(ref).cuda()).cpu().numpy()
    assert np.array_equal(sig, np.maximum(q, 0).reshape(N, N, N))


def test_remap_equals_cv2_fixture(golden_dir):
    d = np.load(os.path.join(golden_dir, "remap_cv2.npz"))
    out = _nb().mesh.remap_bilinear(torch.from_numpy(d["image"]).cuda(), torch.from_numpy(d["xy"]).cuda())
    assert np.array_equal(out.cpu().numpy(), d["out"])


def test_trained_mesh_is_the_union_of_spheres():
    nb = _nb()
    N = 128
    v, t = nb.extract_mesh(_fine_model(), N, RANGE, RANGE, RANGE, 20.0)
    v, t = v.cpu().numpy(), t.cpu().numpy()
    kv, kt = mo.keep_largest_cluster(v, t)
    assert len(kt) == len(t) and len(t) > 1000     # one component (the net leaves small floaters: filtered)
    # undo the reference transform (divide by N, not N - 1): the equal cube ranges make the x/y swap moot
    true = RANGE[0] + (v.astype(np.float64) - RANGE[0]) * N / (N - 1)
    sd = (np.linalg.norm(true[:, None, :] - CENTERS[None], axis=-1) - RADII).min(1)
    d = np.abs(sd)
    print(f"trained mesh: {len(v)} vertices, {len(t)} triangles, |distance to spheres| median {np.median(d):.4f}, "
          f"p99 {np.quantile(d, 0.99):.4f}, max {d.max():.4f}")
    # the bound is what these weights give (H100: median 0.101, p99 0.569, max 0.783).  The gap belongs to the
    # network: the float64 evaluation's 20-level set sits at the same distance (median 0.1016, p99 0.566, max 0.783,
    # tests/test_gpu_mesh_field.py), so this pins the extraction, not the training
    assert np.median(d) < 0.12 and np.quantile(d, 0.99) < 0.6 and d.max() < 0.8


def _look_at(eye):
    eye = np.asarray(eye, np.float64)
    f = -eye / np.linalg.norm(eye)
    r = np.cross(f, [0, 0, 1.0])
    r /= np.linalg.norm(r)
    u = np.cross(r, f)
    return np.stack([r, u, -f, eye], 1)


def _border_vertices(pose, focal, W, H):
    """World points that project onto x = W - 1, beyond the image on each side, closer than near (1.0) and behind
    the camera of ``pose`` (camera looks along -column 2)."""
    c2w = np.asarray(pose, np.float64)
    d = 2.0
    cam = [[((W - 1) - W / 2) * d / focal, 0.0, -d], [(W / 2 + 40) * d / focal, 0.0, -d],
           [-(W / 2 + 40) * d / focal, 0.0, -d], [0.0, (H / 2 + 40) * d / focal, -d], [0.0, -(H / 2 + 3), -d / 20],
           [0.1, 0.1, -0.4], [0.2, -0.1, 1.5]]
    return np.array([c2w[:, :3] @ np.array(c) + c2w[:, 3] for c in cam])


def test_fused_colours_equal_numpy_restatement():
    nb = _nb()
    model = _fine_model()
    v, _ = nb.extract_mesh(model, 64, RANGE, RANGE, RANGE, 20.0)
    n_mesh = v.shape[0]
    focal, near = 70.0, 1.0
    poses = [_look_at(e) for e in ([3.5, 0.4, 0.8], [-1.2, 3.1, -0.6], [0.3, -2.6, 2.4])]
    # even and odd sizes (the principal point on a half pixel), a non-square image
    for H, W in ((60, 80), (61, 81), (45, 97)):
        extra = np.concatenate([_border_vertices(p, focal, W, H) for p in poses]).astype(np.float32)
        vv = torch.cat([v, torch.from_numpy(extra).cuda()])
        yy, xx = np.mgrid[0:H, 0:W]
        images = np.stack([np.stack([(xx * 3 + k * 40) % 256, (yy * 4 + k * 17) % 256, (xx + yy + 60 * k) % 256],
                                    -1) for k in range(3)]).astype(np.uint8)
        cols, opac = nb.fuse_vertex_colors(model, vv, torch.from_numpy(images).cuda(), poses, focal, near,
                                           N_samples=64, return_opacities=True)
        vn, on = vv.cpu().numpy(), opac.cpu().numpy()
        ref = mo.fuse_colors(vn, images, poses, focal, on, 0.2)
        assert np.array_equal(cols.cpu().numpy(), ref)
        # the opacities are render_rays on the device-built rays, and, on the mesh, the oracle's within 1e-3
        emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
        for k in range(len(poses)):
            _, _, rays = nb.mesh.project_view(vv, torch.from_numpy(images[k]).cuda(), poses[k], focal, near)
            with torch.no_grad():
                r = nb.render_rays([model], emb, rays, 64, False, 0, 0, 0, 32768, False, test_time=True,
                                   match_reference_rng=False)["opacity_coarse"]
            assert torch.equal(r, opac[k])
            sel = np.arange(0, n_mesh, max(1, n_mesh // 1500))
            o = orc.render_rays([cases.trained_weights()[1]], rays.cpu().numpy()[sel], 64, False, 0.0, 0.0, 0, False,
                                True)
            assert np.abs(o["opacity_coarse"] - on[k][sel]).max() < 1e-3


def test_write_ply_roundtrip(tmp_path):
    v = np.random.default_rng(0).normal(size=(5, 3)).astype(np.float32)
    t = np.array([[0, 1, 2], [2, 3, 4]], np.int32)
    c = np.arange(15, dtype=np.uint8).reshape(5, 3)
    path = str(tmp_path / "m.ply")
    _nb().write_ply(path, v, t, c)
    raw = open(path, "rb").read()
    head, body = raw.split(b"end_header\n")
    assert b"element vertex 5" in head and b"property list uchar int vertex_indices" in head
    vert = np.frombuffer(body[:5 * 15], dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("r", "u1"), ("g", "u1"),
                                               ("b", "u1")])
    assert np.array_equal(vert["x"], v[:, 0]) and np.array_equal(vert["b"], c[:, 2])
    face = np.frombuffer(body[5 * 15:], dtype=[("n", "u1"), ("i", "<i4", (3,))])
    assert np.array_equal(face["i"], t) and (face["n"] == 3).all()
