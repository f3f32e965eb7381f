"""The sigma field of mesh extraction against float64, and marching cubes / the cluster filter / colour
accumulation at their edges.

A. The two sigma paths (``NeRF.forward(.., sigma_only=True)`` and ``query_sigma`` / ``sigma_grid``) equal the
   pinned full forward bit for bit (the in-kernel encoding up to the fp16 roundings it may legitimately pick,
   tests/sigma_ref.py).
B. The trained network's extracted surface is its own sigma = threshold level set: device sigma against float64
   within multiples of the fp16 replay's error, and the level set's distance to the analytic spheres.
C. marching_cubes and keep_largest_cluster against oracle/mesh_oracle.py on degenerate grids and meshes, at both
   launch shapes.
D. The colour accumulation with NaN opacities and opacities exactly at the occlusion threshold.
"""
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as mo
from oracle import nerf_oracle as orc
from tests import cases
from tests import sigma_ref as sr

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CENTERS = np.array([[0.0, 0.0, 0.0], [0.9, 0.3, -0.2], [-0.6, -0.7, 0.4]])
RADII = np.array([0.8, 0.45, 0.55])
CUBE = ((-1.5, 1.5),) * 3
UNEQUAL = ((-1.5, 1.5), (-1.2, 1.4), (-1.5, 1.3))
REVERSED = ((1.5, -1.5), (-1.2, 1.4), (1.3, -1.5))
THR = 20.0


def _nb():
    import nerf_pl_b200 as nb
    return nb


def _weights(kind):
    return cases.trained_weights()[1] if kind == "trained" else orc.make_weights(11)


_MODELS = {}


def _model(kind):
    if kind not in _MODELS:
        m = _nb().NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in _weights(kind).items()})
        _MODELS[kind] = m.cuda().eval()
    return _MODELS[kind]


def _lib():
    return _nb()._lib.load()


def _stream():
    from nerf_pl_b200.nerf import _stream_ptr
    return _stream_ptr()


def _blob(model):
    from nerf_pl_b200.nerf import packed_weights
    return packed_weights(model)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------- A
@pytest.mark.parametrize("kind", ["random", "trained"])
@pytest.mark.parametrize("B", [1, 127, 128, 129, 132 * 128 - 1, 132 * 128 + 1, (1 << 21) + 5])
def test_sigma_only_forward_is_column_3_of_the_full_forward(kind, B):
    model = _model(kind)
    g = torch.Generator(device="cuda").manual_seed(B)
    x = torch.rand(B, 90, device="cuda", generator=g) * 2 - 1
    with torch.no_grad():
        full = model(x)
        so = model(x[:, :63], sigma_only=True)
    assert so.shape == (B, 1)
    assert torch.equal(_bits(so[:, 0]), _bits(full[:, 3]))
    # the C ABI reading the 63 xyz columns of the 90-wide rows in place (extract_color_mesh.py's layout)
    out = torch.full((B,), float("nan"), device="cuda")
    _nb()._lib.check(_lib().nerfb200_nerf_forward(x.data_ptr(), B, 90, _blob(model).data_ptr(), 1, out.data_ptr(),
                                                  _stream()), "nerfb200_nerf_forward")
    assert torch.equal(_bits(out), _bits(full[:, 3]))


def _points(name):
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    if name == "uniform":
        return rng.uniform(-1.5, 1.5, (60000, 3)).astype(np.float32)
    if name == "wide":
        p = rng.uniform(-61, 61, (20000, 3))
        p[:6] = [[61, -61, 0], [-61, 61, 61], [60.99, -0.0, 1e-30], [0, 0, 0], [-0.0, -0.0, -0.0], [1e-7, -1e-7, 3]]
        return p.astype(np.float32)
    if name == "grid":
        parts = [mo.grid_positions(n, *r) for n, r in ((17, UNEQUAL), (17, REVERSED), (33, CUBE), (2, UNEQUAL))]
        p = np.concatenate(parts)
        neg = p.copy()
        neg[p == 0] = -0.0
        return np.concatenate([p, neg[(p == 0).any(1)]]).astype(np.float32)
    n = {"n1": 1, "n127": 127, "n129": 129, "n_sms_minus": _sms() * 128 - 1, "n_sms_plus": _sms() * 128 + 1,
         "n_two_rounds": 2 * _sms() * 128 + 77}[name]
    return rng.uniform(-1.5, 1.5, (n, 3)).astype(np.float32)


@pytest.mark.parametrize("name", ["uniform", "wide", "grid", "n1", "n127", "n129", "n_sms_minus", "n_sms_plus",
                                  "n_two_rounds"])
def test_query_sigma_equals_forward_on_the_fp16_encoding(name):
    nb = _nb()
    model = _model("trained")
    xyz = _points(name)
    dev = nb.query_sigma(model, torch.from_numpy(xyz).cuda()).cpu().numpy()
    rows, owner, choices = sr.candidate_encodings(xyz)
    with torch.no_grad():
        cand = model(torch.from_numpy(rows).cuda(), sigma_only=True)[:, 0].cpu().numpy()
    n = len(xyz)
    included = choices <= sr.MAX_ROUNDINGS
    hit = sr.matches_a_rounding(dev, cand, owner, n)
    exact = choices == 1
    print(f"\nquery_sigma {name}: {n} points, {int(exact.sum())} unambiguous, {int((included & ~exact).sum())} with "
          f"2-16 roundings, {int((~included).sum())} excluded (more than 16 roundings)")
    assert hit[exact].all(), np.nonzero(exact & ~hit)[0][:10]
    assert hit[included].all(), np.nonzero(included & ~hit)[0][:10]
    assert included.mean() > 0.8


def test_query_sigma_reads_xyz_with_a_row_stride():
    model = _model("trained")
    n = 3 * 128 * _sms() + 5
    rays = torch.rand(n, 8, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5)) * 3 - 1.5
    out = torch.full((n,), float("nan"), device="cuda")
    _nb()._lib.check(_lib().nerfb200_query_sigma(rays.data_ptr(), n, 8, _blob(model).data_ptr(), out.data_ptr(),
                                                 _stream()), "nerfb200_query_sigma")
    ref = _nb().query_sigma(model, rays[:, :3].contiguous())
    assert torch.equal(_bits(out), _bits(ref))


@pytest.mark.parametrize("N", [2, 17, 33])
@pytest.mark.parametrize("ranges", [CUBE, UNEQUAL, REVERSED], ids=["cube", "unequal", "reversed"])
def test_sigma_grid_equals_relu_of_query_sigma_for_every_chunk(N, ranges):
    nb = _nb()
    model = _model("trained")
    pts = nb.mesh.grid_positions(N, *ranges)
    assert np.array_equal(pts.cpu().numpy(), mo.grid_positions(N, *ranges))
    q = nb.query_sigma(model, pts).cpu().numpy()
    for chunk in (127, 128, 129, 4999, N ** 3 - 1, N ** 3):
        grid = nb.sigma_grid(model, N, *ranges, chunk=chunk).cpu().numpy()
        assert sr.grid_mismatches(grid, q, N) == 0, chunk


# ---------------------------------------------------------------------------------------------- B
def _sphere_distance(world):
    return np.abs((np.linalg.norm(world[:, None, :] - CENTERS[None], axis=-1) - RADII).min(1))


def _dist_stats(d):
    return {"median": float(np.median(d)), "p99": float(np.quantile(d, 0.99)), "max": float(d.max())}


@pytest.mark.parametrize("ranges", [CUBE, UNEQUAL], ids=["cube", "unequal"])
def test_trained_surface_is_the_networks_level_set(ranges):
    nb = _nb()
    N = 128
    w = _weights("trained")
    model = _model("trained")
    grid = nb.sigma_grid(model, N, *ranges)
    v_dev, _ = nb.marching_cubes(grid, THR)
    dev = grid.cpu().numpy().reshape(-1).astype(np.float64)
    v_dev = v_dev.cpu().numpy()
    pts = mo.grid_positions(N, *ranges)
    s64 = np.maximum(sr.sigma64(w, pts, device="cuda"), 0)
    rep = np.maximum(sr.sigma_fp16_replay(w, pts, device="cuda"), 0)
    # points on a sign-changing edge of either field, and all the others
    _, ends_dev = sr.crossings(dev.reshape(N, N, N), THR)
    pos64, ends64 = sr.crossings(s64.reshape(N, N, N), THR)
    near = np.zeros(N ** 3, bool)
    near[ends_dev.ravel()] = True
    near[ends64.ravel()] = True
    print(f"\nlevel set {ranges}: {len(v_dev)} device crossings, {len(pos64)} float64 crossings, "
          f"{int(near.sum())} edge endpoints, {int((~near).sum())} other grid points")
    for what, m in (("edge endpoints", near), ("off the surface", ~near)):
        r = sr.field_report(dev[m], s64[m], rep[m], THR)
        print(f"  {what}: device |sigma - float64| max {r['dev']['max']:.4g} p99 {r['dev']['p99']:.4g} "
              f"mean {r['dev']['mean']:.4g}; fp16 replay max {r['replay']['max']:.4g} p99 {r['replay']['p99']:.4g} "
              f"mean {r['replay']['mean']:.4g}; points classified unlike float64 {r['flips']} "
              f"(largest |sigma64 - thr| {r['flip_gap']:.4g}, bar {r['bars']['max']:.4g})")
        assert all(r["ok"].values()), r
    key = lambda e: e[:, 0] * 3 + np.where(e[:, 1] - e[:, 0] == 1, 2, np.where(e[:, 1] - e[:, 0] == N, 1, 0))
    k_dev, k64 = set(key(ends_dev).tolist()), set(key(ends64).tolist())
    print(f"  edges whose sign change differs from float64: {len(k_dev ^ k64)}")
    # the float64 level set and the mesh sit at the same distance from the analytic spheres
    d_dev = _sphere_distance(sr.index_to_world(v_dev, N, *ranges))
    d64 = _sphere_distance(sr.index_to_world(pos64, N, *ranges))
    s_dev, s64d = _dist_stats(d_dev), _dist_stats(d64)
    print(f"  distance to the analytic spheres: mesh {s_dev}, float64 level set {s64d}")
    assert abs(s_dev["median"] - s64d["median"]) < 2e-3
    assert abs(s_dev["p99"] - s64d["p99"]) < 1e-2
    assert abs(s_dev["max"] - s64d["max"]) < 2e-2


# ---------------------------------------------------------------------------------------------- C
def _mc(sigma, thr):
    v, t = _nb().marching_cubes(torch.from_numpy(np.ascontiguousarray(sigma)).cuda(), thr)
    torch.cuda.synchronize()
    return v.cpu().numpy(), t.cpu().numpy()


def _special_grids():
    rng = np.random.default_rng(21)
    g = rng.normal(0, 1, (20, 21, 22)).astype(np.float32)
    inf = g.copy()
    inf.ravel()[rng.choice(inf.size, 600, replace=False)] = np.inf
    inf.ravel()[rng.choice(inf.size, 300, replace=False)] = -np.inf
    nan = inf.copy()
    nan.ravel()[rng.choice(nan.size, 700, replace=False)] = np.nan
    allnan = np.full((5, 6, 7), np.nan, np.float32)
    return {"inf": inf, "nan": nan, "all_nan": allnan}


@pytest.mark.parametrize("name", ["inf", "nan", "all_nan"])
@pytest.mark.parametrize("thr", [0.2, np.inf, -np.inf, 0.0])
def test_marching_cubes_with_inf_and_nan_entries(name, thr):
    sigma = _special_grids()[name]
    v, t = _mc(sigma, thr)
    rv, rt = mo.marching_cubes(sigma, thr)
    assert v.dtype == np.float64 and t.dtype == np.int32 and v.shape[1:] == (3,) and t.shape[1:] == (3,)
    assert np.array_equal(v, rv, equal_nan=True)
    assert np.array_equal(t, rt)
    # NaN is outside
    inside = sigma.astype(np.float64) > thr
    assert not inside[np.isnan(sigma)].any()
    if name == "nan" and np.isfinite(thr):
        assert len(v) > 0 and np.isnan(v).any()


def _mesh_case(v, t):
    return np.ascontiguousarray(v, np.float32), np.ascontiguousarray(t, np.int32)


def _tet(o):
    return np.array([[0, 1, 2], [0, 3, 1], [0, 2, 3], [1, 3, 2]]) + o


def _soup(V, rng, T=300, pool=48):
    idx = np.concatenate([np.arange(pool), np.arange(V - pool, V)])
    t = rng.choice(idx, (T, 3))
    t = t[(t[:, 0] != t[:, 1]) & (t[:, 1] != t[:, 2]) & (t[:, 0] != t[:, 2])]
    return np.concatenate([t, [[V - 3, V - 2, V - 1], [V - 1, V - 2, 0]]])


def _cluster_cases(trained_v, trained_t, noise_v, noise_t):
    rng = np.random.default_rng(8)
    rv = lambda V: rng.normal(size=(V, 3))
    c = {
        "trained_256": (trained_v, trained_t),
        "noise_components": (noise_v, noise_t),
        "isolated_triangles": (rv(3000), np.arange(3000).reshape(1000, 3)),
        "equal_pair_reversed": (rv(8), np.concatenate([_tet(4), _tet(0)])),
        "nonmanifold_edge": (rv(14), np.array([[10, 11, 12], [11, 12, 13], [0, 1, 2], [1, 0, 3], [0, 1, 4],
                                               [1, 4, 6]])),
        "duplicates": (rv(9), np.array([[5, 6, 7], [5, 7, 8], [0, 1, 2], [0, 1, 2], [2, 1, 0], [2, 1, 3]])),
        "unreferenced_between": (rv(30), np.array([[3, 5, 7], [5, 7, 9], [20, 22, 24], [7, 9, 11]])),
        "single": (rv(3), np.array([[0, 1, 2]])),
        "single_high": (rv(10), np.array([[7, 2, 9]])),
    }
    for k in (1, 10, 16, 20):
        for V in (1 << k, (1 << k) + 1):
            if V < 4:
                c[f"V_{V}"] = (rv(V), np.array([[0, 1, V - 1]])) if V == 3 else (rv(V), np.array([[0, V - 1, 1 % V]]))
                continue
            c[f"V_{V}"] = (rv(V), _soup(V, rng))
    return {k: _mesh_case(*v) for k, v in c.items()}


_SUBPROCESS = r"""
import sys
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
import nerf_pl_b200 as nb
z = np.load(sys.argv[2])
out = {}
v, t = nb.marching_cubes(torch.from_numpy(z["grid"]).cuda(), float(z["thr"]))
out["mc_v"], out["mc_t"] = v.cpu().numpy(), t.cpu().numpy()
for name in [k[2:] for k in z.files if k.startswith("v_")]:
    kv, kt = nb.mesh.keep_largest_cluster(torch.from_numpy(z["v_" + name]).cuda(), torch.from_numpy(z["t_" + name]).cuda())
    out["kv_" + name], out["kt_" + name] = kv.cpu().numpy(), kt.cpu().numpy()
np.savez(sys.argv[3], **out)
"""


@pytest.fixture(scope="module")
def scale_cases(tmp_path_factory):
    """The trained N = 256 grid and its unfiltered mesh, a noise mesh, the hand-built meshes, and what a
    NERFB200_MAX_CTAS=1 process computes from them."""
    nb = _nb()
    N = 256
    grid = nb.sigma_grid(_model("trained"), N, *CUBE).cpu().numpy()
    v, t = _mc(grid, THR)
    vw = mo.to_world(v, N, *CUBE)
    noise = np.random.default_rng(9).uniform(0, 1, (48, 48, 48)).astype(np.float32)
    nv, nt = _mc(noise, 0.97)      # 3,043 components, the four largest of equal size
    meshes = _cluster_cases(vw, t, mo.to_world(nv, 48, *CUBE), nt)
    d = tmp_path_factory.mktemp("mesh_field")
    arrays = {"grid": grid, "thr": np.float64(THR)}
    for k, (mv, mt) in meshes.items():
        arrays["v_" + k], arrays["t_" + k] = mv, mt
    np.savez(d / "in.npz", **arrays)
    env = dict(os.environ, NERFB200_MAX_CTAS="1")
    subprocess.run([sys.executable, "-c", _SUBPROCESS, ROOT, str(d / "in.npz"), str(d / "out.npz")], check=True,
                   env=env, cwd=ROOT)
    return {"grid": grid, "mc": (v, t), "meshes": meshes, "one_cta": dict(np.load(d / "out.npz"))}


def test_marching_cubes_on_the_trained_256_grid(scale_cases):
    grid = scale_cases["grid"]
    v, t = scale_cases["mc"]
    rv, rt = mo.marching_cubes(grid, THR)
    print(f"\ntrained N=256 mesh: {len(v)} vertices, {len(t)} triangles")
    assert len(v) > 250_000
    assert np.array_equal(v, rv) and np.array_equal(t, rt)
    one = scale_cases["one_cta"]
    assert np.array_equal(one["mc_v"], v) and np.array_equal(one["mc_t"], t)
    v2, t2 = _mc(grid, THR)
    assert np.array_equal(v2, v) and np.array_equal(t2, t)


def _components(t):
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    t = t.astype(np.int64)
    e = np.sort(np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]]), 1)
    tid = np.tile(np.arange(len(t)), 3)
    o = np.lexsort((e[:, 1], e[:, 0]))
    e, tid = e[o], tid[o]
    same = (e[1:] == e[:-1]).all(1)
    g = coo_matrix((np.ones(int(same.sum())), (tid[1:][same], tid[:-1][same])), shape=(len(t), len(t)))
    _, lab = connected_components(g, directed=False)
    return np.bincount(lab)


CLUSTER_NAMES = ["trained_256", "noise_components", "isolated_triangles", "equal_pair_reversed", "nonmanifold_edge",
                 "duplicates", "unreferenced_between", "single", "single_high", "V_2", "V_3", "V_1024", "V_1025",
                 "V_65536", "V_65537", "V_1048576", "V_1048577"]


@pytest.mark.parametrize("name", CLUSTER_NAMES)
def test_largest_cluster_equals_scipy_at_its_edges(scale_cases, name):
    v, t = scale_cases["meshes"][name]
    sizes = _components(t)
    top = np.sort(sizes)[::-1]
    print(f"\ncluster {name}: V {len(v)}, T {len(t)}, {len(sizes)} components, largest {top[:3].tolist()}, "
          f"{int((sizes == top[0]).sum())} of the largest size")
    rv, rt = mo.keep_largest_cluster(v, t)
    runs = []
    for _ in range(2):
        kv, kt = _nb().mesh.keep_largest_cluster(torch.from_numpy(v).cuda(), torch.from_numpy(t).cuda())
        runs.append((kv.cpu().numpy(), kt.cpu().numpy()))
    for kv, kt in runs:
        assert np.array_equal(kv, rv) and np.array_equal(kt, rt)
    one = scale_cases["one_cta"]
    assert np.array_equal(one["kv_" + name], rv) and np.array_equal(one["kt_" + name], rt)
    if name == "isolated_triangles":
        assert np.array_equal(rt, [[0, 1, 2]]) and np.array_equal(rv, v[:3])
    if name == "equal_pair_reversed":                 # the component listed first holds triangle 0
        assert np.array_equal(rv, v[4:8])
    if name == "noise_components":
        assert len(sizes) > 1000 and (sizes == top[0]).sum() > 1


# ---------------------------------------------------------------------------------------------- D
def _look_at(eye):
    eye = np.asarray(eye, np.float64)
    f = -eye / np.linalg.norm(eye)
    r = np.cross(f, [0, 0, 1.0])
    r /= np.linalg.norm(r)
    u = np.cross(r, f)
    return np.stack([r, u, -f, eye], 1)


def test_colour_accumulate_nan_and_threshold_opacities():
    nb = _nb()
    lib = _lib()
    rng = np.random.default_rng(12)
    H, W, focal, near, occ = 45, 97, 70.0, 1.0, 0.2
    eyes = np.array([[3.5, 0.4, 0.8], [-1.2, 3.1, -0.6], [0.3, -2.6, 2.4]])
    poses = [_look_at(e) for e in eyes]
    # behind the first camera, closer than near, and far outside the image on both sides
    side = poses[0][:, 0]
    extra = [eyes[0] * 1.3, eyes[0] * 0.8, eyes[0] * 0.5 + 40 * side, eyes[0] * 0.5 - 40 * side,
             eyes[0] * 0.5 + 40 * poses[0][:, 1]]
    v = np.concatenate([rng.uniform(-1, 1, (5000, 3)), extra]).astype(np.float32)
    images = rng.integers(0, 256, (3, H, W, 3), dtype=np.uint8)
    t32 = np.float32(occ)
    special = np.array([np.nan, t32, np.nextafter(t32, np.float32(0)), np.nextafter(t32, np.float32(1)), 0.0, 1.0,
                        -0.0, np.inf, -np.inf], np.float32)
    opac = rng.uniform(0, 0.4, (3, len(v))).astype(np.float32)
    for k in range(3):
        idx = rng.choice(len(v), 2000, replace=False)
        opac[k, idx] = special[rng.integers(0, len(special), 2000)]
    vt = torch.from_numpy(v).cuda()
    sum4 = torch.zeros(len(v), 4, dtype=torch.float64, device="cuda")
    for k in range(3):
        colors, depth, _ = nb.mesh.project_view(vt, torch.from_numpy(images[k]).cuda(), poses[k], focal, near)
        o = torch.from_numpy(opac[k]).cuda()
        nb._lib.check(lib.nerfb200_color_accumulate(colors.data_ptr(), depth.data_ptr(), o.data_ptr(), len(v),
                                                    float(t32), sum4.data_ptr(), _stream()), "color_accumulate")
    out = torch.empty(len(v), 3, dtype=torch.uint8, device="cuda")
    nb._lib.check(lib.nerfb200_color_finalize(sum4.data_ptr(), len(v), out.data_ptr(), _stream()), "color_finalize")
    ref = mo.fuse_colors(v, images, poses, focal, opac, occ)
    assert np.array_equal(out.cpu().numpy(), ref)
