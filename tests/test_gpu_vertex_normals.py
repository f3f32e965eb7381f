"""The vertex-normal colouring method on the device (nerf_pl_b200.mesh.vertex_normals / normal_rays /
normal_vertex_colors): open3d's vertex normals bit for bit against the numpy restatement (tests/normals_ref.py), the
rays bit for bit against the reference's torch expression, the colours against the fused renderer and against the
unmodified reference (tests/golden/vertex_normal_colors.part*.npz)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import cases, normals_ref as nr, npz_parts
from tests.test_gpu_mesh import _grids

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
RANGE = (-1.5, 1.5)


def _nb():
    import nerf_pl_b200 as nb
    return nb


def _model(tag):
    m = _nb().NeRF()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in cases.trained_weights()[tag == "fine"].items()})
    return m.cuda().eval()


def _soup(V, T, seed):
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(V, 3)).astype(np.float32)
    t = rng.integers(0, V, (T, 3)).astype(np.int32)
    t[: T // 10, 1] = t[: T // 10, 0]          # some degenerate corners
    return v, t


@pytest.fixture(scope="module")
def meshes():
    """name -> (vertices (V, 3) float32, triangles (T, 3) int32) on the host."""
    nb = _nb()
    out = {}
    v, t = nb.extract_mesh(_model("fine"), 128, RANGE, RANGE, RANGE, 20.0)
    out["trained128"] = (v.cpu().numpy(), t.cpu().numpy())
    for name, (sigma, thr) in _grids().items():
        vi, ti = nb.marching_cubes(torch.from_numpy(sigma).cuda(), thr)
        out[f"mc_{name}"] = (vi.cpu().numpy().astype(np.float32), ti.cpu().numpy())
    for name, (hv, ht, _) in nr.hand_meshes().items():
        out[f"hand_{name}"] = (hv, ht)
    out["soup_2p20"] = _soup(2 ** 20 + 3, 2 ** 21 + 1, 5)
    return out


def _device_normals(v, t):
    return _nb().vertex_normals(torch.from_numpy(v).cuda(), torch.from_numpy(t).cuda()).cpu().numpy()


MESH_NAMES = ["trained128"] + [f"mc_{n}" for n in _grids()] + [f"hand_{n}" for n in nr.hand_meshes()] + ["soup_2p20"]


@pytest.mark.parametrize("name", MESH_NAMES)
def test_vertex_normals_equal_the_restatement_bit_for_bit(meshes, name):
    v, t = meshes[name]
    n = _device_normals(v, t)
    assert n.dtype == np.float64 and n.shape == (len(v), 3)
    assert nr.same_bits(n, nr.vertex_normals(v, t))
    assert nr.same_bits(n, _device_normals(v, t))      # repeatable
    if name.startswith("hand_") and nr.hand_meshes()[name[5:]][2] is not None:
        assert nr.same_bits(n, nr.hand_meshes()[name[5:]][2])


def test_vertex_normals_do_not_depend_on_the_launch_shape(meshes, tmp_path):
    np.savez(tmp_path / "m.npz", **{f"{k}.v": v for k, (v, t) in meshes.items()},
             **{f"{k}.t": t for k, (v, t) in meshes.items()})
    script = ("import sys, numpy as np, torch; sys.path.insert(0, %r); import nerf_pl_b200 as nb;"
              "z = np.load(%r); names = sorted({k[:-2] for k in z.files});"
              "out = {k: nb.vertex_normals(torch.from_numpy(z[k + '.v']).cuda(), torch.from_numpy(z[k + '.t']).cuda())"
              ".cpu().numpy() for k in names}; np.savez(%r, **out)") % (ROOT, str(tmp_path / "m.npz"),
                                                                       str(tmp_path / "o.npz"))
    subprocess.run([sys.executable, "-c", script], check=True, env=dict(os.environ, NERFB200_MAX_CTAS="1"), cwd=ROOT)
    one = np.load(tmp_path / "o.npz")
    assert sorted(one.files) == sorted(meshes)
    for name, (v, t) in meshes.items():
        assert nr.same_bits(one[name], _device_normals(v, t)), name


def test_no_triangles_gives_zero_normals_and_empty_meshes_work():
    nb = _nb()
    v = torch.randn(7, 3, device="cuda")
    n = nb.vertex_normals(v, torch.zeros(0, 3, dtype=torch.int32, device="cuda"))
    assert n.shape == (7, 3) and n.dtype == torch.float64 and not n.any()
    e = nb.vertex_normals(v[:0], torch.zeros(0, 3, dtype=torch.int64, device="cuda"))
    assert e.shape == (0, 3)
    assert nb.normal_rays(v[:0], e, 2.0, 6.0).shape == (0, 8)


@pytest.mark.parametrize("bad", [-1, 9, 2 ** 31 - 1, 2 ** 32 + 1, -2 ** 40])
def test_out_of_range_indices_raise_and_the_next_call_works(bad):
    nb = _nb()
    v, t = nr.hand_meshes()["cube"][:2]
    vd = torch.from_numpy(v).cuda()
    tt = torch.from_numpy(t).to(torch.int64)
    tt[5, 2] = bad
    if -2 ** 31 <= bad < 2 ** 31:
        with pytest.raises(ValueError, match="outside"):
            nb.vertex_normals(vd, tt.to(torch.int32).cuda())
    with pytest.raises(ValueError, match="outside"):
        nb.vertex_normals(vd, tt.cuda())
    assert nr.same_bits(nb.vertex_normals(vd, torch.from_numpy(t).cuda()).cpu().numpy(), nr.vertex_normals(v, t))


def test_argument_errors():
    nb = _nb()
    v = torch.randn(4, 3, device="cuda")
    t = torch.tensor([[0, 1, 2]], dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError):
        nb.vertex_normals(v.cpu(), t)
    with pytest.raises(RuntimeError):
        nb.vertex_normals(v, t.cpu())
    with pytest.raises(ValueError):
        nb.vertex_normals(v[:, :2], t)
    with pytest.raises(ValueError):
        nb.vertex_normals(v, t.float())
    with pytest.raises(ValueError):
        nb.vertex_normals(v.to(torch.int32), t)
    with pytest.raises(ValueError):
        nb.normal_rays(v, torch.zeros(3, 3, dtype=torch.float64, device="cuda"), 2.0, 6.0)
    with pytest.raises(RuntimeError):
        nb.normal_rays(v, torch.zeros(4, 3, dtype=torch.float64), 2.0, 6.0)
    coarse, fine = _model("coarse"), _model("fine")
    with pytest.raises(ValueError):
        nb.normal_vertex_colors(coarse, fine, v, t, 2.0, 6.0, N_importance=0)
    with pytest.raises(RuntimeError):
        nb.normal_vertex_colors(coarse.cpu(), fine, v, t, 2.0, 6.0)


def test_orientation_on_exact_geometry():
    """sphere48 (inside: sigma > 0): in index space every vertex normal with a nonzero sum points away from the
    centre; through the reference's world transform (which swaps x and y, a reflection) every one points towards it."""
    nb = _nb()
    sigma, thr = _grids()["sphere48"]
    centre = np.array([23.2, 24.7, 22.9])
    vi, t = nb.marching_cubes(torch.from_numpy(sigma).cuda(), thr)
    n_idx = nb.vertex_normals(vi, t).cpu().numpy()
    nz = np.linalg.norm(n_idx, axis=1) > 0
    assert nz.mean() > 0.99
    vi32 = vi.cpu().numpy().astype(np.float32).astype(np.float64)
    assert (np.einsum("ij,ij->i", n_idx, vi32 - centre)[nz] > 0).all()
    vw = nb.mesh.to_world(vi, 48, RANGE, RANGE, RANGE)
    n_w = nb.vertex_normals(vw, t).cpu().numpy()
    nzw = np.linalg.norm(n_w, axis=1) > 0
    c_w = np.array([centre[1], centre[0], centre[2]]) / 48 * (RANGE[1] - RANGE[0]) + RANGE[0]
    assert (np.einsum("ij,ij->i", n_w, vw.cpu().numpy().astype(np.float64) - c_w)[nzw] < 0).all()


def _fixture():
    z = npz_parts.load(GOLDEN, "vertex_normal_colors")
    return z, json.loads(str(z["meta"]))


@pytest.mark.parametrize("bounds, near_t", [((2.0, 6.0), 1.0), ((1.7, 6.1), 1.1), ((0.1, 1e3), 2.5),
                                            ((0.3, 4.7), 0.9), ((2.0, 6.0), 1e-3)])
def test_normal_rays_equal_the_torch_expression(bounds, near_t):
    nb = _nb()
    z, _ = _fixture()
    v, n = z["vertices"], z["blender.normals"]
    rays = nb.normal_rays(torch.from_numpy(v).cuda(), torch.from_numpy(n).cuda(), min(bounds), max(bounds), near_t)
    ref = nr.normal_rays_torch(v, n, np.array(bounds), near_t)
    assert np.array_equal(rays.cpu().numpy().view(np.uint32), ref.view(np.uint32))


def test_to_uint8_equals_numpy_on_every_float_in_0_1():
    """``(rgb * 255.0).astype(uint8)`` for every float32 in [0, 1] (the colours step of :281-284); outside it the
    kernel clamps (> 1 and +inf -> 255, < 0, -inf and NaN -> 0), where numpy's cast is undefined."""
    nb = _nb()
    top = int(np.float32(1.0).view(np.int32))
    step = 1 << 27
    for lo in range(0, top + 1, step):
        bits = torch.arange(lo, min(lo + step, top + 1), dtype=torch.int32, device="cuda")
        x = bits.view(torch.float32)
        assert torch.equal(nb.to_uint8(x), (x * 255.0).to(torch.uint8)), lo
    spot = np.float32([0.0, 0.5, 1 / 255, 0.99999994, 1.0])
    assert np.array_equal(nb.to_uint8(torch.from_numpy(spot).cuda()).cpu().numpy(), (spot * 255.0).astype(np.uint8))
    odd = torch.tensor([1.5, 1.0000001, -0.5, float("nan"), float("inf"), -float("inf")], device="cuda")
    assert nb.to_uint8(odd).tolist() == [255, 255, 0, 0, 255, 0]


@pytest.mark.parametrize("K, white_back, near_t", [(64, True, 1.0), (128, False, 1.1), (64, False, 0.8),
                                                   (128, True, 1.0)])
def test_colours_are_the_fused_render_of_the_normal_rays(K, white_back, near_t):
    nb = _nb()
    coarse, fine = _model("coarse"), _model("fine")
    v, t = nb.extract_mesh(fine, 64, RANGE, RANGE, RANGE, 20.0)
    cols = nb.normal_vertex_colors(coarse, fine, v, t, 2.0, 6.0, N_importance=K, near_t=near_t, white_back=white_back)
    rays = nb.normal_rays(v, nb.vertex_normals(v, t), 2.0, 6.0, near_t)
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    with torch.no_grad():
        res = nb.render_rays([coarse, fine], emb, rays, 64, False, 0, 0, K, 32768, white_back, test_time=True,
                             match_reference_rng=False)
    assert cols.dtype == torch.uint8 and cols.shape == (v.shape[0], 3)
    assert torch.equal(cols, nb.to_uint8(res["rgb_fine"]))
    assert torch.equal(cols, (res["rgb_fine"] * 255.0).to(torch.uint8))


# max / p99 / mean |rgb_fine - reference| on the fixture's rays (DESIGN.md section 9, "Vertex-normal colours")
RGB_BARS = {"max": 1e-3, "p99": 1e-3, "mean": 1e-4}


@pytest.mark.parametrize("name", ["blender", "inexact"])
def test_against_the_reference_fixture(name):
    nb = _nb()
    z, meta = _fixture()
    c = meta["cases"][name]
    v, t = torch.from_numpy(z["vertices"]).cuda(), torch.from_numpy(z["triangles"]).cuda()
    n = nb.vertex_normals(v, t)
    assert nr.same_bits(n.cpu().numpy(), z[f"{name}.normals"])
    near, far = min(c["bounds"]), max(c["bounds"])
    rays = nb.normal_rays(v, n, near, far, c["near_t"])
    assert np.array_equal(rays.cpu().numpy().view(np.uint32), z[f"{name}.rays"].view(np.uint32))
    coarse, fine = _model("coarse"), _model("fine")
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    with torch.no_grad():
        rgb = nb.render_rays([coarse, fine], emb, rays, c["N_samples"], False, 0, 0, c["N_importance"], 32768,
                             c["white_back"], test_time=True, match_reference_rng=False)["rgb_fine"].cpu().numpy()
    cols = nb.normal_vertex_colors(coarse, fine, v, t, near, far, c["N_samples"], c["N_importance"], c["near_t"],
                                   c["white_back"]).cpu().numpy()
    assert np.array_equal(cols, (rgb * np.float32(255.0)).astype(np.uint8))
    e = np.abs(rgb - z[f"{name}.rgb_fine"])
    stats = {"max": float(e.max()), "p99": float(np.quantile(e, 0.99)), "mean": float(e.mean())}
    diff = cols.astype(np.int32) - z[f"{name}.colors"]
    print(f"{name}: |rgb_fine - reference| max {stats['max']:.3g} p99 {stats['p99']:.3g} mean {stats['mean']:.3g}; "
          f"colour bytes differing {np.mean(diff != 0):.4f} (by 1: {np.mean(np.abs(diff) == 1):.4f}, "
          f"max |diff| {np.abs(diff).max()})")
    for k, bar in RGB_BARS.items():
        assert stats[k] <= bar, (k, stats)
    assert np.abs(diff).max() <= 1


def test_trained_colours_match_the_analytic_scene():
    """On the N_grid 128 mesh, the colours against the scene the weights were trained on (tools/train_sharp_weights.py
    ``ground_truth``, on the same rays with the reference's divide-by-N transform undone)."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from train_sharp_weights import ground_truth
    nb = _nb()
    coarse, fine = _model("coarse"), _model("fine")
    N = 128
    v, t = nb.extract_mesh(fine, N, RANGE, RANGE, RANGE, 20.0)
    cols = nb.normal_vertex_colors(coarse, fine, v, t, 2.0, 6.0, white_back=True).float() / 255.0
    n = nb.vertex_normals(v, t).float()
    true = RANGE[0] + (v - RANGE[0]) * (N / (N - 1))
    rays = torch.cat([true - n * 2.0, n, torch.tensor([[2.0, 6.0]], device="cuda").expand(n.shape[0], 2)], 1)
    gt = torch.cat([ground_truth(rays[i:i + 8192]) for i in range(0, rays.shape[0], 8192)])
    err = (cols - gt).abs().mean().item()
    white = (1.0 - gt).abs().mean().item()
    print(f"trained mesh ({v.shape[0]} vertices): mean |colour - analytic| {err:.4f}, white-background error {white:.4f}")
    # H100: 0.092 against 0.496 (55,208 vertices).  The bar leaves a 1.6x margin; part of the error is the mesh's
    # inner surfaces, where the learned density dips below the threshold inside the spheres
    assert err < 0.15 and err < 0.3 * white
