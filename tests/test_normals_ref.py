"""The numpy restatement of open3d's vertex normals (tests/normals_ref.py) on hand-computed meshes and at its edges,
and the reference fixture of the vertex-normal colours (tests/golden/vertex_normal_colors.part*.npz) against it."""
import json
import os

import numpy as np
import pytest

from tests import normals_ref as nr
from tests import npz_parts

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("name", list(nr.hand_meshes()))
def test_hand_meshes(name):
    v, t, expected = nr.hand_meshes()[name]
    n = nr.vertex_normals(v, t)
    assert n.dtype == np.float64 and n.shape == (len(v), 3)
    if expected is not None:
        assert nr.same_bits(n, expected), n
    assert nr.same_bits(n, nr.vertex_normals_loop(v, t))


def test_closed_meshes_point_outwards_in_index_order():
    for name in ("tetrahedron", "cube"):
        v, t, _ = nr.hand_meshes()[name]
        n = nr.vertex_normals(v, t)
        c = v.astype(np.float64).mean(0)
        assert (np.einsum("ij,ij->i", n, v - c) > 0).all()
        assert np.allclose(np.linalg.norm(n, axis=1), 1.0, rtol=0, atol=1e-15)


def test_summation_follows_triangle_order_not_corner_columns():
    v, t, _ = nr.order_mesh()
    n = nr.vertex_normals(v, t)
    col = nr.vertex_normals_column_order(v, t)
    # triangle order: x = (1 + 2^-60) - 1 = 0; column order keeps 2^-60
    assert nr.same_bits(n[0], [0.0, 1.0, 0.0])
    assert col[0, 0] == 2.0 ** -60
    assert not nr.same_bits(n, col)
    assert nr.same_bits(n, nr.vertex_normals_loop(v, t))


def test_no_triangles_and_no_vertices():
    v = np.float32(np.random.default_rng(0).normal(size=(5, 3)))
    assert nr.same_bits(nr.vertex_normals(v, np.zeros((0, 3), np.int32)), np.zeros((5, 3)))
    assert nr.vertex_normals(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32)).shape == (0, 3)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_vectorised_sum_equals_open3d_loop_on_random_soups(seed):
    rng = np.random.default_rng(seed)
    V = 60
    # non-manifold: repeated corners, repeated triangles, vertices of high degree, wide magnitudes
    v = (rng.normal(size=(V, 3)) * 10.0 ** rng.integers(-6, 6, (V, 1))).astype(np.float32)
    t = rng.integers(0, V, (400, 3)).astype(np.int32)
    t[:20] = t[20:40]
    t[40:50, 1] = t[40:50, 0]
    assert nr.same_bits(nr.vertex_normals(v, t), nr.vertex_normals_loop(v, t))


@pytest.mark.parametrize("bounds, near_t", [((2.0, 6.0), 1.0), ((1.7, 6.1), 1.1), (np.float32([0.3, 4.7]), 0.9),
                                            ((0.1, 1e3), 2.5), ((2.0, 6.0), 1e-3)])
def test_ray_expression_is_float32_step_by_step(bounds, near_t):
    """The torch expression of :190-193 rounds near, far and near_t to float32 and each product once: what
    nerfb200_normal_rays computes."""
    rng = np.random.default_rng(7)
    v = rng.normal(size=(500, 3)).astype(np.float32)
    n = nr.normalize(rng.normal(size=(500, 3)))
    rays = nr.normal_rays_torch(v, n, np.asarray(bounds), near_t)
    f32 = np.float32
    d = n.astype(f32)
    near, far, nt = f32(np.min(bounds)), f32(np.max(bounds)), f32(near_t)
    o = v - (d * near) * nt
    assert rays.dtype == np.float32
    assert np.array_equal(rays.view(np.uint32), np.concatenate(
        [o, d, np.full((500, 1), near), np.full((500, 1), far)], 1).view(np.uint32))


def _fixture():
    return npz_parts.load(GOLDEN, "vertex_normal_colors")


def test_fixture_normals_rays_and_colours_are_consistent():
    z = _fixture()
    meta = json.loads(str(z["meta"]))
    v, t = z["vertices"], z["triangles"]
    assert v.dtype == np.float32 and t.dtype == np.int32 and len(v) > 1000
    assert set(meta["cases"]) == {"blender", "inexact"}
    for name, c in meta["cases"].items():
        n = z[f"{name}.normals"]
        assert nr.same_bits(n, nr.vertex_normals(v, t))
        rays = nr.normal_rays_torch(v, n, np.array(c["bounds"]), c["near_t"])
        assert np.array_equal(rays.view(np.uint32), z[f"{name}.rays"].view(np.uint32))
        rgb = z[f"{name}.rgb_fine"]
        assert rgb.shape == (len(v), 3) and rgb.min() >= 0 and rgb.max() <= 1
        assert np.array_equal(z[f"{name}.colors"], (rgb * 255.0).astype(np.uint8))
    # the two cases differ where they should: bounds, near_t
    assert not np.array_equal(z["blender.rays"][:, :3], z["inexact.rays"][:, :3])
    assert float(np.float32(1.7)) != 1.7 and z["inexact.rays"][0, 6] == np.float32(1.7)


def test_fixture_stays_under_one_megabyte_per_part():
    parts = [f for f in os.listdir(GOLDEN) if f.startswith("vertex_normal_colors.part")]
    assert parts and all(os.path.getsize(os.path.join(GOLDEN, f)) < 1_000_000 for f in parts)
