"""The view readers (nerf_pl_b200/views.py) and the float32 emulation of view_batch_kernel (tests/views_ref.py)
against what the unmodified reference dataset classes made of two tiny scenes (tests/golden/views_*.npz, written by
tests/golden/make_views_golden.py).  CPU only.

- Readers: uint8 images (their ToTensor equals the reference's bit for bit), focal, near / far, bounds, poses, the
  val view and the test paths exactly.
- Emulation: its colours equal the reference's all_rgbs and val / test rgbs exactly; its rays are within the
  tolerance tests/test_oracle_golden.py grants generate_rays (the reference rotates through a CPU matmul), and its
  near / far columns are exact.
- The colour path against torchvision's ToTensor plus the blend for all 65,536 (value, alpha) pairs, bit for bit.
"""
import os

import numpy as np
import pytest
import torch

import nerf_pl_b200 as nb
from tests import cases
from tests import units_ref as ur
from tests import views_ref as vr

F32 = np.float32
RAY_TOL = {False: dict(atol=2e-6, rtol=0), True: dict(atol=5e-6, rtol=1e-5)}     # test_oracle_golden.py:79-80


def _golden(name):
    return np.load(os.path.join(cases.GOLDEN, f"views_{name}.npz"))


@pytest.fixture(scope="module")
def blender_scene(tmp_path_factory):
    pytest.importorskip("PIL")
    g = _golden("blender")
    root = str(tmp_path_factory.mktemp("blender"))
    vr.write_blender_scene(root, g)
    return g, root


@pytest.fixture(scope="module")
def llff_scene(tmp_path_factory):
    pytest.importorskip("PIL")
    g = _golden("llff")
    root = str(tmp_path_factory.mktemp("llff"))
    vr.write_llff_scene(root, g)
    return g, root


def _to_tensor(images):
    """(V, H, W, C) uint8 -> (V, C, H, W) as T.ToTensor() makes each: float, then div(255)."""
    return torch.from_numpy(np.ascontiguousarray(images)).permute(0, 3, 1, 2).float().div(255).numpy()


def _same_bits(a, b):
    return ur.bitwise_differ(a, b) == 0 and np.shape(a) == np.shape(b)


def _all_ids(images):
    return np.arange(int(np.prod(images.shape[:3])), dtype=np.int64)


# --------------------------------------------------------------------------------------------------------- Blender
def test_blender_reader_equals_the_reference(blender_scene):
    g, root = blender_scene
    v = nb.read_blender_views(root, "train", vr.BLENDER_WH)
    assert v.images.dtype == np.uint8 and v.images.shape == (3, 21, 21, 4)
    assert _same_bits(_to_tensor(v.images), g["blender.train.to_tensor"])
    assert v.focal == float(g["blender.focal"]) and (v.near, v.far) == tuple(g["blender.near_far"])
    assert v.c2w.dtype == np.float64 and np.array_equal(v.c2w, g["blender.train.poses"])
    assert (v.ndc, v.white_back) == (False, True)
    for split in ("val", "test"):
        s = nb.read_blender_views(root, split, vr.BLENDER_WH)
        assert _same_bits(_to_tensor(s.images), g[f"blender.{split}.to_tensor"])
        assert np.array_equal(s.c2w.astype(F32), g[f"blender.{split}.c2w"])
        assert np.array_equal(s.images[..., 3].reshape(len(s.images), -1) > 0, g[f"blender.{split}.valid_mask"])
    with pytest.raises(ValueError, match="width must equal"):
        nb.read_blender_views(root, "train", (21, 20))


def test_blender_emulation_equals_the_reference(blender_scene):
    g, root = blender_scene
    v = nb.read_blender_views(root, "train", vr.BLENDER_WH)
    rays, rgbs = vr.view_batch32(v.images, v.c2w, v.focal, v.near, v.far, v.ndc, _all_ids(v.images))
    assert _same_bits(rgbs, g["blender.train.rgbs"])
    ref = g["blender.train.rays"]
    np.testing.assert_allclose(rays, ref, **RAY_TOL[False])
    assert _same_bits(rays[:, :3], ref[:, :3]) and _same_bits(rays[:, 6:], ref[:, 6:])
    for split in ("val", "test"):
        s = nb.read_blender_views(root, split, vr.BLENDER_WH)
        rays, rgbs = vr.view_batch32(s.images, s.c2w, s.focal, s.near, s.far, s.ndc, _all_ids(s.images))
        n = len(s.images)
        assert _same_bits(rgbs, g[f"blender.{split}.rgbs"].reshape(-1, 3))
        np.testing.assert_allclose(rays, g[f"blender.{split}.rays"].reshape(-1, 8), **RAY_TOL[False])
        assert rays.shape == (n * 441, 8)


# ------------------------------------------------------------------------------------------------------------ LLFF
@pytest.mark.parametrize("tag,spheric", [("ndc", False), ("spheric", True)])
def test_llff_reader_equals_the_reference(llff_scene, tag, spheric):
    g, root = llff_scene
    v = nb.read_llff_views(root, "train", vr.LLFF_WH, spheric_poses=spheric)
    val_idx = int(g[f"llff.{tag}.val_idx"])
    keep = [k for k in range(vr.LLFF_N) if k != val_idx]
    assert v.images.dtype == np.uint8 and v.images.shape == (vr.LLFF_N - 1, 18, 24, 3)
    assert _same_bits(_to_tensor(v.images), g[f"llff.{tag}.train.to_tensor"])
    assert v.focal == float(g[f"llff.{tag}.focal"])
    poses = g[f"llff.{tag}.poses"]
    assert np.array_equal(v.c2w, poses[keep])
    bounds = g[f"llff.{tag}.bounds"]
    if spheric:
        assert v.near == bounds.min() and v.far == min(8 * bounds.min(), bounds.max())
        assert not v.ndc
    else:
        assert (v.near, v.far, v.ndc) == (0.0, 1.0, True)
    assert not v.white_back
    val = nb.read_llff_views(root, "val", vr.LLFF_WH, spheric_poses=spheric)
    assert np.array_equal(val.c2w[0], poses[val_idx])
    assert np.array_equal(val.c2w[0].astype(F32), g[f"llff.{tag}.val.c2w"])
    test = nb.read_llff_views(root, "test", vr.LLFF_WH, spheric_poses=spheric)
    assert test.images is None and np.array_equal(test.c2w, g[f"llff.{tag}.test.poses"])
    assert test.c2w.shape == (120, 3, 4)
    assert np.array_equal(nb.read_llff_views(root, "test_train", vr.LLFF_WH, spheric_poses=spheric).c2w, poses)
    with pytest.raises(ValueError, match="aspect ratio"):
        nb.read_llff_views(root, "train", (24, 17), spheric_poses=spheric)


@pytest.mark.parametrize("tag,spheric", [("ndc", False), ("spheric", True)])
def test_llff_emulation_equals_the_reference(llff_scene, tag, spheric):
    g, root = llff_scene
    v = nb.read_llff_views(root, "train", vr.LLFF_WH, spheric_poses=spheric)
    rays, rgbs = vr.view_batch32(v.images, v.c2w, v.focal, v.near, v.far, v.ndc, _all_ids(v.images))
    assert _same_bits(rgbs, g[f"llff.{tag}.train.rgbs"])
    ref = g[f"llff.{tag}.train.rays"]
    np.testing.assert_allclose(rays, ref, **RAY_TOL[v.ndc])
    assert _same_bits(rays[:, 6:], ref[:, 6:])
    val = nb.read_llff_views(root, "val", vr.LLFF_WH, spheric_poses=spheric)
    rays, rgbs = vr.view_batch32(val.images, val.c2w, val.focal, val.near, val.far, val.ndc, _all_ids(val.images))
    assert _same_bits(rgbs, g[f"llff.{tag}.val.rgbs"])
    np.testing.assert_allclose(rays, g[f"llff.{tag}.val.rays"], **RAY_TOL[v.ndc])
    test = nb.read_llff_views(root, "test", vr.LLFF_WH, spheric_poses=spheric)
    H, W = 18, 24
    j, i = np.divmod(np.arange(H * W), W)
    rays0 = vr.pixel_rays32(i, j, H, W, test.focal, test.c2w[0], test.near, test.far, test.ndc)
    np.testing.assert_allclose(rays0, g[f"llff.{tag}.test.rays0"], **RAY_TOL[v.ndc])


# ------------------------------------------------------------------------------------------------ the emulation
@pytest.mark.parametrize("ndc", [False, True])
@pytest.mark.parametrize("H,W", [(1, 1), (7, 5), (24, 36)])
def test_pixel_rays_equal_generate_rays32(H, W, ndc):
    """The per-pixel emulation is units_ref.generate_rays32 bit for bit, on the raygen golden's pose."""
    g = np.load(os.path.join(cases.GOLDEN, "raygen.npz"))
    f = float(g["focal"])
    j, i = np.divmod(np.arange(H * W), W)
    assert _same_bits(vr.pixel_rays32(i, j, H, W, f, g["c2w"], 2.0, 6.0, ndc),
                      ur.generate_rays32(H, W, f, g["c2w"], 2.0, 6.0, ndc))


def test_view_batch_emulation_decodes_view_row_column():
    rng = np.random.default_rng(3)
    V, H, W = 3, 5, 7
    images = rng.integers(0, 256, (V, H, W, 4), dtype=np.uint8)
    c2w = rng.normal(size=(V, 3, 4)).astype(F32)
    ids = rng.permutation(V * H * W)
    rays, rgbs = vr.view_batch32(images, c2w, 6.0, 2.0, 6.0, False, ids)
    for k, p in enumerate(ids):
        v, rem = divmod(int(p), H * W)
        assert _same_bits(rays[k], ur.generate_rays32(H, W, 6.0, c2w[v], 2.0, 6.0)[rem])
        assert _same_bits(rgbs[k], vr.colours32(images[v].reshape(-1, 4)[rem:rem + 1])[0])


def test_colour_path_against_to_tensor_for_every_value_and_alpha():
    """All 65,536 (value, alpha) pairs through torchvision's ToTensor on a PIL RGBA image and blender.py:58's blend
    == colours32 bit for bit; and RGB through ToTensor == u8 / 255.  The division is what ToTensor does: a
    multiplication by float32(1 / 255) differs on 126 of the 256 values."""
    T = pytest.importorskip("torchvision.transforms")
    Image = pytest.importorskip("PIL.Image")
    val, alpha = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8), indexing="ij")
    rgba = np.stack([val, 255 - val, val[::-1], alpha], -1)              # every pair in each colour channel
    img = T.ToTensor()(Image.fromarray(rgba, "RGBA"))                      # (4, 256, 256)
    img = img.view(4, -1).permute(1, 0)
    ref = (img[:, :3] * img[:, -1:] + (1 - img[:, -1:])).numpy()          # blender.py:58
    assert _same_bits(vr.colours32(rgba.reshape(-1, 4)), ref)
    rgb = T.ToTensor()(Image.fromarray(np.ascontiguousarray(rgba[..., :3]), "RGB")).view(3, -1).permute(1, 0).numpy()
    assert _same_bits(vr.colours32(rgba[..., :3].reshape(-1, 3)), rgb)
    u = np.arange(256, dtype=np.uint8)
    mul = (u.astype(F32) * F32(1 / 255)).astype(F32)
    assert ur.bitwise_differ(mul, vr.colours32(np.stack([u, u, u], 1))[:, 0]) == 126


def test_reader_signatures():
    import inspect
    assert list(inspect.signature(nb.read_blender_views).parameters) == ["root_dir", "split", "img_wh"]
    p = inspect.signature(nb.read_llff_views).parameters
    assert list(p) == ["root_dir", "split", "img_wh", "spheric_poses", "val_num"]
    assert p["img_wh"].default == (504, 378) and p["spheric_poses"].default is False and p["val_num"].default == 1
    assert inspect.signature(nb.read_blender_views).parameters["img_wh"].default == (800, 800)
