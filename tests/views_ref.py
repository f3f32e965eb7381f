"""Float32 emulation of view_batch_kernel (csrc/aux_kernels.cuh) and the synthetic scenes of the views goldens.

  * `pixel_rays32`: generate_rays_kernel's per-pixel body for chosen pixels, operation by operation; equal to
    `units_ref.generate_rays32` on whole images (tests/test_views_ref.py checks it), but needs no H x W buffer, so it
    also reaches pixels of views larger than memory.
  * `colours32`: the colour path, T.ToTensor()'s division by 255 and, for RGBA, blender.py:58's blend, one float32
    rounding per torch op.
  * `view_batch32`: both for pixel ids of the reference's concatenation order, p = (v H + j) W + i.
  * `blender_sources` / `write_blender_scene`, `llff_sources` / `write_llff_scene`: the seeded tiny scenes
    tests/golden/make_views_golden.py runs the reference on; the tests rewrite them from the stored sources (PNG is
    lossless, so the files decode to the same pixels).
Imports nothing from the product.
"""
from __future__ import annotations

import json
import os

import numpy as np

F32 = np.float32


def pixel_rays32(i, j, H: int, W: int, focal, c2w, near, far, ndc: bool = False):
    """Rays (len(i), 8) of pixels (row j, column i) of an H x W view; c2w (3, 4) or one pose per pixel (n, 3, 4)."""
    i, j = np.asarray(i, np.int64), np.asarray(j, np.int64)
    n = i.shape[0]
    f = F32(focal)
    c = np.broadcast_to(np.asarray(c2w, F32).reshape(-1, 3, 4), (n, 3, 4))
    dx = ((i.astype(F32) - F32(0.5) * F32(W)).astype(F32) / f).astype(F32)
    dy = -((j.astype(F32) - F32(0.5) * F32(H)).astype(F32) / f).astype(F32)
    dz = F32(-1)
    d = [(((dx * c[:, r, 0]).astype(F32) + (dy * c[:, r, 1]).astype(F32)).astype(F32)
          + (dz * c[:, r, 2]).astype(F32)).astype(F32) for r in range(3)]
    nrm = np.sqrt(((d[0] * d[0]).astype(F32) + (d[1] * d[1]).astype(F32)).astype(F32)
                  + (d[2] * d[2]).astype(F32)).astype(F32)
    d = [(x / nrm).astype(F32) for x in d]
    o = [c[:, r, 3].astype(F32).copy() for r in range(3)]
    nr, fr = np.full(n, F32(near), F32), np.full(n, F32(far), F32)
    if ndc:
        tt = -((F32(1) + o[2]).astype(F32) / d[2]).astype(F32)
        o = [(o[r] + (tt * d[r]).astype(F32)).astype(F32) for r in range(3)]
        ox, oy = (o[0] / o[2]).astype(F32), (o[1] / o[2]).astype(F32)
        sx = F32(-1) / F32(F32(W) / F32(F32(2) * f))
        sy = F32(-1) / F32(F32(H) / F32(F32(2) * f))
        o2 = (F32(1) + (F32(2) / o[2]).astype(F32)).astype(F32)
        d0 = (sx * ((d[0] / d[2]).astype(F32) - ox).astype(F32)).astype(F32)
        d1 = (sy * ((d[1] / d[2]).astype(F32) - oy).astype(F32)).astype(F32)
        o = [(sx * ox).astype(F32), (sy * oy).astype(F32), o2]
        d = [d0, d1, (F32(1) - o2).astype(F32)]
        nr, fr = np.zeros(n, F32), np.ones(n, F32)
    return np.stack(o + d + [nr, fr], 1).astype(F32)


def colours32(px):
    """(n, 3) float32 colours of (n, 3) RGB or (n, 4) RGBA uint8 pixels: u8 / 255 (the quotient rounded once, as
    torch's CPU div does), then for RGBA rgb * a + (1 - a) as three rounded ops."""
    px = np.asarray(px, np.uint8)
    x = (px.astype(F32) / F32(255)).astype(F32)
    if px.shape[1] == 3:
        return x
    a = x[:, 3:4]
    return ((x[:, :3] * a).astype(F32) + (F32(1) - a).astype(F32)).astype(F32)


def view_batch32(images, c2w, focal, near, far, ndc, ids):
    """view_batch_kernel for pixel ids `ids` of (V, H, W, C) `images` with (V, 3, 4) poses -> (rays, rgbs)."""
    V, H, W, C = images.shape
    ids = np.asarray(ids, np.int64)
    v, rem = np.divmod(ids, H * W)
    j, i = np.divmod(rem, W)
    rays = pixel_rays32(i, j, H, W, focal, np.asarray(c2w, F32)[v], near, far, ndc)
    return rays, colours32(images[v, j, i])


# ------------------------------------------------------------------------------------------------ golden scenes
BLENDER_SPLITS = {"train": 3, "val": 2, "test": 2}
BLENDER_SRC = 48                    # source PNG side
BLENDER_WH = (21, 21)               # odd: W / 2 = 10.5
BLENDER_ANGLE = 0.6911112070083618  # camera_angle_x of the reference's synthetic scenes
LLFF_N, LLFF_SRC_WH, LLFF_WH, LLFF_FOCAL = 5, (48, 36), (24, 18), 40.0


def _rotation(rng, scale):
    """A rotation close to the identity (scale = 1: anywhere), from a random skew matrix."""
    w = rng.normal(0, scale, 3)
    K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    th = np.linalg.norm(w)
    return np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th ** 2 * K @ K


def blender_sources(seed: int = 0):
    """{'blender.src.<split>': (F, 48, 48, 4) uint8, 'blender.pose.<split>': (F, 4, 4) float64}: RGBA frames with
    transparent, opaque and partly transparent regions, cameras on a radius-4 sphere."""
    rng = np.random.default_rng(seed)
    out = {}
    for split, F in BLENDER_SPLITS.items():
        img = rng.integers(0, 256, (F, BLENDER_SRC, BLENDER_SRC, 4), dtype=np.uint8)
        img[:, :12, :, 3] = 0
        img[:, 12:30, :, 3] = 255
        poses = np.zeros((F, 4, 4))
        for f in range(F):
            R = _rotation(rng, 1.0)
            poses[f, :3, :3] = R
            poses[f, :3, 3] = 4.0 * R[:, 2]
            poses[f, 3, 3] = 1.0
        out[f"blender.src.{split}"] = img
        out[f"blender.pose.{split}"] = poses
    return out


def write_blender_scene(root: str, src) -> None:
    from PIL import Image
    for split in BLENDER_SPLITS:
        os.makedirs(os.path.join(root, split), exist_ok=True)
        frames = []
        for f, (img, pose) in enumerate(zip(src[f"blender.src.{split}"], src[f"blender.pose.{split}"])):
            Image.fromarray(np.asarray(img), "RGBA").save(os.path.join(root, split, f"r_{f}.png"))
            frames.append({"file_path": f"./{split}/r_{f}", "transform_matrix": np.asarray(pose).tolist()})
        with open(os.path.join(root, f"transforms_{split}.json"), "w") as fh:
            json.dump({"camera_angle_x": BLENDER_ANGLE, "frames": frames}, fh)


def llff_sources(seed: int = 0):
    """{'llff.src': (5, 36, 48, 3) uint8, 'llff.poses_bounds': (5, 17) float64}: forward-facing cameras (final
    "right up back" rotations near the identity, stored in LLFF's "down right back" columns), hwf (36, 48, 40),
    bounds near in [1.5, 2.5], far in [12, 20]."""
    rng = np.random.default_rng(seed)
    W, H = LLFF_SRC_WH
    img = rng.integers(0, 256, (LLFF_N, H, W, 3), dtype=np.uint8)
    pb = np.zeros((LLFF_N, 17))
    for k in range(LLFF_N):
        R = _rotation(rng, 0.08)                 # columns x (right), y (up), z (back)
        t = np.array([rng.uniform(-0.6, 0.6), rng.uniform(-0.4, 0.4), rng.uniform(-0.2, 0.2)])
        raw = np.stack([-R[:, 1], R[:, 0], R[:, 2], t, np.array([H, W, LLFF_FOCAL])], 1)
        pb[k, :15] = raw.reshape(-1)
        pb[k, 15:] = rng.uniform(1.5, 2.5), rng.uniform(12.0, 20.0)
    return {"llff.src": img, "llff.poses_bounds": pb}


def write_llff_scene(root: str, src) -> None:
    from PIL import Image
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    for k, img in enumerate(src["llff.src"]):
        Image.fromarray(np.asarray(img), "RGB").save(os.path.join(root, "images", f"IMG_{k:03d}.png"))
    np.save(os.path.join(root, "poses_bounds.npy"), np.asarray(src["llff.poses_bounds"]))
