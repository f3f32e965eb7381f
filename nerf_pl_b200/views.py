"""Host readers of the reference's two dataset formats that stop at the views: uint8 images and camera poses, no
rays.  ``DeviceViewBatches`` (data.py) turns them into training batches on the GPU and ``generate_rays`` into
validation and test rays, so a user gets from ``root_dir`` to training without kornia and without a host
``all_rays``.

``read_blender_views`` follows ``datasets/blender.py`` (``BlenderDataset``) and ``read_llff_views``
``datasets/llff.py`` (``LLFFDataset``): the same files, the same PIL calls (``resize(img_wh, LANCZOS)``,
``convert('RGB')``), so the uint8 pixels are the reference's, and the same float64 pose arithmetic, so focal, bounds
and poses are the reference's bit for bit.  PIL is imported inside the readers: the package does not need it.
"""
from __future__ import annotations

import glob
import json
import os
from typing import NamedTuple, Optional, Tuple

import numpy as np

__all__ = ["Views", "read_blender_views", "read_llff_views"]


class Views(NamedTuple):
    """One split of a dataset.  ``images``: (V, H, W, C) uint8 (C = 4 for Blender, 3 for LLFF), or None for the
    LLFF test path, which has poses only.  ``c2w``: (V, 3, 4) float64 camera-to-world poses, as the reference holds
    them (it casts each to float32 with ``torch.FloatTensor`` before making rays).  ``focal``, ``near``, ``far``:
    the values the reference writes into its rays (``ndc``: LLFF's forward-facing NDC, near/far 0 and 1).
    ``white_back``: the ``white_back`` the reference's training passes to ``render_rays``."""
    images: Optional[np.ndarray]
    c2w: np.ndarray
    focal: float
    near: float
    far: float
    ndc: bool
    white_back: bool


def _load_rgba(path: str, img_wh: Tuple[int, int]) -> np.ndarray:
    from PIL import Image
    img = Image.open(path).resize(tuple(img_wh), Image.LANCZOS)
    arr = np.array(img, dtype=np.uint8)
    if arr.ndim != 3 or arr.shape[2] != 4:
        raise ValueError(f"{path}: a Blender view must be RGBA (blender.py:57 views it as 4 channels)")
    return arr


def read_blender_views(root_dir: str, split: str = "train", img_wh: Tuple[int, int] = (800, 800)) -> Views:
    """``BlenderDataset(root_dir, split, img_wh)`` (datasets/blender.py:11-69) as views: every frame of
    ``transforms_{split}.json`` in file order, RGBA at ``img_wh``.  Focal ``0.5 * 800 / tan(0.5 * camera_angle_x)``
    rescaled by ``img_wh[0] / 800``, bounds 2 and 6, white background.  The reference validates only the first 8
    frames of the val split (blender.py:77-78); all frames are returned here."""
    w, h = img_wh
    if w != h:
        raise ValueError("image width must equal image height (blender.py:15)")
    with open(os.path.join(root_dir, f"transforms_{split}.json"), "r") as f:
        meta = json.load(f)
    focal = 0.5 * 800 / np.tan(0.5 * meta["camera_angle_x"])      # the focal length at W = 800
    focal *= img_wh[0] / 800
    images, poses = [], []
    for frame in meta["frames"]:
        poses.append(np.array(frame["transform_matrix"])[:3, :4])
        images.append(_load_rgba(os.path.join(root_dir, f"{frame['file_path']}.png"), img_wh))
    return Views(np.stack(images), np.stack(poses), float(focal), 2.0, 6.0, False, True)


# ------------------------------------------------------------------------------------------------------------ LLFF
def _unit(v: np.ndarray) -> np.ndarray:
    return v / np.linalg.norm(v)


def _mean_pose(poses: np.ndarray) -> np.ndarray:
    """llff.py:17-52: the (3, 4) pose whose origin is the mean camera centre, z the normalised mean z axis, x the
    normalised cross product of the mean y axis with z, and y = z x x."""
    origin = poses[..., 3].mean(0)
    z = _unit(poses[..., 2].mean(0))
    x = _unit(np.cross(poses[..., 1].mean(0), z))
    return np.stack([x, np.cross(z, x), z, origin], 1)


def _recentre(poses: np.ndarray) -> np.ndarray:
    """llff.py:55-79: every pose expressed in the frame of the mean pose (inverse of the homogeneous mean pose times
    each homogeneous pose)."""
    to_mean = np.eye(4)
    to_mean[:3] = _mean_pose(poses)
    bottom = np.tile(np.array([0, 0, 0, 1]), (len(poses), 1, 1))
    return (np.linalg.inv(to_mean) @ np.concatenate([poses, bottom], 1))[:, :3]


def _spiral_path(radii: np.ndarray, focus_depth: float, n_poses: int = 120) -> np.ndarray:
    """llff.py:82-113: two turns of a spiral of the given radii whose cameras look at (0, 0, -focus_depth)."""
    out = []
    for t in np.linspace(0, 4 * np.pi, n_poses + 1)[:-1]:
        centre = np.array([np.cos(t), -np.sin(t), -np.sin(0.5 * t)]) * radii
        z = _unit(centre - np.array([0, 0, -focus_depth]))
        x = _unit(np.cross(np.array([0, 1, 0]), z))
        out.append(np.stack([x, np.cross(z, x), z, centre], 1))
    return np.stack(out, 0)


def _spheric_path(radius: float, n_poses: int = 120) -> np.ndarray:
    """llff.py:116-158: a circle of cameras 36 degrees above the object (rotation about y by theta, about x by
    -pi/5, translation (0, -0.9 r, r)), in the reference's axis convention."""
    def homog(rows):
        return np.array(rows)

    phi = -np.pi / 5
    rot_phi = homog([[1, 0, 0, 0], [0, np.cos(phi), -np.sin(phi), 0], [0, np.sin(phi), np.cos(phi), 0], [0, 0, 0, 1]])
    shift = homog([[1, 0, 0, 0], [0, 1, 0, -0.9 * radius], [0, 0, 1, radius], [0, 0, 0, 1]])
    axes = homog([[-1, 0, 0, 0], [0, 0, 1, 0], [0, 1, 0, 0], [0, 0, 0, 1]])
    out = []
    for th in np.linspace(0, 2 * np.pi, n_poses + 1)[:-1]:
        rot_th = homog([[np.cos(th), 0, -np.sin(th), 0], [0, 1, 0, 0], [np.sin(th), 0, np.cos(th), 0], [0, 0, 0, 1]])
        out.append((axes @ (rot_th @ rot_phi @ shift))[:3])
    return np.stack(out, 0)


def read_llff_views(root_dir: str, split: str = "train", img_wh: Tuple[int, int] = (504, 378),
                    spheric_poses: bool = False, val_num: int = 1) -> Views:
    """``LLFFDataset(root_dir, split, img_wh, spheric_poses, val_num)`` (datasets/llff.py:161-292) as views.

    Poses from ``poses_bounds.npy``: the focal rescaled to ``img_wh``, the axes turned from "down right back" to
    "right up back", the poses re-centred on their mean pose and scaled so that the nearest bound is 1 / 0.75.  The
    val view is the camera closest to the centre; ``'train'`` is every other image of ``images/`` (sorted), ``'val'``
    that one image.  Any other split is a test path with no images: the poses themselves for a split ending in
    ``'train'``, else a 120-pose spiral (forward-facing) or circle (``spheric_poses``).  Forward-facing scenes use
    NDC (near 0, far 1); spheric ones the scaled bounds: near = min, far = min(8 near, max).  ``val_num`` only sets
    how often the reference repeats the val view (llff.py:281-282) and does not change what is returned."""
    del val_num
    poses_bounds = np.load(os.path.join(root_dir, "poses_bounds.npy"))
    image_paths = sorted(glob.glob(os.path.join(root_dir, "images/*")))
    if split in ("train", "val") and len(poses_bounds) != len(image_paths):
        raise ValueError("Mismatch between number of images and number of poses! Please rerun COLMAP!")
    raw = poses_bounds[:, :15].reshape(-1, 3, 5)
    bounds = poses_bounds[:, -2:]
    H, W, focal = raw[0, :, -1]
    if H * img_wh[0] != W * img_wh[1]:
        raise ValueError(f"You must set @img_wh to have the same aspect ratio as ({W}, {H}) !")
    focal *= img_wh[0] / W
    # "down right back" -> "right up back" (x' = y, y' = -x), the hwf column dropped
    poses = _recentre(np.concatenate([raw[..., 1:2], -raw[..., :1], raw[..., 2:4]], -1))
    val_idx = int(np.argmin(np.linalg.norm(poses[..., 3], axis=1)))
    scale = bounds.min() * 0.75            # the nearest depth lands at 1 / 0.75
    bounds = bounds / scale
    poses[..., 3] /= scale
    if spheric_poses:
        near = bounds.min()
        far = min(8 * near, bounds.max())
    else:
        near, far = 0, 1

    def load(path):
        from PIL import Image
        img = Image.open(path).convert("RGB")
        if img.size[1] * img_wh[0] != img.size[0] * img_wh[1]:
            raise ValueError(f"{path} has different aspect ratio than img_wh, please check your data!")
        return np.array(img.resize(tuple(img_wh), Image.LANCZOS), dtype=np.uint8)

    if split == "train":
        keep = [i for i in range(len(image_paths)) if i != val_idx]
        images, c2w = np.stack([load(image_paths[i]) for i in keep]), poses[keep]
    elif split == "val":
        images, c2w = load(image_paths[val_idx])[None], poses[val_idx][None]
    else:
        images = None
        if split.endswith("train"):
            c2w = poses
        elif not spheric_poses:
            c2w = _spiral_path(np.percentile(np.abs(poses[..., 3]), 90, axis=0), 3.5)
        else:
            c2w = _spheric_path(1.1 * bounds.min())
    return Views(images, c2w, float(focal), float(near), float(far), not spheric_poses, False)
