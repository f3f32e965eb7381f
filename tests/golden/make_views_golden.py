"""Write tests/golden/views_blender.npz and views_llff.npz: what the UNMODIFIED reference dataset classes
(datasets/blender.py BlenderDataset, datasets/llff.py LLFFDataset) make of two tiny seeded scenes
(tests/views_ref.py blender_sources / llff_sources), on the CPU.

- Blender: RGBA PNGs of 48 x 48 resized to 21 x 21, train / val / test splits.  Stored: the sources and poses, the
  train split's all_rays / all_rgbs, focal and poses, every val and test sample (rays, rgbs, valid_mask, c2w), and
  the (4, h, w) float tensor ``T.ToTensor()`` made of each frame.
- LLFF: five RGB PNGs of 48 x 36 and poses_bounds.npy, img_wh 24 x 18, forward-facing (NDC) and spheric.  Stored per
  variant: the train split's all_rays / all_rgbs, the val sample, focal, bounds, poses, the val index and the test
  path (spiral or circle).

``datasets/ray_utils.py:2`` imports ``kornia.create_meshgrid``; kornia is not installed, so that one function is
shimmed (the un-normalised pixel grid, x = column, y = row), as tests/golden/make_golden.py shims it.  The classes are
subclassed only to record what their ``self.transform`` (``T.ToTensor()``) returns; nothing they compute is changed.

    NERF_PL_REFERENCE=/path/to/nerf_pl python tests/golden/make_views_golden.py
"""
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from tests import views_ref as vr  # noqa: E402

REF = os.environ.get("NERF_PL_REFERENCE", "/root/reference")


def import_datasets():
    kor = types.ModuleType("kornia")

    def create_meshgrid(H, W, normalized_coordinates=False):      # kornia shim (see the module docstring)
        assert not normalized_coordinates
        ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32),
                                indexing="ij")
        return torch.stack([xs, ys], -1)[None]
    kor.create_meshgrid = create_meshgrid
    sys.modules["kornia"] = kor
    sys.path.insert(0, REF)
    from datasets.blender import BlenderDataset
    from datasets.llff import LLFFDataset
    return BlenderDataset, LLFFDataset


def recording(cls):
    class Recording(cls):
        def define_transforms(self):
            super().define_transforms()
            inner, self.to_tensor = self.transform, []

            def transform(img):
                t = inner(img)
                self.to_tensor.append(t.clone())
                return t
            self.transform = transform
    return Recording


def blender(BlenderDataset, out):
    src = vr.blender_sources(0)
    out.update(src)
    Rec = recording(BlenderDataset)
    with tempfile.TemporaryDirectory() as root:
        vr.write_blender_scene(root, src)
        tr = Rec(root, "train", vr.BLENDER_WH)
        out["blender.train.rays"] = tr.all_rays.numpy()
        out["blender.train.rgbs"] = tr.all_rgbs.numpy()
        out["blender.train.to_tensor"] = torch.stack(tr.to_tensor).numpy()
        out["blender.train.poses"] = np.stack(tr.poses)
        out["blender.focal"] = np.float64(tr.focal)
        out["blender.near_far"] = np.array([tr.near, tr.far])
        for split in ("val", "test"):
            ds = Rec(root, split, vr.BLENDER_WH)
            samples = [ds[k] for k in range(vr.BLENDER_SPLITS[split])]
            for key in ("rays", "rgbs", "valid_mask", "c2w"):
                out[f"blender.{split}.{key}"] = torch.stack([s[key] for s in samples]).numpy()
            out[f"blender.{split}.to_tensor"] = torch.stack(ds.to_tensor).numpy()
    print("blender", {k: v.shape for k, v in out.items() if k.startswith("blender.")})


def llff(LLFFDataset, out):
    src = vr.llff_sources(0)
    out.update(src)
    Rec = recording(LLFFDataset)
    with tempfile.TemporaryDirectory() as root:
        vr.write_llff_scene(root, src)
        for tag, spheric in (("ndc", False), ("spheric", True)):
            tr = Rec(root, "train", vr.LLFF_WH, spheric_poses=spheric)
            out[f"llff.{tag}.train.rays"] = tr.all_rays.numpy()
            out[f"llff.{tag}.train.rgbs"] = tr.all_rgbs.numpy()
            out[f"llff.{tag}.train.to_tensor"] = torch.stack(tr.to_tensor).numpy()
            out[f"llff.{tag}.focal"] = np.float64(tr.focal)
            out[f"llff.{tag}.bounds"] = tr.bounds
            out[f"llff.{tag}.poses"] = tr.poses
            val = Rec(root, "val", vr.LLFF_WH, spheric_poses=spheric)
            s = val[0]
            out[f"llff.{tag}.val.rays"] = s["rays"].numpy()
            out[f"llff.{tag}.val.rgbs"] = s["rgbs"].numpy()
            out[f"llff.{tag}.val.c2w"] = s["c2w"].numpy()
            names = sorted(os.listdir(os.path.join(root, "images")))
            out[f"llff.{tag}.val_idx"] = np.int64(names.index(os.path.basename(val.image_path_val)))
            te = Rec(root, "test", vr.LLFF_WH, spheric_poses=spheric)
            out[f"llff.{tag}.test.poses"] = te.poses_test
            out[f"llff.{tag}.test.rays0"] = te[0]["rays"].numpy()
    print("llff", {k: v.shape for k, v in out.items() if k.startswith("llff.")})


def main():
    torch.set_num_threads(1)
    BlenderDataset, LLFFDataset = import_datasets()
    import PIL
    import torchvision
    meta = {"PIL": PIL.__version__, "torchvision": torchvision.__version__, "numpy": np.__version__,
            "torch": torch.__version__}
    for name, fn, cls in (("views_blender", blender, BlenderDataset), ("views_llff", llff, LLFFDataset)):
        arrays = {}
        fn(cls, arrays)
        arrays["meta"] = np.array(json.dumps(meta))
        path = os.path.join(HERE, f"{name}.npz")
        np.savez_compressed(path, **arrays)
        print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
