"""Write tests/golden/depth_viz.npz: what the reference's ``visualize_depth`` (utils/visualization.py:6-18, default
``cmap=cv2.COLORMAP_JET``) returns for a set of depth maps, by the UNMODIFIED reference file on the CPU.

``utils/visualization.py`` is loaded by path (the package's ``__init__`` would pull in the optimisers); it needs cv2,
PIL and torchvision.  The maps:
- ``trained``: ``depth_fine`` of a 200 x 200 Blender-style view of the trained scene (bench.blender_rays, seed 71,
  radius-4 camera, near 2, far 6), rendered at 64 + 64 samples by the CPU oracle (oracle/nerf_oracle.py) from the
  committed trained weights;
- ``nan``, ``posinf``, ``neginf``: positive depths with a few NaN, +inf or -inf (each alone);
- ``negative`` (depths of both signs), ``constant``, ``one`` (1 x 1) and ``odd`` (37 x 53).
A map holding both +inf and -inf is not stored: its normalised values are NaN, whose uint8 cast numpy does not define.
Stored per map: ``<name>.depth`` (float32) and ``<name>.out`` ((3, H, W) float32, channel 0 = cv2's blue).

    NERF_PL_REFERENCE=/path/to/nerf_pl python tests/golden/make_depth_viz_golden.py
"""
import importlib.util
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from oracle import nerf_oracle as orc  # noqa: E402
from tests import cases  # noqa: E402

REF = os.environ.get("NERF_PL_REFERENCE", "/root/reference")
NAME = "depth_viz"
SIDE, SEED, CHUNK = 200, 71, 2000


def reference_visualize_depth():
    spec = importlib.util.spec_from_file_location("reference_visualization",
                                                  os.path.join(REF, "utils", "visualization.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.visualize_depth


def trained_depth():
    ws = cases.trained_weights()
    rays = bench.blender_rays(0, SEED, W=SIDE, H=SIDE, pixels="all")
    depth = [orc.render_rays(ws, rays[i:i + CHUNK], 64, False, 0.0, 0.0, 64, True, True)["depth_fine"]
             for i in range(0, len(rays), CHUNK)]
    return np.concatenate(depth).astype(np.float32).reshape(SIDE, SIDE)


def synthetic_maps():
    rng = np.random.default_rng(2024)
    base = rng.uniform(2.0, 6.0, (64, 48)).astype(np.float32)
    maps = {}
    for name, val in (("nan", np.nan), ("posinf", np.inf), ("neginf", -np.inf)):
        m = base.copy()
        m[rng.random(m.shape) < 0.05] = val
        maps[name] = m
    maps["negative"] = rng.normal(0.0, 3.0, (40, 30)).astype(np.float32)
    maps["constant"] = np.full((16, 24), 3.25, np.float32)
    maps["one"] = np.array([[4.5]], np.float32)
    maps["odd"] = rng.uniform(0.0, 10.0, (37, 53)).astype(np.float32)
    return maps


def main():
    visualize_depth = reference_visualize_depth()
    maps = {"trained": trained_depth(), **synthetic_maps()}
    arrays = {}
    for name, depth in maps.items():
        out = visualize_depth(torch.from_numpy(depth.copy()))
        assert out.dtype == torch.float32 and out.shape == (3,) + depth.shape, (name, out.dtype, out.shape)
        arrays[f"{name}.depth"] = depth
        arrays[f"{name}.out"] = out.numpy()
    import cv2
    import PIL
    import torchvision
    meta = {"maps": list(maps), "side": SIDE, "seed": SEED, "cv2": cv2.__version__, "PIL": PIL.__version__,
            "torchvision": torchvision.__version__, "numpy": np.__version__, "torch": torch.__version__}
    arrays["meta"] = np.array(json.dumps(meta))
    path = os.path.join(HERE, f"{NAME}.npz")
    np.savez_compressed(path, **arrays)
    print(f"wrote {path} ({os.path.getsize(path)} bytes): {meta}")


if __name__ == "__main__":
    main()
