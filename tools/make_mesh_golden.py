"""Write tests/golden/remap_cv2.npz: cv2.remap(INTER_LINEAR) samples of a random uint8 image, the fixture the
bilinear sampler of nerf_pl_b200.mesh (and its numpy restatement) must reproduce bit for bit.

Points: every (fx, fy) pair of 1/32-pixel fractions, random points, and the borders up to x = W-1, y = H-1.
Run: python tools/make_mesh_golden.py  (needs OpenCV)
"""
import os

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "..", "tests", "golden", "remap_cv2.npz")


def points(H, W, rng):
    f = np.arange(32, dtype=np.float32) / 32
    fx, fy = np.meshgrid(f, f)
    base = np.stack([3 + fx.ravel(), 5 + fy.ravel()], 1)                    # all 32 x 32 fraction pairs
    rnd = rng.uniform(0, 1, (4000, 2)).astype(np.float32) * np.float32([W - 1, H - 1])
    t = np.linspace(0, 1, 200, dtype=np.float32)
    edges = np.concatenate([
        np.stack([t * (W - 1), np.full_like(t, H - 1)], 1), np.stack([np.full_like(t, W - 1), t * (H - 1)], 1),
        np.stack([t * (W - 1), np.zeros_like(t)], 1), np.stack([np.zeros_like(t), t * (H - 1)], 1),
        np.float32([[W - 1, H - 1], [0, 0], [W - 1 - 1 / 64, H - 1 - 1 / 64], [W - 1.5, H - 1.5]])])
    return np.concatenate([base, rnd, edges]).astype(np.float32)


def main():
    rng = np.random.default_rng(7)
    H, W = 40, 50
    image = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    xy = points(H, W, rng)
    out = cv2.remap(image, xy[:, 0].copy(), xy[:, 1].copy(), interpolation=cv2.INTER_LINEAR)[:, 0]
    np.savez_compressed(OUT, image=image, xy=xy, out=out, opencv=np.array(cv2.__version__))
    print(f"wrote {os.path.normpath(OUT)}: {len(xy)} samples, OpenCV {cv2.__version__}")


if __name__ == "__main__":
    main()
