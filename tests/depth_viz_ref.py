"""numpy restatement of the reference's ``visualize_depth`` (utils/visualization.py:6-18) with the default
``cmap=cv2.COLORMAP_JET``, for the tests; no cv2, PIL or torchvision needed.

The table is the one the device kernel uses, read from nerf_pl_b200/csrc/jet_lut.h (tools/gen_jet_lut.py).  Every
step is the reference's in float32: nan_to_num, min and max, (x - mi) / (ma - mi + 1e-8) (NEP 50: the Python float
is float32 here), 255 * y truncated to uint8, the JET lookup, and ToTensor's u8 / 255.  The channels stay in cv2's
(B, G, R) order, because the reference passes cv2's BGR array to ``Image.fromarray`` as RGB.

Outside the contract: a map holding both +inf and -inf (its normalised values are NaN, whose uint8 cast numpy does
not define)."""
import os
import re

import numpy as np

LUT_H = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "nerf_pl_b200", "csrc",
                     "jet_lut.h")


def jet_lut():
    """(256, 3) uint8, (B, G, R), as committed in jet_lut.h."""
    body = open(LUT_H).read().split("= {", 1)[1]
    vals = [int(v) for v in re.findall(r"\d+", body.split("};", 1)[0])]
    table = np.array(vals, np.uint8).reshape(256, 3)
    return table


def to_uint8(depth):
    """The uint8 index map of the reference (before the colour lookup)."""
    x = np.nan_to_num(np.asarray(depth, np.float32))
    mi, ma = np.min(x), np.max(x)
    y = (x - mi) / (ma - mi + np.float32(1e-8))
    assert y.dtype == np.float32
    with np.errstate(invalid="ignore"):
        return (np.float32(255) * y).astype(np.uint8)


def visualize_depth(depth):
    """(H, W) float32 -> (3, H, W) float32 in [0, 1], channel 0 = blue."""
    rgb = jet_lut()[to_uint8(depth)]                       # (H, W, 3), cv2's BGR order
    return (rgb.transpose(2, 0, 1).astype(np.float32) / np.float32(255)).astype(np.float32)
