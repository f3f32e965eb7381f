"""A numpy restatement of extract_mesh.ipynb's "Generate .vol file for volume rendering in Unity" cell
(tests/test_volume_oracle.py, tests/test_gpu_volume.py).

The cell works on the (N^3, 4) ``rgbsigma`` of "Search for tight bounds", with sigma+ = max(sigma, 0):
* alpha a = 1 - exp(c sigma+) in float32, c = -(xmax - xmin) / N a Python float that numpy rounds to float32
  before the multiply;
* the kept points are those with a > 0, in increasing flat index i;
* each is written as the uint32 pair (i, r << 24 + g << 16 + b << 8 + trunc(255 a)), with r = trunc(255 rgb).

``exp="numpy"`` takes the cell's own float32 ``np.exp``, which is not correctly rounded and differs between numpy's
SIMD paths (AVX-512 vs AVX2 vs scalar); ``exp="f64"`` takes exp in float64 rounded once to float32, which is what
the device computes.
"""
from __future__ import annotations

import json

import numpy as np

from tests import npz_parts

EXPS = ("numpy", "f64")
MAX_N = 1625          # N^3 < 2^32: the cell casts the indices to uint32


def scale(x_range, N: int) -> np.float32:
    """The cell's ``-(xmax-xmin)/N``: a Python float, rounded to float32 when it meets the float32 sigma."""
    xmin, xmax = (float(v) for v in x_range)
    return np.float32(-(xmax - xmin) / N)


def exp_term(sigma_raw, x_range, N: int, exp: str = "f64") -> np.ndarray:
    """float32 ``exp(fl32(c) * max(sigma, 0))`` of raw sigma (any shape), flattened."""
    if exp not in EXPS:
        raise ValueError(f"exp must be one of {EXPS}")
    s = np.maximum(np.asarray(sigma_raw, np.float32).reshape(-1), np.float32(0))    # NaN stays NaN
    with np.errstate(invalid="ignore", over="ignore"):
        x = scale(x_range, N) * s
        return np.exp(x) if exp == "numpy" else np.exp(x.astype(np.float64)).astype(np.float32)


def alpha(sigma_raw, x_range, N: int, exp: str = "f64") -> np.ndarray:
    """float32 ``1 - exp(fl32(c) * max(sigma, 0))`` of raw sigma (any shape), flattened."""
    with np.errstate(invalid="ignore"):
        return (np.float32(1) - exp_term(sigma_raw, x_range, N, exp)).astype(np.float32)


def pack(rgbsigma, a) -> np.ndarray:
    """(M, 2) uint32 rows [i, s] of the points with a > 0, from the flattened (P, 4) rgbsigma and float32 a."""
    g = np.asarray(rgbsigma, np.float32).reshape(-1, 4)
    a = np.asarray(a, np.float32).reshape(-1)
    with np.errstate(invalid="ignore"):
        rgb = (g[:, :3] * 255).astype(np.uint32)
        i = np.where(a > 0)[0]
        s = rgb[i].dot(np.array([1 << 24, 1 << 16, 1 << 8])) + (a[i] * 255).astype(np.uint32)
    return np.stack([i, s], -1).astype(np.uint32).reshape(-1, 2)


def pack_volume(rgbsigma, x_range, exp: str = "f64") -> np.ndarray:
    """The cell on an (N, N, N, 4) (or (N^3, 4) with N given by its size) rgbsigma grid with raw sigma."""
    g = np.asarray(rgbsigma, np.float32).reshape(-1, 4)
    N = int(round(len(g) ** (1 / 3)))
    if N ** 3 != len(g) or N < 2 or N > MAX_N:
        raise ValueError("rgbsigma must hold N^3 points, 2 <= N <= 1625")
    return pack(g, alpha(g[:, 3], x_range, N, exp))


def vol_bytes(packed) -> bytes:
    """``res.tobytes()``: the rows as little-endian uint32."""
    return np.ascontiguousarray(np.asarray(packed).reshape(-1), dtype="<u4").tobytes()


def unpack(buf: bytes) -> np.ndarray:
    return np.frombuffer(buf, dtype="<u4").reshape(-1, 2)


def smallest_positive_alpha_sigma(x_range, N: int) -> np.float32:
    """The smallest non-negative float32 sigma whose alpha (float64-then-round exp) is > 0."""
    lo, hi = 0, int(np.float32(np.inf).view(np.int32))     # ordinals of non-negative float32
    while lo < hi:
        mid = (lo + hi) // 2
        if alpha(np.int32(mid).view(np.float32), x_range, N)[0] > 0:
            hi = mid
        else:
            lo = mid + 1
    return np.int32(lo).view(np.float32)


def numpy_simd() -> str:
    """The SIMD extensions this numpy dispatches to (what decides the float32 np.exp's last bits)."""
    try:
        return ",".join(np.show_config(mode="dicts")["SIMD Extensions"]["found"]) or "unknown"
    except Exception:
        return "unknown"


def load_golden(golden_dir: str):
    """{case name: dict(rgbsigma (N^3, 4), a (N^3,), vol bytes, N, ranges)} from tests/golden/volume_unity.part*.npz
    (rgbsigma is stored one channel per array)."""
    z = npz_parts.load(golden_dir, "volume_unity")
    meta = json.loads(str(z["meta"]))
    out = {}
    for name, m in meta["cases"].items():
        rgbsigma = np.stack([z[f"{name}.rgbsigma{ch}"] for ch in range(4)], 1)
        out[name] = {"rgbsigma": rgbsigma, "a": z[f"{name}.a"], "vol": z[f"{name}.vol"].tobytes(),
                     "N": m["N"], "ranges": [tuple(r) for r in m["ranges"]]}
    return out, meta
