"""Float64 numpy restatement of the density grid update (nerf_pl_b200.DensityGrid, csrc/density_kernels.cuh,
include/nerf_pl_b200.h; DESIGN.md "Keeping the grid current during training").

For an N-point grid over ranges ((xmin, xmax), (ymin, ymax), (zmin, zmax)), M = N - 1 cells per axis and cell
c = (cz * M + cy) * M + cx, one update from a network with key s is:

1. u_a = philox.uniform(s, ray = c, i = a, stream = 2), a = 0, 1, 2 (tests/philox.py, the render kernel's generator);
2. p_a = float32(lo_a + (double(cell_a) + double(u_a)) * ((hi_a - lo_a) / M)): numpy float64 rounds each operation
   on its own, as the device's __dadd_rn / __dmul_rn / __ddiv_rn do;
3. sigma_c = the network's sigma at p (the caller supplies it);
4. density_c = fmax(float32(decay * density_c), sigma_c > 0 ? sigma_c : 0) in float32 (NaN sigma counts as 0);
5. occupied iff float64(density_c) > threshold, dilated by ``dilate`` cells (Chebyshev) and packed as
   tests/occupancy_ref.py packs; the bits past the last cell are 0;
6. key + 1.

Initial state: density 0, every cell occupied, key = seed.
"""
import numpy as np

from . import occupancy_ref as oc
from . import philox

MASK64 = (1 << 64) - 1


def cells(N, start=0, count=None):
    """(count, 3) int64 (cx, cy, cz) of cells [start, start + count)."""
    M = N - 1
    count = M ** 3 - start if count is None else count
    c = np.arange(start, start + count, dtype=np.int64)
    return np.stack([c % M, (c // M) % M, c // (M * M)], 1)


def points(seed, N, ranges, start=0, count=None):
    """Steps 1-2: (count, 3) float32 points of cells [start, start + count) for key ``seed``."""
    M = N - 1
    count = M ** 3 - start if count is None else count
    u = philox.uniform(int(seed) & MASK64, count, 3, 2, ray0=start).astype(np.float64)
    lo = np.array([float(r[0]) for r in ranges])
    hi = np.array([float(r[1]) for r in ranges])
    step = (hi - lo) / float(M)
    return (lo + (cells(N, start, count).astype(np.float64) + u) * step).astype(np.float32)


def decay_max(density, sigma, decay):
    """Step 4 in float32."""
    s = np.asarray(sigma, np.float32)
    s = np.where(s > 0, s, np.float32(0))
    return np.fmax(np.float32(decay) * np.asarray(density, np.float32), s).astype(np.float32)


def occupied(density, N, threshold, dilate):
    """Step 5 before packing: occ[cx, cy, cz] bool of a density in cell order."""
    M = N - 1
    occ = (np.asarray(density, np.float32).astype(np.float64) > float(threshold)).reshape(M, M, M).transpose(2, 1, 0)
    return oc.dilate(occ, dilate)


def bits(density, N, threshold, dilate):
    return oc.pack_bits(occupied(density, N, threshold, dilate))


def initial(N, seed):
    """The state of a fresh or reset grid."""
    C = (N - 1) ** 3
    return {"density": np.zeros(C, np.float32), "bits": oc.pack_bits(np.ones((N - 1,) * 3, bool)), "key": int(seed)}


def update(state, sigma_fn, N, ranges, threshold, decay, dilate):
    """Steps 1-6: the next state; ``sigma_fn(points (C, 3) float32) -> (C,) float32``."""
    p = points(state["key"], N, ranges)
    d = decay_max(state["density"], sigma_fn(p), decay)
    return {"density": d, "bits": bits(d, N, threshold, dilate), "key": state["key"] + 1}
