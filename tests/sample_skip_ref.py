"""Float64 numpy reference of the per-sample rule of ``skip="samples"`` (nerf_pl_b200.culling, DESIGN.md "Skipping
empty samples").

A sample of a ray ``[o, d, near, far]`` at depth ``z`` is the float32 point ``x = o + d z`` (a product, then a sum,
each rounded to float32, as the render kernel encodes it).  It is *evaluated* iff ``x`` lies in the closed box of an
occupied cell: in grid coordinates ``g = (x - lo) * (N - 1) / (hi - lo)`` (double, per axis, ranges may be
reversed) cell ``c`` spans ``[c, c + 1]``, so a coordinate on a boundary touches both cells and a point on a face,
edge or corner checks every cell it touches.  Outside ``[0, N - 1]^3`` (or NaN) nothing is evaluated.  A ray with a
non-finite value or ``far <= near``, and a pass whose interval lengths ``delta |d|`` are not all finite, is
evaluated at every sample of that pass.
"""
import numpy as np

F32 = np.float32


def sample_points(rays, z):
    """(R, S, 3) float32 points o + d z of rays (R, 8) at depths z (R, S), rounded as encode_row rounds them."""
    r = np.asarray(rays, F32)
    z = np.asarray(z, F32)
    return (r[:, None, 0:3] + (r[:, None, 3:6] * z[:, :, None]).astype(F32)).astype(F32)


def bit(words, c):
    w = np.asarray(words).view(np.uint32)
    return ((w[c >> 5] >> np.uint32(c & 31)) & 1) == 1


def point_evaluated(x, words, N, ranges):
    """bool (...) for float32 points x (..., 3): inside the closed box of an occupied cell of the grid
    (bits ``words``, ``N`` points per axis, ``ranges`` = (xmin, xmax, ymin, ymax, zmin, zmax))."""
    x = np.asarray(x, F32)
    M = N - 1
    flat = x.reshape(-1, 3)
    out = np.zeros(flat.shape[0], bool)
    lo = np.array(ranges[0::2], np.float64)
    hi = np.array(ranges[1::2], np.float64)
    scale = float(M) / (hi - lo)
    g = (flat.astype(np.float64) - lo) * scale
    for p in range(flat.shape[0]):
        v = g[p]
        if not np.all((v >= 0.0) & (v <= M)):
            continue
        cells = []
        for a in range(3):
            f = np.floor(v[a])
            c1 = min(int(f), M - 1)
            c0 = int(f) - 1 if (f == v[a] and f > 0) else c1
            cells.append(range(c0, c1 + 1))
        out[p] = any(bit(words, (cz * M + cy) * M + cx) for cz in cells[2] for cy in cells[1] for cx in cells[0])
    return out.reshape(x.shape[:-1])


def touched_cells(x, N, ranges):
    """(P, 8) int64 cell indices ``(cz * M + cy) * M + cx`` of the closed cell boxes holding each float32 point of x
    (..., 3), flattened: point_evaluated's rule with every point at once (a cell is repeated when the point touches
    fewer than 8); -1 for a point outside the box or NaN."""
    M = N - 1
    flat = np.asarray(x, F32).reshape(-1, 3).astype(np.float64)
    lo = np.array(ranges[0::2], np.float64)
    hi = np.array(ranges[1::2], np.float64)
    scale = float(M) / (hi - lo)
    g = (flat - lo) * scale
    with np.errstate(invalid="ignore"):
        inside = ((g >= 0.0) & (g <= M)).all(1)
    g = np.where(inside[:, None], g, 0.0)
    f = np.floor(g)
    fl = f.astype(np.int64)
    c1 = np.minimum(fl, M - 1)
    c0 = np.where((f == g) & (fl > 0), fl - 1, c1)
    cells = np.stack([(cz[:, 2] * M + cy[:, 1]) * M + cx[:, 0]
                      for cz in (c0, c1) for cy in (c0, c1) for cx in (c0, c1)], 1)
    cells[~inside] = -1
    return cells


def point_evaluated_vec(x, words, N, ranges):
    """point_evaluated without the loop over points."""
    cells = touched_cells(x, N, ranges)
    w = np.asarray(words).view(np.uint32)
    c = np.maximum(cells, 0)
    on = ((w[c >> 5] >> (c & 31).astype(np.uint32)) & 1) == 1
    return (on & (cells >= 0)).any(1).reshape(np.shape(x)[:-1])


def plain_rays(rays):
    """(R,) bool: the rays evaluated at every sample of both passes (a non-finite value or far <= near)."""
    r = np.asarray(rays, F32)
    return ~np.isfinite(r).all(1) | ~(r[:, 7] > r[:, 6])


def plain_pass(rays, z):
    """(R,) bool: the pass at depths z (R, S) is evaluated at every sample (plain ray, or some delta |d| not finite)."""
    r = np.asarray(rays, F32)
    z = np.asarray(z, F32)
    d = r[:, 3:6]
    with np.errstate(over="ignore", invalid="ignore"):
        dn = np.sqrt(((d[:, 0] * d[:, 0]).astype(F32) + (d[:, 1] * d[:, 1]).astype(F32)).astype(F32)
                     + (d[:, 2] * d[:, 2]).astype(F32)).astype(F32)
        delta = np.concatenate([(z[:, 1:] - z[:, :-1]).astype(F32), np.full((z.shape[0], 1), 1e10, F32)], 1)
        bad = ~np.isfinite((delta * dn[:, None]).astype(F32)).all(1)
    return plain_rays(r) | bad


def evaluated(rays, z, words, N, ranges):
    """(R, S) bool: the evaluated samples of one pass."""
    ev = point_evaluated_vec(sample_points(rays, z), words, N, ranges)
    ev[plain_pass(rays, z)] = True
    return ev


def mask_bits(mask_words, S):
    """(R, S) bool from the (R, 6) int32 mask words of nerfb200_render_samples."""
    w = np.asarray(mask_words).view(np.uint32)
    i = np.arange(S)
    return ((w[:, i >> 5] >> (i & 31).astype(np.uint32)) & 1) == 1


def z_base(rays, S, use_disp=False):
    """The coarse depths of render_rays at perturb = 0, in the kernel's float32 steps (render_kernel.cuh z_base)."""
    r = np.asarray(rays, F32)
    if S <= 1:
        t = np.zeros(S, F32)
    else:
        step = F32(1) / F32(S - 1)
        i = np.arange(S)
        t = np.where(i < S // 2, (step * i.astype(F32)).astype(F32),
                     (F32(1) - (step * (S - 1 - i).astype(F32)).astype(F32)).astype(F32)).astype(F32)
    omt = (F32(1) - t).astype(F32)
    if use_disp:
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            a = ((F32(1) / r[:, 6:7]).astype(F32) * omt).astype(F32)
            b = ((F32(1) / r[:, 7:8]).astype(F32) * t).astype(F32)
            return (F32(1) / (a + b).astype(F32)).astype(F32)
    return ((r[:, 6:7] * omt).astype(F32) + (r[:, 7:8] * t).astype(F32)).astype(F32)
