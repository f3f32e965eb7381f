"""Float64 restatement of the baked-volume render (nb.render_baked, DESIGN.md §10j) over a dense (N, N, N, 4) grid in
rgb_sigma_grid's layout: dense[i, j, k] is the value at (x_j, y_i, z_k).

The sample positions are defined by float32 operations (|d|, dt = s / |d|, K, t_k = near + (k + 1/2) dt,
p = o + t d and u = (p - lo) * scale, each rounded once in that order), which this module repeats in numpy float32 so
that it picks the same samples and cells as the kernel; everything after (trilinear interpolation, alpha, compositing)
is float64.  A grid point outside the stored bricks of a volume holds 0 in its dense grid, so this restatement never
skips anything: it evaluates every sample."""
import numpy as np

F = np.float32


def default_step(N, ranges):
    return min(abs(ranges[2 * a + 1] - ranges[2 * a]) for a in range(3)) / (N - 1)


def samples(N, ranges, rays, step):
    """Per ray its sample count K, dt, and the (n, Kmax) depths t and (n, Kmax, 3) index coordinates u (float32)."""
    rays = np.asarray(rays, F)
    o, d, near, far = rays[:, 0:3], rays[:, 3:6], rays[:, 6], rays[:, 7]
    s = F(step)
    with np.errstate(all="ignore"):
        nd = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        dt = s / nd
        kf = np.floor((far - near) / dt)
        ok = np.isfinite(rays).all(1) & (far > near) & (dt > 0) & np.isfinite(dt)
    K = np.where(ok, kf, 0).astype(np.int64)
    Kmax = int(K.max()) if len(K) else 0
    k = np.arange(Kmax, dtype=F)[None, :]
    lo = np.array([F(ranges[2 * a]) for a in range(3)], F)
    scale = np.array([F((N - 1) / (ranges[2 * a + 1] - ranges[2 * a])) for a in range(3)], F)
    with np.errstate(all="ignore"):
        t = near[:, None] + (k + F(0.5)) * np.where(ok, dt, F(0))[:, None]
        p = o[:, None, :] + t[:, :, None] * d[:, None, :]
        u = (p - lo) * scale
    return K, t, u


def render(dense, ranges, rays, step=None, white_back=False, early_stop=0.0):
    """{"rgb", "depth", "opacity"} in float64, and per ray "cut" (ended early), "T_cut" (its transmittance after
    the last sample it composited; 0 for a ray that is not cut) and "t_max" (its largest sample depth)."""
    g = np.asarray(dense, np.float64)
    N = g.shape[0]
    step = default_step(N, ranges) if step is None else step
    K, t, u = samples(N, ranges, rays, step)
    n, Kmax = t.shape
    valid = np.arange(Kmax)[None, :] < K[:, None]
    with np.errstate(all="ignore"):
        inside = valid & np.all((u >= 0) & (u <= F(N - 1)), axis=2)
    uu = np.where(inside[..., None], u, 0).astype(np.float64)
    cell = np.minimum(np.floor(uu), N - 2).astype(np.int64)
    f = uu - cell
    sig = g[..., 3]
    field = np.concatenate([g[..., :3], np.where(sig < 0, 0.0, sig)[..., None]], -1)
    val = np.zeros((n, Kmax, 4))
    cx, cy, cz = cell[..., 0], cell[..., 1], cell[..., 2]
    fx, fy, fz = f[..., 0:1], f[..., 1:2], f[..., 2:3]
    for di in (0, 1):
        for dj in (0, 1):
            for dk in (0, 1):
                w = (fy if di else 1 - fy) * (fx if dj else 1 - fx) * (fz if dk else 1 - fz)
                val += w * field[cy + di, cx + dj, cz + dk]
    val = np.where(inside[..., None], val, 0.0)
    s = float(F(step))
    alpha = 1 - np.exp(-val[..., 3] * s)
    T_after = np.cumprod(1 - alpha, axis=1)
    cut = np.zeros(n, bool)
    T_cut = np.zeros(n)
    if early_stop > 0:
        below = valid & (T_after < early_stop) & (alpha != 0)
        for r in range(n):
            hit = np.nonzero(below[r])[0]
            if len(hit):
                k0 = hit[0]
                cut[r] = k0 < K[r] - 1
                T_cut[r] = T_after[r, k0]
                alpha[r, k0 + 1:] = 0
    T = np.concatenate([np.ones((n, 1)), np.cumprod(1 - alpha, axis=1)[:, :-1]], 1)
    w = alpha * T
    opacity = w.sum(1)
    rgb = (w[..., None] * val[..., :3]).sum(1) + (1.0 if white_back else 0.0) * (1 - opacity)[:, None]
    depth = (w * t.astype(np.float64)).sum(1)
    t_max = np.where(K > 0, np.take_along_axis(t, np.maximum(K - 1, 0)[:, None], 1)[:, 0], 0).astype(np.float64) \
        if Kmax else np.zeros(n)
    return {"rgb": rgb, "depth": depth, "opacity": opacity, "cut": cut, "T_cut": T_cut, "t_max": t_max, "K": K}
