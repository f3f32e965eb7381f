"""Float64 restatement of the view-dependent bake (nb.query_rgb_sh, nb.render_baked of a view-dependent volume,
DESIGN.md §10k): the degree-2 basis of PlenOctrees' eval_sh, the 64 Fibonacci-sphere directions, P = pinv(Y), the
per-point fit from a network's weights, and the render over a dense (N, N, N, 28) grid.

The render's sample positions come from tests/baked_ref.samples (the kernel's float32 operations repeated); the ray
direction is normalised in float32 as the kernel does (d / |d|, |d| the float32 norm the sample spacing uses), and
everything after (basis, trilinear interpolation, colour, alpha, compositing) is float64."""
import numpy as np

from tests import baked_ref as br

F = np.float32
C0 = 0.28209479177387814
C1 = 0.4886025119029199
C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
D = 64
CHANNELS = 28


def basis(d):
    """(n, 9) float64 basis at the directions d (n, 3), taken as given (not normalised)."""
    d = np.asarray(d, np.float64)
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    return np.stack([np.full_like(x, C0), -C1 * y, C1 * z, -C1 * x, C2[0] * x * y, C2[1] * y * z,
                     C2[2] * (2.0 * z * z - x * x - y * y), C2[3] * x * z, C2[4] * (x * x - y * y)], 1)


def directions():
    """(64, 3) float32: z_j = 1 - (2 j + 1) / 64, phi_j = j pi (3 - sqrt 5), in float64, rounded once."""
    j = np.arange(D, dtype=np.float64)
    z = 1.0 - (2.0 * j + 1.0) / D
    phi = j * np.pi * (3.0 - np.sqrt(5.0))
    r = np.sqrt(1.0 - z * z)
    return np.stack([r * np.cos(phi), r * np.sin(phi), z], 1).astype(F)


def basis_matrix():
    """Y (64, 9) float64 at the float32 directions."""
    return basis(directions())


def projection():
    """P = pinv(Y) (9, 64) in float64."""
    return np.linalg.pinv(basis_matrix())


def slot_of(m, ch):
    """The index of coefficient m, channel ch among the 28 floats of a point."""
    return ch if m == 0 else 4 + 3 * (m - 1) + ch


def coefficient_slots():
    """(9, 3) int: slot_of(m, ch); slot 3 is sigma."""
    return np.array([[slot_of(m, ch) for ch in range(3)] for m in range(9)])


def pack_points(coef, sigma):
    """(n, 28) float64 from coefficients (n, 9, 3) and sigma (n,)."""
    coef = np.asarray(coef, np.float64)
    out = np.zeros((coef.shape[0], CHANNELS))
    out[:, coefficient_slots()] = coef
    out[:, 3] = sigma
    return out


def unpack_points(pts):
    """(n, 9, 3) coefficients and (n,) sigma of (n, 28) points."""
    pts = np.asarray(pts, np.float64)
    return pts[:, coefficient_slots()], pts[:, 3]


# ---- the fit from a network's weights --------------------------------------------------------------------------------
def _embed(x, n_freqs):
    out = [x]
    for k in range(n_freqs):
        out.append(np.sin(2.0 ** k * x))
        out.append(np.cos(2.0 ** k * x))
    return np.concatenate(out, -1)


def _lin(w, name, x):
    return x @ w[name + ".weight"].astype(np.float64).T + w[name + ".bias"].astype(np.float64)


def direction_colours(w, xyz, dirs):
    """(n, len(dirs), 3) float64 sigmoid rgb and (n,) raw sigma of the NeRF with the fp32 weights w at the raw
    positions xyz (n, 3), for each direction in dirs; the trunk is evaluated once."""
    enc = _embed(np.asarray(xyz, F).astype(np.float64), 10)
    h = enc
    for i in range(8):
        if i == 4:
            h = np.concatenate([enc, h], -1)
        h = np.maximum(_lin(w, f"xyz_encoding_{i + 1}.0", h), 0.0)
    sigma = _lin(w, "sigma", h)[:, 0]
    feat = _lin(w, "xyz_encoding_final", h)
    out = np.empty((len(h), len(dirs), 3))
    for j, d in enumerate(np.asarray(dirs, F).astype(np.float64)):
        denc = np.broadcast_to(_embed(d[None, :], 4), (len(h), 27))
        a = np.maximum(_lin(w, "dir_encoding.0", np.concatenate([feat, denc], -1)), 0.0)
        out[:, j] = 1.0 / (1.0 + np.exp(-_lin(w, "rgb.0", a)))
    return out, sigma


def query(w, xyz, proj):
    """(n, 28) float64: the fit c_{ch,m} = sum_j proj[m, j] f_{j,ch} of the per-direction colours, and raw sigma."""
    f, sigma = direction_colours(w, xyz, directions())
    coef = np.einsum("mj,njc->nmc", np.asarray(proj, np.float64), f)
    return pack_points(coef, sigma)


# ---- the render -------------------------------------------------------------------------------------------------------
def unit_dirs(rays):
    """(n, 3) float32 d / |d| with the float32 norm of baked_ref.samples."""
    d = np.asarray(rays, F)[:, 3:6]
    with np.errstate(all="ignore"):
        nd = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        return d / nd[:, None]


def render(dense, ranges, rays, step=None, white_back=False, early_stop=0.0):
    """As baked_ref.render over a dense (N, N, N, 28) grid: a sample's colour is clamp(sum_m cbar_m Y_m(d / |d|), 0, 1),
    cbar the trilinear coefficients."""
    g = np.asarray(dense, np.float64)
    N = g.shape[0]
    step = br.default_step(N, ranges) if step is None else step
    K, t, u = br.samples(N, ranges, rays, step)
    n, Kmax = t.shape
    valid = np.arange(Kmax)[None, :] < K[:, None]
    with np.errstate(all="ignore"):
        inside = valid & np.all((u >= 0) & (u <= F(N - 1)), axis=2)
    uu = np.where(inside[..., None], u, 0).astype(np.float64)
    cell = np.minimum(np.floor(uu), N - 2).astype(np.int64)
    f = uu - cell
    field = g.copy()
    field[..., 3] = np.where(g[..., 3] < 0, 0.0, g[..., 3])
    val = np.zeros((n, Kmax, CHANNELS))
    cx, cy, cz = cell[..., 0], cell[..., 1], cell[..., 2]
    fx, fy, fz = f[..., 0:1], f[..., 1:2], f[..., 2:3]
    for di in (0, 1):
        for dj in (0, 1):
            for dk in (0, 1):
                w = (fy if di else 1 - fy) * (fx if dj else 1 - fx) * (fz if dk else 1 - fz)
                val += w * field[cy + di, cx + dj, cz + dk]
    val = np.where(inside[..., None], val, 0.0)
    with np.errstate(all="ignore"):
        Y = basis(unit_dirs(rays).astype(np.float64))
    Y = np.where(np.isfinite(Y), Y, 0.0)
    coef = val[..., coefficient_slots()]                       # (n, K, 9, 3)
    col = np.clip(np.einsum("nkmc,nm->nkc", coef, Y), 0.0, 1.0)
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
    rgb = (w[..., None] * col).sum(1) + (1.0 if white_back else 0.0) * (1 - opacity)[:, None]
    depth = (w * t.astype(np.float64)).sum(1)
    t_max = np.where(K > 0, np.take_along_axis(t, np.maximum(K - 1, 0)[:, None], 1)[:, 0], 0).astype(np.float64) \
        if Kmax else np.zeros(n)
    return {"rgb": rgb, "depth": depth, "opacity": opacity, "cut": cut, "T_cut": T_cut, "t_max": t_max, "K": K}
