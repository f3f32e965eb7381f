"""Float64 restatements of the stand-alone kernels of csrc/aux_kernels.cuh, and numpy float32 emulations of the
kernels whose operation order is fully determined.

Bit-exact emulations (every step is one correctly rounded float32 or float64 operation in the kernel's order):
  * `generate_rays32`: generate_rays_kernel, blender and NDC, with the kernel's float32 `sx = -1 / (W / (2 f))`;
  * `mse_psnr32`: mse_psnr_kernel's two MSEs (1024 strided double partials, xor butterfly, thread 0 over 32 warps)
    and their float32 sum;
  * sample_pdf_kernel: tests/render_tape.py `cdf_standalone` + `inverse_cdf`;
  * `pack_image`'s plain slices: the packed weight image is float16(W) there, bit for bit.
Bounded against float64 (the kernel calls sinf / cosf / expf / log10f, or sums 256 fmaf products):
  * `embed64` (Embedding.forward: documented 2-ulp sinf / cosf), `generate_rays64` (the reference's formulas with a
    double focal), `check_packed` (the folded W' and b' within the fmaf chain's bound), composite via
    tests/render_tape.py `composite_errors`.
`searchsorted_bisect` restates the torchsearchsorted CUDA kernel's search for the CPU tests, which check the
oracle's comparison semantics (ties, +-0, +-inf, NaN) against it.  Imports nothing from the product: used by
tests/test_units_ref.py (CPU) and tests/test_gpu_units.py.
"""
from __future__ import annotations

from typing import Optional

import numpy as np

F16, F32, F64 = np.float16, np.float32, np.float64
U32 = 2.0 ** -24
LANES = 32


def ulp32(x):
    """Spacing of float32 at |x| (float64 result)."""
    return np.spacing(np.abs(np.asarray(x, F64)).astype(F32)).astype(F64)


def bitwise_differ(got, ref) -> int:
    """Elements of `got` whose float32 bits differ from `ref` (NaN equals NaN whatever its payload)."""
    g, r = np.asarray(got, F32), np.asarray(ref, F32)
    same = (g.view(np.uint32) == r.view(np.uint32)) | (np.isnan(g) & np.isnan(r))
    return int((~same).sum())


# --------------------------------------------------------------------------------------------- generate_rays
def generate_rays32(H: int, W: int, focal, c2w, near, far, ndc: bool = False, defect: Optional[str] = None):
    """generate_rays_kernel in float32, operation by operation -> (H W, 8).  `defect="sx_f64"` forms sx and sy in
    double, as the oracle does, instead of the kernel's float32 `-1.f / (W / (2.f * focal))`."""
    f = F32(focal)
    c = np.asarray(c2w, F32).reshape(3, 4)
    idx = np.arange(H * W, dtype=np.int64)
    j, i = idx // W, idx % W
    dx = ((i.astype(F32) - F32(0.5) * F32(W)).astype(F32) / f).astype(F32)
    dy = -((j.astype(F32) - F32(0.5) * F32(H)).astype(F32) / f).astype(F32)
    dz = F32(-1)
    d = [((dx * c[r, 0]).astype(F32) + (dy * c[r, 1]).astype(F32)).astype(F32) + F32(dz * c[r, 2]) for r in range(3)]
    d = [x.astype(F32) for x in d]
    nrm = np.sqrt(((d[0] * d[0]).astype(F32) + (d[1] * d[1]).astype(F32)).astype(F32) + (d[2] * d[2]).astype(F32))
    nrm = nrm.astype(F32)
    d = [(x / nrm).astype(F32) for x in d]
    o = [np.full(H * W, c[r, 3], F32) for r in range(3)]
    nr, fr = np.full(H * W, F32(near), F32), np.full(H * W, F32(far), F32)
    if ndc:
        tt = -((F32(1) + o[2]).astype(F32) / d[2]).astype(F32)
        o = [(o[r] + (tt * d[r]).astype(F32)).astype(F32) for r in range(3)]
        ox, oy = (o[0] / o[2]).astype(F32), (o[1] / o[2]).astype(F32)
        if defect == "sx_f64":
            sx, sy = F32(-1.0 / (W / (2.0 * float(f)))), F32(-1.0 / (H / (2.0 * float(f))))
        else:
            sx = F32(-1) / F32(F32(W) / F32(F32(2) * f))
            sy = F32(-1) / F32(F32(H) / F32(F32(2) * f))
        o2 = (F32(1) + (F32(2) / o[2]).astype(F32)).astype(F32)
        d0 = (sx * ((d[0] / d[2]).astype(F32) - ox).astype(F32)).astype(F32)
        d1 = (sy * ((d[1] / d[2]).astype(F32) - oy).astype(F32)).astype(F32)
        o = [(sx * ox).astype(F32), (sy * oy).astype(F32), o2]
        d = [d0, d1, (F32(1) - o2).astype(F32)]
        nr, fr = np.zeros(H * W, F32), np.ones(H * W, F32)
    return np.stack(o + d + [nr, fr], 1)


def generate_rays64(H: int, W: int, focal: float, c2w, near, far, ndc: bool = False, idx=None):
    """datasets/ray_utils.py get_ray_directions / get_rays / get_ndc_rays (llff.py: near plane 1.0) in float64, with
    `focal` a Python double as the reference holds it and c2w the float32 pose; the pixels `idx` (default all).  Also
    returns the magnitude scale of each output column (the largest |value| of its o or d triple), the unit the
    comparisons measure ulps in."""
    c = np.asarray(c2w, F32).astype(F64).reshape(3, 4)
    idx = np.arange(H * W, dtype=np.int64) if idx is None else np.asarray(idx, np.int64)
    j, i = np.divmod(idx, W)
    dirs = np.stack([(i - W / 2) / focal, -(j - H / 2) / focal, -np.ones(len(idx))], 1)
    d = dirs @ c[:, :3].T
    d = d / np.linalg.norm(d, axis=1, keepdims=True)
    o = np.broadcast_to(c[:, 3], d.shape).copy()
    nf = np.broadcast_to(np.array([near, far], F64), (len(idx), 2))
    if ndc:
        t = -(1.0 + o[:, 2]) / d[:, 2]
        o = o + t[:, None] * d
        o_n = np.stack([-1 / (W / (2 * focal)) * o[:, 0] / o[:, 2], -1 / (H / (2 * focal)) * o[:, 1] / o[:, 2],
                        1 + 2 * 1.0 / o[:, 2]], 1)
        d_n = np.stack([-1 / (W / (2 * focal)) * (d[:, 0] / d[:, 2] - o[:, 0] / o[:, 2]),
                        -1 / (H / (2 * focal)) * (d[:, 1] / d[:, 2] - o[:, 1] / o[:, 2]), -2 * 1.0 / o[:, 2]], 1)
        o, d = o_n, d_n
        nf = np.broadcast_to(np.array([0.0, 1.0]), (len(idx), 2))
    out = np.concatenate([o, d, nf], 1)
    so = np.abs(o).max(1, keepdims=True)
    sd = np.abs(d).max(1, keepdims=True)
    scale = np.concatenate([np.repeat(so, 3, 1), np.repeat(sd, 3, 1), np.abs(nf)], 1)
    return out, scale


def ray_ulps(got, ref64, scale):
    """Per-element error of float32 rays against `generate_rays64` in ulps of the triple's magnitude."""
    return np.abs(np.asarray(got, F64) - ref64) / np.maximum(ulp32(scale), 2.0 ** -149)


# --------------------------------------------------------------------------------------------- mse / psnr
def _thread_sums(x, t):
    """sum over i of (x_i - t_i)^2 in mse_psnr_kernel's order: thread p of 1024 adds elements p, p + 1024, .. in
    double (the float32 difference squared is exact in double, so an fma and a mul + add agree); xor butterfly per
    warp; thread 0 adds the 32 warp sums in order."""
    d = (np.asarray(x, F32).reshape(-1) - np.asarray(t, F32).reshape(-1)).astype(F32).astype(F64)
    sq = d * d
    m = -(-sq.size // 1024)
    buf = np.zeros(m * 1024, F64)
    buf[:sq.size] = sq
    acc = np.cumsum(buf.reshape(m, 1024), axis=0)[-1].reshape(32, LANES)
    lanes = np.arange(LANES)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[:, lanes ^ o]
    s = 0.0
    for w in range(32):
        s = s + float(acc[w, 0])
    return s


def mse_psnr32(rgb_coarse, rgb_fine, target):
    """(mse_coarse, mse_fine, mse_coarse + mse_fine) as mse_psnr_kernel forms them, bit for bit (float32), and the
    psnr argument (the finest mse present).  mse_fine is 0 without rgb_fine."""
    n = np.asarray(target).size
    mc = F32(_thread_sums(rgb_coarse, target) / float(n)) if rgb_coarse is not None else F32(0)
    mf = F32(_thread_sums(rgb_fine, target) / float(n)) if rgb_fine is not None else F32(0)
    return mc, mf, F32(mc + mf), (mf if rgb_fine is not None else mc)


def mse64(rgb, target):
    return float(np.mean((np.asarray(rgb, F64) - np.asarray(target, F64)) ** 2))


def psnr_bar(mse32: float, psnr32: float) -> float:
    """|psnr - (-10 log10 mse64)|: the float32 rounding of the mse (10 / ln 10 * 2^-24 relative), log10f's documented
    2 ulps times 10, and the rounding of the product."""
    lg = abs(np.log10(max(float(mse32), 1e-45)))
    return 10 / np.log(10) * U32 + 20 * float(ulp32(lg)) + float(ulp32(psnr32))


# --------------------------------------------------------------------------------------------- searchsorted
def searchsorted_bisect(a_row, v, side: str = "left"):
    """torchsearchsorted's CUDA search (searchsorted_cuda_kernel.cu:3-81) restated on one row: it looks for the column
    `col` with a[col] < v <= a[col + 1] ('left') or a[col] <= v < a[col + 1] ('right'), treats the last column as
    `a[-1] <= v` for both sides, and returns col + 1 (0 when v lies below a[0])."""
    a = [F32(x) for x in np.asarray(a_row, F32)]
    n = len(a)
    out = np.empty(len(v), np.int64)
    for q, val in enumerate(np.asarray(v, F32)):
        def rel(col):
            if col == n - 1:
                return 1 if a[col] <= val else -1
            lower = a[col] < val if side == "left" else a[col] <= val
            higher = a[col + 1] >= val if side == "left" else a[col + 1] > val
            return 0 if (lower and higher) else (1 if lower else -1)
        left, right, res = 0, n, -1
        while right >= left:
            mid = left + (right - left) // 2
            r = rel(mid)
            if r == 0:
                res = mid
                break
            if r > 0:
                if mid == n - 1:
                    res = n - 1
                    break
                left = mid
            else:
                if mid == 0:
                    break
                right = mid
        out[q] = res + 1
    return out


# --------------------------------------------------------------------------------------------- Embedding
def embed64(x, n_freqs: int, freqs=None):
    """Embedding.forward (models/nerf.py:33-38) in float64 of the float32 products f x (f = 2^k is exact), channel
    order [x, sin f0 x, cos f0 x, sin f1 x, ..]; `freqs` overrides the bands (float32 values)."""
    x = np.asarray(x, F32)
    fs = [F32(2.0 ** k) for k in range(n_freqs)] if freqs is None else [F32(f) for f in freqs]
    out = [x.astype(F64)]
    with np.errstate(invalid="ignore", over="ignore"):
        for f in fs:
            a = (f * x).astype(F32).astype(F64)
            out += [np.sin(a), np.cos(a)]
    return np.concatenate(out, -1)


def embed_ulps(got, ref64):
    """|got - ref64| in ulps of float32(ref64); non-finite references must give NaN (sin / cos of +-inf or NaN), and
    those elements count as 0 when they do and as inf when they do not."""
    got = np.asarray(got, F64)
    with np.errstate(invalid="ignore"):
        e = np.abs(got - ref64) / np.maximum(ulp32(ref64), 2.0 ** -149)
    fin = np.isfinite(ref64)
    e = np.where(fin, e, np.where(np.isnan(got) == np.isnan(ref64), 0.0, np.inf))
    return np.where(np.isnan(e), np.inf, e)


EMBED_ULPS = 2.0     # CUDA's documented maximum error of sinf / cosf over the whole range (Programming Guide, App. G)


# --------------------------------------------------------------------------------------------- packed weight image
SLICE256, SLICE128 = 256 * 128, 128 * 128
OFF_DIR = 30 * SLICE256
HALF_BYTES = OFF_DIR + 5 * SLICE128
F32_BIAS, F32_WSIGMA = 0, 9 * 256
F32_BSIGMA = F32_WSIGMA + 256
F32_WRGB = F32_BSIGMA + 4
F32_BRGB = F32_WRGB + 3 * 128
F32_WDIR = F32_BRGB + 4
F32_COUNT = F32_WDIR + 28 * 128
FWD_BYTES = HALF_BYTES + 4 * F32_COUNT
OFF_BWD = (FWD_BYTES + 1023) & ~1023
PACKED_BYTES = OFF_BWD + 30 * SLICE256
PACK_DEFECTS = ("slice_swap", "no_swizzle", "bwd_wrong_layer", "fold_no_bias", "zero_col_63")


def sw128_off(row, k):
    """csrc/ptx.cuh sw128_off: row n at n * 128 bytes, 16-byte chunk k / 8 at position (k / 8) ^ (n & 7)."""
    row, k = np.asarray(row), np.asarray(k)
    return row * 128 + ((((k >> 3) ^ (row & 7)) & 7) << 4) + ((k & 7) << 1)


def _params(w):
    """The 24 tensors in layout.h's order from a state_dict-like dict of float32 arrays."""
    names = ([f"xyz_encoding_{i}.0" for i in range(1, 9)]
             + ["xyz_encoding_final", "dir_encoding.0", "sigma", "rgb.0"])
    return [np.asarray(w[f"{n}.{s}"], F32) for n in names for s in ("weight", "bias")]


def _plain_slices(p):
    """{slice: (N, 64) float32 matrix} of every forward slice that is a copy of one weight (zero-padded)."""
    out = {}
    for s in range(35):
        if 30 <= s <= 33:
            continue
        N = 256 if s < 30 else 128
        m = np.zeros((N, 64), F32)
        if s == 0:
            m[:, :63] = p[0]
        elif s <= 12:
            l = 1 + (s - 1) // 4
            ko = ((s - 1) % 4) * 64
            m[:] = p[2 * l][:, ko:ko + 64]
        elif s == 13:
            m[:, :63] = p[8][:, :63]
        elif s <= 17:
            ko = 63 + (s - 14) * 64
            m[:] = p[8][:, ko:ko + 64]
        elif s <= 29:
            l = 5 + (s - 18) // 4
            ko = ((s - 18) % 4) * 64
            m[:] = p[2 * l][:, ko:ko + 64]
        else:
            m[:, :27] = p[18][:, 256:283]
        out[s] = m
    return out


def _bwd_plain(p):
    """{backward slice: (256, 64) B[n][k] = W[k0 + k][n0 + n]} for slices 2..29."""
    out = {}
    for s in range(2, 30):
        step, kb = (s - 2) // 4, (s - 2) % 4
        L = 8 - step
        n0 = 63 if L == 5 else 0
        out[s] = np.ascontiguousarray(p[2 * (L - 1)][kb * 64:kb * 64 + 64, n0:n0 + 256].T)
    return out


def fold64(p):
    """W' = W_dir[:, :256] W_final, b' = b_dir + W_dir[:, :256] b_final in float64, and their fmaf-chain bounds
    gamma_256 sum |terms| (fp32: acc = fmaf(a, b, acc) over 256 terms, from 0 or from b_dir)."""
    wd = p[18][:, :256].astype(F64)
    wf, bf, bd = p[16].astype(F64), p[17].astype(F64), p[19].astype(F64)
    g = 256 * U32 / (1 - 256 * U32)
    return wd @ wf, g * (np.abs(wd) @ np.abs(wf)), bd + wd @ bf, g * (np.abs(bd) + np.abs(wd) @ np.abs(bf))


def _f32_region(p, bprime):
    o = np.zeros(F32_COUNT, F32)
    for l in range(8):
        o[256 * l:256 * l + 256] = p[2 * l + 1]
    o[8 * 256:8 * 256 + 128] = bprime
    o[F32_WSIGMA:F32_WSIGMA + 256] = p[20].reshape(-1)
    o[F32_BSIGMA] = p[21][0]
    o[F32_WRGB:F32_WRGB + 384] = p[22].reshape(-1)
    o[F32_BRGB:F32_BRGB + 3] = p[23]
    o[F32_WDIR:F32_WDIR + 27 * 128] = p[18][:, 256:283].T.reshape(-1)
    return o


def _put(img, base, m, swizzle=True):
    N = m.shape[0]
    n, k = np.meshgrid(np.arange(N), np.arange(64), indexing="ij")
    off = base + (sw128_off(n, k) if swizzle else n * 128 + k * 2)
    img.view(F16)[off.reshape(-1) // 2] = m.astype(F16).reshape(-1)


def pack_image(w, defect: Optional[str] = None) -> np.ndarray:
    """csrc/layout.h's packed image of the weights `w` as uint8 bytes (PACKED_BYTES; the alignment gap before the
    backward region is 0).  W' and b' are float64 rounded to float32 (within the kernel's fmaf bound).  A `defect`
    of PACK_DEFECTS plants one wrong slice / region for the CPU tests."""
    p = _params(w)
    wp64, _, bp64, _ = fold64(p)
    wp = wp64.astype(F32)
    img = np.zeros(PACKED_BYTES, np.uint8)
    sw = defect != "no_swizzle"
    plain = _plain_slices(p)
    if defect == "slice_swap":
        plain[5], plain[6] = plain[6], plain[5]
    if defect == "zero_col_63":
        plain[0][:, 63] = p[8][:, 0]
    for s, m in plain.items():
        _put(img, s * SLICE256 if s < 30 else OFF_DIR + (s - 30) * SLICE128, m, sw)
    for s in range(30, 34):
        _put(img, OFF_DIR + (s - 30) * SLICE128, wp[:, (s - 30) * 64:(s - 30) * 64 + 64], sw)
    bprime = (p[18][:, :256].astype(F64) @ p[17].astype(F64)).astype(F32) if defect == "fold_no_bias" else bp64
    img[HALF_BYTES:FWD_BYTES] = _f32_region(p, np.asarray(bprime, F32)).view(np.uint8)
    bwd = _bwd_plain(p)
    if defect == "bwd_wrong_layer":
        bwd[9] = bwd[5].copy()
    for s in (0, 1):
        bwd[s] = np.ascontiguousarray(wp[s * 64:s * 64 + 64, :].T)
    for s, m in bwd.items():
        _put(img, OFF_BWD + s * SLICE256, m, sw)
    return img


def _get(img, base, N):
    n, k = np.meshgrid(np.arange(N), np.arange(64), indexing="ij")
    return np.asarray(img).view(F16)[(base + sw128_off(n, k)) // 2]


def check_packed(img, w) -> dict:
    """Decodes every written element of the packed image `img` (uint8) of the weights `w`.  Returns
    {'plain_differ': plain fp16 / fp32 elements not bit-equal to float16(W) / W (zero padding included),
     'fold_outside': W' / b' elements outside the fmaf chain's bound, 'fold_worst': the largest |W' - W'64| in units
     of that bound (0 when exact), 'fold_twins_differ': W' elements of the forward slices that differ from the same
     element of the transposed backward slices}."""
    img = np.asarray(img, np.uint8)
    p = _params(w)
    wp64, wpb, bp64, bpb = fold64(p)
    differ = 0
    for s, m in _plain_slices(p).items():
        got = _get(img, s * SLICE256 if s < 30 else OFF_DIR + (s - 30) * SLICE128, m.shape[0])
        differ += int((got.view(np.uint16) != m.astype(F16).view(np.uint16)).sum())
    for s, m in _bwd_plain(p).items():
        got = _get(img, OFF_BWD + s * SLICE256, 256)
        differ += int((got.view(np.uint16) != m.astype(F16).view(np.uint16)).sum())
    f32 = img[HALF_BYTES:FWD_BYTES].view(F32)
    exp = _f32_region(p, np.zeros(128, F32))
    rest = np.ones(F32_COUNT, bool)
    rest[8 * 256:8 * 256 + 128] = False
    differ += int((f32[rest].view(np.uint32) != exp[rest].view(np.uint32)).sum())
    # folded W' (forward slices 30..33, [n][k]) and its transposed twins (backward slices 0, 1, [n][k] = W'[k][n])
    fwd = np.concatenate([_get(img, OFF_DIR + s * SLICE128, 128) for s in range(4)], 1)        # (128, 256)
    bwd = np.concatenate([_get(img, OFF_BWD + s * SLICE256, 256).T for s in range(2)], 0)        # (128, 256)
    twins = int((fwd.view(np.uint16) != bwd.view(np.uint16)).sum())
    lo = (wp64 - wpb).astype(F16).astype(F64)
    hi = (wp64 + wpb).astype(F16).astype(F64)
    fv = fwd.astype(F64)
    out_w = ~((fv >= lo) & (fv <= hi))
    bv = f32[8 * 256:8 * 256 + 128].astype(F64)
    out_b = ~(np.abs(bv - bp64) <= bpb)
    with np.errstate(divide="ignore", invalid="ignore"):
        ew = np.abs(fv - wp64) / (wpb + 0.5 * np.spacing(np.abs(wp64).astype(F16)).astype(F64))
        eb = np.abs(bv - bp64) / bpb
    worst = float(np.nanmax(np.concatenate([ew.reshape(-1), eb])))
    return {"plain_differ": differ, "fold_outside": int(out_w.sum() + out_b.sum()), "fold_worst": worst,
            "fold_twins_differ": twins}
