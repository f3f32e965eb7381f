"""Numpy reader of the training workspace and float64 references of every backward stage.

The fused training forward leaves per sample, in the workspace, what the backward reads (csrc/render_kernel.cuh
PassBufs); the backward kernels leave their per-sample outputs next to it.  This module

  * mirrors the per-pass part of csrc/capi.cu make_train_layout (`layout`),
  * decodes the tiled 16-bit arrays of csrc/layout.h (`untile`) and the ReLU sign bits the forward's
    epi_hidden writes (csrc/mlp_engine.cuh: bit 2 (j & 15) + e of word j >> 4 of entry (row, q) is the sign of
    column 8 j + 2 q + e; `decode_masks`),
  * recovers the per-level power-of-two gradient scales from the data (`pow2_ratio`),
  * and compares each stage with a float64 reference built from the DEVICE's own stored inputs of that stage
    (`check_*`), so that each comparison isolates one kernel and its bar is set by fp32 / fp16 rounding.

Used by tests/test_gpu_train_stages.py (real workspaces), tests/test_train_tape.py (synthetic ones, with injected
defects) and tools/bwd_debug.py.  Levels: v = 0 is dd (dL/d of the direction layer's pre-activation), v = 1..8
is dpre_{9-v} (dL/d of xyz_encoding_{9-v}'s pre-activation).
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np

F16_MAX = 65504.0
F64 = np.float64
EPS32 = 2.0 ** -23
N_LAYERS = 8
DIR_SLICES = 64            # csrc/bwd_kernels.cuh kDirSlices


# --------------------------------------------------------------------------------------------- layout
def _take(state, nbytes):
    o = state[0]
    state[0] += (nbytes + 1023) // 1024 * 1024
    return o


def layout(n_rays: int, S_c: int, K: int) -> List[dict]:
    """Byte offsets of the per-pass buffers: the first part of csrc/capi.cu make_train_layout."""
    st = [0]
    passes = []
    for ps in range(2 if K > 0 else 1):
        S = S_c + K if ps else S_c
        n = n_rays * S
        npad = (n + 127) // 128 * 128
        P = dict(S=S, n=n, n_pad=npad, n_rays=n_rays)
        P["enc"] = _take(st, npad * 128)
        P["act"] = _take(st, npad * 512 * 8)
        P["mask"] = _take(st, npad * 32 * 8)
        P["d"] = _take(st, npad * 256)
        P["sigma"] = _take(st, npad * 4)
        P["rgb"] = _take(st, npad * 12)
        P["z"] = _take(st, n * 4)
        P["dsigma"] = _take(st, npad * 4)
        P["dprergb"] = _take(st, npad * 12)
        P["dd"] = _take(st, npad * 256)
        P["dpre"] = _take(st, npad * 512 * 8)
        passes.append(P)
    return passes


_SWZ = np.arange(8)[None, :] ^ (np.arange(64)[:, None] & 7)        # (row in block, logical chunk) -> physical chunk


def untile(region: np.ndarray, n_pad: int, C: int, chunks: Optional[np.ndarray] = None) -> np.ndarray:
    """Tiled (n_pad, C) 16-bit array (csrc/layout.h: [64 x 64] blocks, SWIZZLE_128B) -> row-major float16.
    `chunks`: the 64-row chunks to decode (default all), returned in that order."""
    nfb = C // 64
    a = np.asarray(region, np.uint8)[:n_pad * C * 2].reshape(n_pad // 64, nfb, 64, 8, 16)
    if chunks is not None:
        a = a[chunks]
    a = np.take_along_axis(a, _SWZ[None, None, :, :, None], axis=3)
    return np.ascontiguousarray(a.transpose(0, 2, 1, 3, 4)).reshape(-1, C * 2).view(np.float16)


def tile(x: np.ndarray) -> np.ndarray:
    """Inverse of `untile` (row-major (n_pad, C) 16-bit -> the tiled bytes)."""
    n_pad, C = x.shape
    a = np.ascontiguousarray(x.astype(np.float16)).view(np.uint8).reshape(n_pad // 64, 64, C // 64, 8, 16)
    a = a.transpose(0, 2, 1, 3, 4)
    out = np.empty_like(a)
    np.put_along_axis(out, np.broadcast_to(_SWZ[None, None, :, :, None], a.shape), a, axis=3)
    return out.reshape(-1)


_COL = np.arange(256)
_J, _Q, _E = _COL >> 3, (_COL >> 1) & 3, _COL & 1
_WORD, _BIT = _J >> 4, (2 * (_J & 15) + _E).astype(np.uint32)


def decode_masks(m: np.ndarray) -> np.ndarray:
    """(rows, 4, 2) uint32 sign-bit entries of one layer -> (rows, 256) bool 'pre-activation negative' in column
    order.  Entry q of a row belongs to the consumer thread with quad lane q; bit 2 (j & 15) + e of its word j >> 4
    is the sign of column 8 j + 2 q + e (csrc/mlp_engine.cuh epi_hidden)."""
    m = np.asarray(m, np.uint32).reshape(-1, 4, 2)
    return ((m[:, _Q, _WORD] >> _BIT[None, :]) & 1).astype(bool)


def encode_masks(neg: np.ndarray) -> np.ndarray:
    """Inverse of `decode_masks`: (rows, 256) bool -> (rows, 4, 2) uint32."""
    neg = np.asarray(neg, bool)
    out = np.zeros((neg.shape[0], 4, 2), np.uint32)
    for c in range(256):
        out[:, _Q[c], _WORD[c]] |= neg[:, c].astype(np.uint32) << _BIT[c]
    return out


def saturated(region_u16: np.ndarray) -> int:
    """Number of 16-bit gradient elements at +-65504 (the saturating conversion's clamp value)."""
    r = np.asarray(region_u16).view(np.uint16)
    return int(np.count_nonzero((r == 0x7BFF) | (r == 0xFBFF)))


# --------------------------------------------------------------------------------------------- tapes
class Tape:
    """The stored values of one pass, restricted to whole 128-sample tiles (`rows`: their global sample indices,
    padding rows dropped).  Subclasses provide the arrays; accessors return float16 / float32 / bool arrays."""
    S: int
    n: int
    rows: np.ndarray

    def ray_of_rows(self):
        return self.rows // self.S

    def parts(self, tiles: int) -> list:
        """The tape as consecutive parts of at most `tiles` 128-sample tiles each (one part where it has no tiles)."""
        return [self]


class WorkspaceTape(Tape):
    """A pass of a real training workspace (`raw`: its bytes as a uint8 array), decoded on demand."""

    def __init__(self, raw: np.ndarray, P: dict, tiles: Optional[np.ndarray] = None):
        self.raw, self.P = raw, P
        self.S, self.n, self.n_pad = P["S"], P["n"], P["n_pad"]
        n_tiles = self.n_pad // 128
        tiles = np.arange(n_tiles) if tiles is None else np.unique(np.asarray(tiles) % n_tiles)
        self.tiles = tiles
        self.chunks = np.stack([2 * tiles, 2 * tiles + 1], 1).reshape(-1)
        rows = (self.chunks[:, None] * 64 + np.arange(64)[None, :]).reshape(-1)
        self.valid = rows < self.n
        self.rows = rows[self.valid]
        self.all_rows = tiles is None or len(tiles) == n_tiles

    def parts(self, tiles: int) -> list:
        return [WorkspaceTape(self.raw, self.P, self.tiles[i:i + tiles]) for i in range(0, len(self.tiles), tiles)]

    def _f32(self, key, width=1):
        a = np.frombuffer(self.raw, np.float32, self.n_pad * width if key != "z" else self.n, self.P[key])
        if key == "z":
            return a.reshape(-1, self.S)
        a = a.reshape(self.n_pad, width)[self.rows]
        return a[:, 0] if width == 1 else a

    def _tiled(self, off, C):
        return untile(self.raw[off:off + self.n_pad * C * 2], self.n_pad, C, self.chunks)[self.valid]

    def z(self):
        return self._f32("z")

    def sigma(self):
        return self._f32("sigma")

    def rgb(self):
        return self._f32("rgb", 3)

    def dsigma(self):
        return self._f32("dsigma")

    def dprergb(self):
        return self._f32("dprergb", 3)

    def enc(self):
        return self._tiled(self.P["enc"], 64)

    def h(self, l):          # output of xyz_encoding_l, l = 1..8
        return self._tiled(self.P["act"] + (l - 1) * self.n_pad * 512, 256)

    def dpre(self, l):       # dL/d pre-activation of xyz_encoding_l (scaled), l = 1..8
        return self._tiled(self.P["dpre"] + (l - 1) * self.n_pad * 512, 256)

    def d(self):
        return self._tiled(self.P["d"], 128)

    def dd(self):
        return self._tiled(self.P["dd"], 128)

    def neg(self, l):
        m = np.frombuffer(self.raw, np.uint32, self.n_pad * 8, self.P["mask"] + (l - 1) * self.n_pad * 32)
        return decode_masks(m.reshape(self.n_pad, 4, 2)[self.rows])

    def saturated(self):
        """Saturated elements over ALL rows of dd and dpre_1..8."""
        P = self.P
        return saturated(self.raw[P["dd"]:P["dd"] + P["n_pad"] * 256]) + \
            saturated(self.raw[P["dpre"]:P["dpre"] + P["n_pad"] * 512 * 8])


class ArrayTape(Tape):
    """A tape held as arrays (all rows), e.g. a synthetic device built in numpy."""

    def __init__(self, S, arrays: dict):
        self.S = S
        self.a = arrays
        self.n = arrays["sigma"].shape[0]
        self.rows = np.arange(self.n)
        self.all_rows = True

    def z(self):
        return self.a["z"]

    def sigma(self):
        return self.a["sigma"]

    def rgb(self):
        return self.a["rgb"]

    def dsigma(self):
        return self.a["dsigma"]

    def dprergb(self):
        return self.a["dprergb"]

    def enc(self):
        return self.a["enc"]

    def h(self, l):
        return self.a["h"][l - 1]

    def dpre(self, l):
        return self.a["dpre"][l - 1]

    def d(self):
        return self.a["d"]

    def dd(self):
        return self.a["dd"]

    def neg(self, l):
        return self.a["neg"][l - 1]

    def saturated(self):
        return sum(int(np.count_nonzero(np.abs(x.astype(F64)) >= F16_MAX)) for x in [self.a["dd"]] + self.a["dpre"])


# --------------------------------------------------------------------------------------------- operands
def r16(x):
    return np.asarray(x, np.float32).astype(np.float16).astype(F64)


def ulp16(x):
    """Spacing of float16 at |x| (2^-24 in the subnormal range)."""
    return np.spacing(np.abs(np.asarray(x, F64)).astype(np.float16)).astype(F64)


def fold(w: Dict[str, np.ndarray]):
    """W' = W_dir[:, :256] W_final and b' = W_dir[:, :256] b_final + b_dir as the pack kernel forms them (fp32,
    one fused multiply-add per term in increasing m; csrc/aux_kernels.cuh)."""
    wd = w["dir_encoding.0.weight"][:, :256].astype(F64)
    wf = w["xyz_encoding_final.weight"].astype(F64)
    bf = w["xyz_encoding_final.bias"].astype(F64)
    acc = np.zeros((128, 256), np.float32)
    bacc = w["dir_encoding.0.bias"].astype(np.float32).copy()
    for m in range(256):
        acc = (wd[:, m:m + 1] * wf[m][None, :] + acc).astype(np.float32)
        bacc = (wd[:, m] * bf[m] + bacc).astype(np.float32)
    return acc, bacc


class Net:
    """The operands of one network as the kernels use them: fp16-rounded big-layer weights (float64 arrays),
    the folded direction layer, fp32 heads."""

    def __init__(self, w: Dict[str, np.ndarray]):
        self.w = w
        self.W = [None] + [r16(w[f"xyz_encoding_{l}.0.weight"]) for l in range(1, 9)]
        self.b = [None] + [w[f"xyz_encoding_{l}.0.bias"].astype(F64) for l in range(1, 9)]
        wp, bp = fold(w)
        self.Wp = r16(wp)                                  # (128, 256)
        self.bp = bp.astype(F64)
        self.Wdir = w["dir_encoding.0.weight"][:, 256:283].astype(F64)
        self.wsig = w["sigma.weight"][0].astype(F64)
        self.bsig = float(w["sigma.bias"][0])
        self.Wrgb = w["rgb.0.weight"].astype(F64)          # (3, 128)
        self.brgb = w["rgb.0.bias"].astype(F64)

    def Wchain(self, l):
        """The matrix step l of the dgrad chain multiplies dpre_l by (only the hidden columns of layer 5)."""
        return self.W[l][:, 63:] if l == 5 else self.W[l]


# --------------------------------------------------------------------------------------------- metrics
def ulp_err(dev, ref, absdot, scale=1.0):
    """max |dev - ref| in units of (one fp16 ulp of ref + one fp32 ulp of the accumulation sum_k |a_k b_k|)."""
    dev, ref = np.asarray(dev, F64), np.asarray(ref, F64)
    if dev.size == 0:
        return 0.0
    den = ulp16(ref) + EPS32 * np.abs(scale) * np.asarray(absdot, F64)
    return float((np.abs(dev - ref) / den).max())


def pow2_ratio(got, ref) -> float:
    """The power of two p with got ~ p ref (the device's per-level scale).  Asserts that the median ratio over the
    large, unsaturated elements is a power of two to within fp16 rounding."""
    got, ref = np.asarray(got, F64), np.asarray(ref, F64)
    nz = np.abs(ref[ref != 0])
    if nz.size == 0:
        return 1.0
    m = (np.abs(ref) > 0.1 * np.quantile(nz, 0.999)) & (got != 0) & (np.abs(got) < F16_MAX)
    if not m.any():
        return 1.0
    r = float(np.median(got[m] / ref[m]))
    assert r > 0, f"scale ratio {r} is not positive"
    p = 2.0 ** np.round(np.log2(r))
    assert abs(r / p - 1) < 2.0 ** -8, f"recovered scale ratio {r!r} is not a power of two"
    return float(p)


def rel_l2(dev, ref):
    dev, ref = np.asarray(dev, F64), np.asarray(ref, F64)
    return float(np.linalg.norm(dev - ref) / max(np.linalg.norm(ref), 1e-300))


def max_rel(dev, ref):
    dev, ref = np.asarray(dev, F64), np.asarray(ref, F64)
    return float(np.abs(dev - ref).max() / max(np.abs(ref).max(), 1e-300))


# --------------------------------------------------------------------------------------------- stages
def check_forward(tape: Tape, net: Net, dir_emb: np.ndarray) -> dict:
    """Each forward layer on the device's own input of that layer.  Returns
    {'h1'..'h8', 'd': ulp errors; 'sigma', 'rgb': errors in units of 2^-11 sum |w h| (the heads use the fp32
    activations, the tape holds their fp16 roundings)}."""
    out = {}
    enc = tape.enc().astype(F64)
    out["enc_col63"] = float(np.abs(enc[:, 63]).max()) if len(enc) else 0.0
    x = enc[:, :63]
    prev = x
    for l in range(1, 9):
        inp = np.concatenate([x, prev], 1) if l == 5 else prev
        W = net.W[l]
        ref = np.maximum(inp @ W.T + net.b[l], 0.0)
        dev = tape.h(l).astype(F64)
        out[f"h{l}"] = ulp_err(dev, ref, np.abs(inp) @ np.abs(W).T)
        prev = dev
    h8 = prev
    rays = tape.ray_of_rows()
    dbias = net.bp[None, :] + dir_emb[rays].astype(F64) @ net.Wdir.T
    ref = np.maximum(h8 @ net.Wp.T + dbias, 0.0)
    d = tape.d().astype(F64)
    out["d"] = ulp_err(d, ref, np.abs(h8) @ np.abs(net.Wp).T + np.abs(dir_emb[rays]) @ np.abs(net.Wdir).T)
    sig = net.bsig + h8 @ net.wsig
    den = 2.0 ** -11 * (np.abs(h8) @ np.abs(net.wsig)) + 1e-30
    out["sigma"] = float((np.abs(tape.sigma() - sig) / den).max()) if len(den) else 0.0
    pre = d @ net.Wrgb.T + net.brgb
    rgb = 1.0 / (1.0 + np.exp(-pre))
    den = 0.25 * 2.0 ** -11 * (np.abs(d) @ np.abs(net.Wrgb).T) + 2.0 ** -24
    out["rgb"] = float((np.abs(tape.rgb() - rgb) / den).max()) if len(den) else 0.0
    return out


def check_masks(tape: Tape) -> dict:
    """Sign bits against h == 0 (h is post-ReLU, so h >= 0).  'illegal': bit says negative but h > 0 - never
    allowed.  'legal': bit says positive and h is exactly 0 (a positive pre-activation below half the smallest
    fp16 subnormal); returned as a fraction of the elements."""
    illegal = legal = total = 0
    for l in range(1, 9):
        neg, h = tape.neg(l), tape.h(l)
        illegal += int(np.count_nonzero(neg & (h != 0)))
        legal += int(np.count_nonzero(~neg & (h == 0)))
        total += neg.size
    return {"illegal": illegal, "legal_frac": legal / max(total, 1)}


def dd_reference(tape: Tape, net: Net):
    """dL/d(direction-layer pre-activation), float64 and un-scaled, from the device's d rgb_pre and d."""
    dp = tape.dprergb().astype(F64)
    return (dp @ net.Wrgb) * (tape.d().astype(F64) > 0), np.abs(dp) @ np.abs(net.Wrgb)


def check_chain(tape: Tape, net: Net) -> dict:
    """dd, then every step of the dgrad chain on the device's own input of that step, and the whole chain in
    float64 on the device's masks.  Returns the recovered scales s[0..8] (level v), per-step ulp errors
    'step{v}', per-level 'acc{v}' relative L2 and 'accmax{v}' (max error / max |ref|) of the accumulated chain."""
    out = {}
    s = [0.0] * 9
    ref0, absd = dd_reference(tape, net)
    dd = tape.dd().astype(F64)
    s[0] = pow2_ratio(dd, ref0)
    out["step0"] = ulp_err(dd, ref0 * s[0], absd, s[0])
    dsig = tape.dsigma().astype(F64)
    # first step: in units of level 0
    a = dd @ net.Wp + (dsig * s[0])[:, None] * net.wsig[None, :]
    absa = np.abs(dd) @ np.abs(net.Wp) + np.abs(dsig * s[0])[:, None] * np.abs(net.wsig)[None, :]
    chain = ref0 @ net.Wp + dsig[:, None] * net.wsig[None, :]         # float64 chain from the float64 seed
    prev_s = s[0]
    for v in range(1, 9):
        l = 9 - v
        keep = ~tape.neg(l)
        dev = tape.dpre(l).astype(F64)
        ratio = pow2_ratio(dev, a * keep)
        s[v] = prev_s * ratio
        out[f"step{v}"] = ulp_err(dev, a * keep * ratio, absa * keep, ratio)
        chain = chain * keep
        out[f"acc{v}"] = rel_l2(dev / s[v], chain)
        out[f"accmax{v}"] = max_rel(dev / s[v], chain)
        if l > 1:
            Wc = net.Wchain(l)
            a, absa = dev @ Wc, np.abs(dev) @ np.abs(Wc)
            chain = chain @ Wc
        prev_s = s[v]
    out["scales"] = s
    out["saturated"] = tape.saturated()
    return out


def check_composite(tape: Tape, rays, g_rgb, g_depth, g_opac, noise, noise_std, white_back):
    """Compositing backward on the device's sigma / rgb / z: d sigma and d rgb_pre, errors relative to the pass's
    largest reference value.  'last' is the last sample of each ray alone (ill-conditioned under sigma noise)."""
    from oracle import nerf_oracle_grad as og
    assert tape.all_rows
    n_rays, S = tape.z().shape
    sig = tape.sigma().reshape(n_rays, S)
    rgb = tape.rgb().reshape(n_rays, S, 3)
    g = np.zeros((n_rays, 3), np.float32) if g_rgb is None else g_rgb
    dsig, drgb = og.volume_render_backward(sig, rgb, tape.z(), rays[:, 3:6], noise, noise_std, white_back, g,
                                           g_depth, g_opac)
    dsig_dev = tape.dsigma().reshape(n_rays, S)
    dp_ref = drgb.astype(F64) * rgb * (1 - rgb.astype(F64))
    dp_dev = tape.dprergb().reshape(n_rays, S, 3)
    den_s = max(np.abs(dsig).max(), 1e-30)
    den_p = max(np.abs(dp_ref).max(), 1e-30)
    es = np.abs(dsig_dev - dsig.astype(F64)) / den_s
    return {"dsigma": float(es[:, :-1].max()) if S > 1 else 0.0, "dsigma_last": float(es[:, -1].max()),
            "dprergb": float((np.abs(dp_dev - dp_ref) / den_p).max())}


def column_sums(a16: np.ndarray, device="cpu") -> np.ndarray:
    """Column sums of a stored 16-bit gradient array the way the wgrad kernel's reduction warps form them: in each
    64-row chunk, rows h 32 + 4 i + p (i = 0..7) are added in fp16, one correctly rounded addition at a time (as
    add.rn.f16x2 does), for each (h, p); those 8-row sums are then exact inputs of a float64 sum.  What is left
    against the device is fp32 summation error only.  Computed in torch on `device`: the float64 sum of two fp16
    values is exact, and its rounding to fp16 through fp32 rounds once (24 >= 2 * 11 + 2 bits)."""
    import torch
    a = torch.from_numpy(np.ascontiguousarray(a16, np.float16)).to(device)
    n, C = a.shape
    pad = torch.zeros(((n + 63) // 64 * 64, C), dtype=torch.float16, device=device)
    pad[:n] = a
    x = pad.view(-1, 2, 8, 4, C)               # [chunk, h, i, p, column] = row h 32 + 4 i + p
    acc = x[:, :, 0]
    for i in range(1, 8):
        acc = (acc.double() + x[:, :, i].double()).half()
    return acc.double().sum((0, 1, 2)).cpu().numpy()


def reference_grads(tape: Tape, net: Net, scales, dir_emb: np.ndarray, device="cpu",
                    tiles_per_part: int = 2048) -> Dict[str, np.ndarray]:
    """The 24 gradient tensors as float64 contractions of the device's own operands (all samples): the wgrad
    GEMMs sum_s dpre_l^T h_{l-1} / s_l and bias sums (with the kernel's fp16 8-row pre-sums, `column_sums`),
    layer 5 as its 63 encoding and 256 hidden columns, the heads, W' from dd, the direction part from the per-ray
    sums of the un-scaled dd, and the unfolding of W' (csrc/bwd_kernels.cuh unfold_kernel).  The sums over samples
    run over `tape.parts(tiles_per_part)` in torch float64 on `device`, so a pass of millions of samples is never
    decoded whole; the parts start on tile boundaries, which keeps every 64-row pre-sum of `column_sums` whole."""
    import torch
    assert tape.all_rows
    w = net.w
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device).double()     # stored 16-bit values go as they are
    acc = {}

    def add(k, v):
        acc[k] = v if k not in acc else acc[k] + v
    n_rays = tape.n // tape.S
    raysum = torch.zeros(n_rays, 128, dtype=torch.float64, device=device)
    for part in tape.parts(tiles_per_part):
        enc = T(part.enc()[:, :63])
        for l in range(1, 9):
            a16 = part.dpre(l)
            if l == 1:
                B = enc
            elif l == 5:
                B = torch.cat([enc, T(part.h(4))], 1)
            else:
                B = T(part.h(l - 1))
            add(f"xyz_encoding_{l}.0.weight", T(a16).T @ B)
            add(f"xyz_encoding_{l}.0.bias", T(column_sums(a16, device)))
        h8 = T(part.h(8))
        dsig = T(part.dsigma())
        add("sigma.weight", (dsig @ h8)[None, :])
        add("sigma.bias", dsig.sum()[None])
        dp = T(part.dprergb())
        add("rgb.0.weight", dp.T @ T(part.d()))
        add("rgb.0.bias", dp.sum(0))
        dd16 = part.dd()
        add("gWp", T(dd16).T @ h8)
        add("gbp", T(column_sums(dd16, device)))
        ref0, _ = dd_reference(part, net)
        raysum.index_add_(0, torch.from_numpy(part.ray_of_rows()).to(device), T(ref0))
    g = {k: v.cpu().numpy() for k, v in acc.items()}
    for l in range(1, 9):
        g[f"xyz_encoding_{l}.0.weight"] /= scales[9 - l]
        g[f"xyz_encoding_{l}.0.bias"] /= scales[9 - l]
    gWp, gbp = g.pop("gWp") / scales[0], g.pop("gbp") / scales[0]
    raysum = raysum.cpu().numpy()
    Wd = w["dir_encoding.0.weight"][:, :256].astype(F64)
    Wf = w["xyz_encoding_final.weight"].astype(F64)
    bf = w["xyz_encoding_final.bias"].astype(F64)
    g["dir_encoding.0.weight"] = np.concatenate([gWp @ Wf.T + np.outer(gbp, bf), raysum.T @ dir_emb.astype(F64)], 1)
    g["dir_encoding.0.bias"] = gbp
    g["xyz_encoding_final.weight"] = Wd.T @ gWp
    g["xyz_encoding_final.bias"] = Wd.T @ gbp
    return g


def check_grads(dev: Dict[str, np.ndarray], ref: Dict[str, np.ndarray]) -> Dict[str, tuple]:
    """Per tensor: (relative L2 error, max abs error / max |ref|) over every element."""
    out = {}
    for k, r in ref.items():
        d = np.asarray(dev[k], F64).reshape(r.shape)
        out[k] = (rel_l2(d, r), max_rel(d, r))
    return out


# --------------------------------------------------------------------------------------------- bars
# Worst values measured on one H100 80GB HBM3 (700 W power limit) over the case matrix of
# tests/test_gpu_train_stages.py stand next to the bars.  The ulp-type metrics are >= 0.5 by construction (one
# rounding to fp16), so their bars leave ~2x over the worst case; the relative ones leave ~10x.
BARS = {
    "h": 2.0,                # units of (fp16 ulp + 2^-23 sum |w h|); worst 1.16 (layer 5, trained weights)
    "d": 2.0,                # same units; worst 0.70
    "head": 2.0,             # units of 2^-11 sum |w h|; worst 0.33
    "enc": 1.0,              # units of (fp16 ulp + 2^-20, the MUFU sin/cos error); worst 0.50
    "mask_legal": 1e-5,      # fraction of sign bits 'positive' with h == 0; worst 6.9e-7
    "dd": 1.0,               # units of (fp16 ulp + 2^-23 sum |w dp|); worst 0.50
    "step": 2.0,             # one dgrad chain step, same units; worst 0.78
    "acc": 5e-3,             # relative L2 per level of the chain vs float64 on the same masks; worst 6.8e-4
    "composite": 1e-3,       # max error / max |ref| of d sigma, d rgb_pre; worst 1.2e-4
    "composite_last": 1e-3,  # the last sample of a ray under sigma noise; worst 0
    "grad_rel": 3e-4,        # relative L2 per gradient tensor; worst 3.1e-5 (1024 rays; biases 3.6e-6)
    "grad_max": 3e-4,        # max abs error / max |ref| per tensor; worst 3.3e-5 (biases 4.6e-6)
}


def failures(forward=None, masks=None, chain=None, composite=None, grads=None, noise=False) -> List[str]:
    """The bars of BARS applied to the outputs of the check_* functions; returns the list of violations."""
    bad = []
    if forward is not None:
        for k, v in forward.items():
            bar = {"sigma": BARS["head"], "rgb": BARS["head"], "d": BARS["d"], "enc_col63": 0.0}.get(k, BARS["h"])
            if not v <= bar:
                bad.append(f"forward {k}: {v:.3g} > {bar}")
    if masks is not None:
        if masks["illegal"]:
            bad.append(f"masks: {masks['illegal']} sign bits contradict h")
        if not masks["legal_frac"] <= BARS["mask_legal"]:
            bad.append(f"masks: legal exceptions {masks['legal_frac']:.3g} > {BARS['mask_legal']}")
    if chain is not None:
        if chain["saturated"]:
            bad.append(f"chain: {chain['saturated']} gradient elements saturated at 65504")
        for v in range(9):
            bar = BARS["dd"] if v == 0 else BARS["step"]
            if not chain[f"step{v}"] <= bar:
                bad.append(f"chain step{v}: {chain[f'step{v}']:.3g} ulp > {bar}")
            if v and not chain[f"acc{v}"] <= BARS["acc"]:
                bad.append(f"chain acc{v}: {chain[f'acc{v}']:.3g} > {BARS['acc']}")
    if composite is not None:
        for k, v in composite.items():
            bar = BARS["composite_last"] if (k == "dsigma_last" and noise) else BARS["composite"]
            if not v <= bar:
                bad.append(f"composite {k}: {v:.3g} > {bar}")
    if grads is not None:
        for k, (r, m) in grads.items():
            if not (r <= BARS["grad_rel"] and m <= BARS["grad_max"]):
                bad.append(f"grad {k}: rel {r:.3g} max {m:.3g}")
    return bad
