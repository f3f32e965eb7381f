"""The float64 restatement the degenerate-ray GPU tests judge poisoned rays by, and their comparators, without a GPU.

`render64` is render_rays (models/rendering.py:175-244) in float64 with the kernel's one documented divergence
applied: sigma -> fmax(sigma, 0), so a NaN sigma is empty space (DESIGN.md section 5).  Where the reference's own fp32
arithmetic decides whether a value is finite, fp32 is kept, because that is what the reference computes:

  * the coarse depths (orc.coarse_depths; the kernel's are bitwise equal): near = 0 with use_disp gives 1 / (inf 0);
  * the bin mid-points 0.5 (z_i + z_(i+1)), which overflow for far ~ 3e38;
  * |d| (`dnorm`): torch's fp32 norm, whose squared sum under- and overflows (|d| ~ 1e-30, ~ 1e20).  The caller
    passes torch's fp32 value; the default here is that fp32 sum.

tests/test_gpu_degenerate_rays.py compares the device's finiteness pattern per output with `render64`'s
(`pattern_mismatch`), and z_vals_fine bitwise with tests/render_tape.py z_fine (torch.sort's NaN-last order).
Hand-computed rays pin `render64` below.  `merge_ranks` and `u_slots` restate the kernel's rank computations
element by element, NaN-aware as now and with the plain < / == they used before; the plain ones leave a slot holding
an earlier ray's value, and both the emulation comparison and the launch-independence comparison reject that.
"""
import numpy as np

from oracle import nerf_oracle as orc
from tests import render_tape as rt

F32, F64 = np.float32, np.float64
OUT_KEYS = ("rgb_coarse", "depth_coarse", "opacity_coarse", "weights_coarse", "rgb_fine", "depth_fine",
            "opacity_fine", "weights_fine")


def dnorm32(d):
    """sqrt of the fp32 sum of squares (torch.norm of fp32 directions on the device)."""
    d = np.asarray(d, F32)
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        s = ((d[:, 0] * d[:, 0]).astype(F32) + (d[:, 1] * d[:, 1]).astype(F32)).astype(F32)
        s = (s + (d[:, 2] * d[:, 2]).astype(F32)).astype(F32)
    return np.sqrt(s).astype(F32)


def _embed64(x, n_freqs):
    out = [x]
    for k in range(n_freqs):
        out += [np.sin(2.0 ** k * x), np.cos(2.0 ** k * x)]
    return np.concatenate(out, -1)


def _mlp64(w, x63, dir27):
    """NeRF.forward in float64; np.maximum keeps NaN as torch.relu does.  -> (sigma, rgb)."""
    L = lambda name, h: h @ w[name + ".weight"].astype(F64).T + w[name + ".bias"].astype(F64)  # noqa: E731
    h = x63
    for i in range(8):
        if i == 4:
            h = np.concatenate([x63, h], -1)
        h = np.maximum(L(f"xyz_encoding_{i + 1}.0", h), 0.0)
    sigma = L("sigma", h)[:, 0]
    d = np.maximum(L("dir_encoding.0", np.concatenate([L("xyz_encoding_final", h), dir27], -1)), 0.0)
    return sigma, 1.0 / (1.0 + np.exp(-L("rgb.0", d)))


def _pass64(w, rays, z, dn, noise, noise_std, white_back):
    """One pass: points, MLP, compositing with fmax(sigma, 0).  -> (weights, rgb, depth, opacity, max finite |x|)."""
    n, S = z.shape
    o, d = rays[:, None, :3].astype(F64), rays[:, None, 3:6].astype(F64)
    x = (o + d * z[:, :, None]).reshape(-1, 3)
    dir27 = np.repeat(_embed64(rays[:, 3:6].astype(F64), 4), S, 0)
    sig, rgb = _mlp64(w, _embed64(x, 10), dir27)
    sig, rgb = sig.reshape(n, S), rgb.reshape(n, S, 3)
    if noise is not None:
        sig = sig + noise.astype(F64) * noise_std
    delta = np.concatenate([z[:, 1:] - z[:, :-1], np.full((n, 1), 1e10)], 1) * dn.astype(F64)[:, None]
    alpha = 1.0 - np.exp(-delta * np.fmax(sig, 0.0))
    T = np.concatenate([np.ones((n, 1)), np.cumprod(1.0 - alpha + 1e-10, 1)[:, :-1]], 1)
    wt = alpha * T
    opac = wt.sum(1)
    col = (wt[..., None] * rgb).sum(1)
    if white_back:
        col = col + (1.0 - opac)[:, None]
    ax = np.abs(x.reshape(n, S, 3))
    xmax = np.where(np.isfinite(ax), ax, 0.0).max((1, 2))
    return wt, col, (wt * z).sum(1), opac, xmax


def render64(ws, rays, S, K, use_disp=False, perturb=0.0, noise_std=0.0, white_back=False, rnd=None, dnorm=None):
    """render_rays in float64 with sigma -> fmax(sigma, 0) (module docstring).  ``rnd``: perturb_rand, u_rand,
    noise_coarse, noise_fine as the kernel takes them.  Returns the OUT_KEYS, z_vals_fine and 'xmax' (per ray, the
    largest finite |o + d z| of either pass)."""
    rnd = rnd or {}
    rays = np.asarray(rays, F32)
    dn = dnorm32(rays[:, 3:6]) if dnorm is None else np.asarray(dnorm, F32)
    with np.errstate(all="ignore"):
        zc32 = orc.coarse_depths(rays, S, use_disp, perturb, rnd.get("perturb_rand"))
        zc = zc32.astype(F64)
        nz = rnd.get("noise_coarse") if noise_std > 0 else None
        w, c, dp, op, xm = _pass64(ws[0], rays, zc, dn, nz, noise_std, white_back)
        res = dict(rgb_coarse=c, depth_coarse=dp, opacity_coarse=op, weights_coarse=w, xmax=xm)
        if K:
            wp = w[:, 1:-1] + 1e-5
            cdf = np.concatenate([np.zeros((len(w), 1)), np.cumsum(wp / wp.sum(1, keepdims=True), 1)], 1)
            u = rt.fine_uniforms(len(rays), K, perturb, rnd.get("u_rand")).astype(F64)
            bins = rt.bins_from_depths(zc32).astype(F64)                  # fp32 mid-points, as the reference
            inds = orc.searchsorted(cdf, u, side="right")
            below, above = np.maximum(inds - 1, 0), np.minimum(inds, S - 2)
            g = lambda a, i: np.take_along_axis(a, i, 1)  # noqa: E731
            den = g(cdf, above) - g(cdf, below)
            den = np.where(den < 1e-5, 1.0, den)
            znew = g(bins, below) + (u - g(cdf, below)) / den * (g(bins, above) - g(bins, below))
            zf = np.sort(np.concatenate([zc, znew], 1), 1)               # NaN last, as torch.sort
            nf = rnd.get("noise_fine") if noise_std > 0 else None
            w, c, dp, op, xm = _pass64(ws[1], rays, zf, dn, nf, noise_std, white_back)
            res.update(rgb_fine=c, depth_fine=dp, opacity_fine=op, weights_fine=w, z_vals_fine=zf,
                       xmax=np.maximum(res["xmax"], xm))
    return res


def pattern_mismatch(dev: dict, ref: dict, rows) -> dict:
    """{key: number of elements of rows `rows` whose finiteness differs between the device's outputs and render64's}
    for the OUT_KEYS both hold; keys without a difference are left out."""
    out = {}
    for k in OUT_KEYS:
        if k in dev and k in ref:
            bad = int((np.isfinite(np.asarray(dev[k])[rows]) != np.isfinite(np.asarray(ref[k])[rows])).sum())
            if bad:
                out[k] = bad
    return out


def position_mismatch(a: dict, b: dict, rows_a, rows_b) -> dict:
    """{key: elements that differ (NaN equal to NaN)} between rows `rows_a` of one render and `rows_b` of another."""
    out = {}
    for k in a:
        if k in b:
            x, y = np.asarray(a[k])[rows_a], np.asarray(b[k])[rows_b]
            bad = int((~((x == y) | (np.isnan(x) & np.isnan(y)))).sum())
            if bad:
                out[k] = bad
    return out


# ------------------------------------------------------------------------------------------------ CPU tests
def _ws():
    return [orc.make_weights(1), orc.make_weights(2)]


def _ray(o=(0.0, 0.0, 4.0), d=(0.0, 0.0, -1.0), near=2.0, far=6.0):
    return np.array([[*o, *d, near, far]], F32)


def test_zero_direction_is_transparent():
    """d = 0: |d| = 0, every delta 0, alpha 0: weights 0, opacity 0, depth 0, rgb the background; the fine pass
    resamples the uniform pdf of the 1e-5 padding."""
    r = render64(_ws(), _ray(d=(0.0, 0.0, 0.0)), 64, 64, white_back=True)
    for k in ("weights_coarse", "weights_fine", "opacity_coarse", "opacity_fine", "depth_coarse", "depth_fine"):
        assert np.all(r[k] == 0), k
    assert np.all(r["rgb_fine"] == 1.0) and np.all(np.isfinite(r["z_vals_fine"]))
    assert np.all(np.diff(r["z_vals_fine"][0]) >= 0) and r["z_vals_fine"][0, 0] == 2 and r["z_vals_fine"][0, -1] == 6


def test_nan_origin_is_empty_space_with_nan_colour():
    """A NaN origin: every point NaN, sigma NaN -> empty (weights, opacity, depth 0), the colour NaN (0 x NaN)."""
    r = render64(_ws(), _ray(o=(np.nan, 0.0, 4.0)), 64, 64, white_back=True)
    for k in ("weights_coarse", "opacity_coarse", "depth_coarse", "weights_fine", "opacity_fine", "depth_fine"):
        assert np.all(r[k] == 0), k
    assert np.all(np.isnan(r["rgb_coarse"])) and np.all(np.isnan(r["rgb_fine"]))


def test_infinite_far_is_nan():
    """far = +inf: the first coarse depth is near 1 + inf 0 = NaN, the others inf; deltas NaN: every output NaN,
    z_vals_fine NaN and inf with the NaNs last."""
    r = render64(_ws(), _ray(far=np.inf), 64, 64)
    for k in OUT_KEYS:
        assert np.all(np.isnan(r[k])), k
    z = r["z_vals_fine"][0]
    assert np.isnan(z[-1]) and not np.isnan(z[0]) or np.all(np.isnan(z))


def test_ndc_use_disp_near_zero():
    """NDC, use_disp, near = 0: 1 / near = inf; the coarse depths are 1 / inf = 0 except the last, 1 / (inf 0) =
    NaN (the reference's own fp32 value).  The last delta is 1e10 |d| at a NaN point (sigma NaN: empty), the one
    before it NaN - 0: weights NaN from sample S - 2 on, so every output of both passes is NaN."""
    rays = orc.make_rays(1, 3, "ndc")
    zc = orc.coarse_depths(rays, 64, True, 0.0)
    assert np.all(zc[0, :-1] == 0) and np.isnan(zc[0, -1])
    r = render64(_ws(), rays, 64, 64, use_disp=True)
    assert np.all(r["weights_coarse"][0, :62] == 0) and np.all(np.isnan(r["weights_coarse"][0, 62:]))
    for k in ("rgb_coarse", "opacity_coarse", "rgb_fine", "opacity_fine"):
        assert np.all(np.isnan(r[k])), k


def test_restatement_agrees_with_fp32_oracle_on_clean_rays():
    """On ordinary rays render64 is the fp32 oracle to fp32 rounding."""
    rays = orc.make_rays(6, 5)
    a = render64(_ws(), rays, 32, 32, white_back=True)
    b = orc.render_rays(_ws(), rays, 32, False, 0.0, 0.0, 32, True)
    for k in ("rgb_coarse", "rgb_fine", "opacity_fine"):
        np.testing.assert_allclose(a[k], b[k], atol=2e-4)


def _before(a, b, nan_aware):
    """csrc/render_kernel.cuh sort_before (nan_aware) or the plain a < b the merge used before."""
    return (a < b) | (nan_aware & np.isnan(b) & ~np.isnan(a))


def _tied(a, b, nan_aware):
    return (a == b) | (nan_aware & np.isnan(a) & np.isnan(b))


def merge_ranks(zc, zn, slots, nan_aware=True):
    """The kernel's merge of ONE ray, element by element: the inversion (and, nan_aware, NaN) check, then ranks from
    the two binary searches or from exhaustive counting, each element written to slots[rank].  `slots` holds what
    the shared-memory array held before (the depths of the ray merged earlier); returns the written copy."""
    zc, zn = np.asarray(zc, F32), np.asarray(zn, F32)
    Sc, K = len(zc), len(zn)
    v_all = np.concatenate([zc, zn])
    inv = bool((zc[1:] < zc[:-1]).any() or (zn[1:] < zn[:-1]).any())
    if nan_aware:
        inv |= bool(np.isnan(v_all).any())
    out = np.array(slots, F32).copy()
    for i, v in enumerate(v_all):
        if not inv:
            other, lo, hi = (zn, 0, K) if i < Sc else (zc, 0, Sc)
            while lo < hi:                         # lower_bound (coarse element) / upper_bound (new element)
                mid = (lo + hi) >> 1
                right = other[mid] < v if i < Sc else other[mid] <= v
                lo, hi = (mid + 1, hi) if right else (lo, mid)
            rank = lo + (i if i < Sc else i - Sc)
        else:
            q = np.arange(Sc + K)
            rank = int((_before(v_all, v, nan_aware) | (_tied(v_all, v, nan_aware) & (q < i))).sum())
        out[rank] = v
    return out


def u_slots(u, prev, nan_aware=True):
    """The slot of each caller-supplied u (its rank, ties by index); returns the slots after the u's are written,
    `prev` where no u was written (the kernel's array then keeps an earlier ray's value)."""
    u = np.asarray(u, F32)
    out = np.full(len(u), prev, F32)
    q = np.arange(len(u))
    for j, uj in enumerate(u):
        out[int((_before(u, uj, nan_aware) | (_tied(u, uj, nan_aware) & (q < j))).sum())] = uj
    return out


def _lists(seed, nan_at=None):
    rs = np.random.RandomState(seed)
    zc = np.sort(rs.uniform(2, 6, 64)).astype(F32)
    zn = np.sort(rs.uniform(2, 6, 64)).astype(F32)
    if nan_at is not None:
        lst, i = nan_at
        (zc if lst == "coarse" else zn)[i] = np.nan
    return zc, zn


def test_merge_ranks_match_torch_sort_and_ignore_stale_slots():
    """The NaN-aware rank merge gives np.sort's NaN-last list whatever the slots held before, on clean lists, lists
    with an inversion, NaN in either list (first, middle, last) and all-NaN new depths."""
    cases_ = [_lists(0), _lists(1, ("coarse", 0)), _lists(2, ("coarse", 30)), _lists(3, ("new", 63)),
              _lists(4, ("new", 10))]
    zc, zn = _lists(5)
    zc[7], zc[8] = zc[8], zc[7]                     # a 1-ulp style inversion: exhaustive branch
    cases_ += [(zc, zn), (_lists(6)[0], np.full(64, np.nan, F32))]
    for zc, zn in cases_:
        want = np.sort(np.concatenate([zc, zn]))
        for prev in (np.full(128, 4.25, F32), np.full(128, -1.0, F32)):
            got = merge_ranks(zc, zn, prev)
            assert np.array_equal(got, want, equal_nan=True)


def test_comparators_reject_the_plain_comparison_merge():
    """The merge as it compared before (plain < / ==): with a NaN in a list the check finds no inversion, the binary
    searches give colliding ranks and a slot keeps the depth of the ray merged before.  Both GPU comparisons reject
    that: the result differs from the NaN-last emulation (render_tape.z_fine's np.sort), and two launches whose
    previous ray differed give different results (position_mismatch)."""
    for lst, i in (("coarse", 0), ("coarse", 30), ("new", 10), ("new", 63)):
        zc, zn = _lists(7 + i, (lst, i))
        want = np.sort(np.concatenate([zc, zn]))
        a = merge_ranks(zc, zn, np.full(128, 4.25, F32), nan_aware=False)
        b = merge_ranks(zc, zn, np.full(128, 5.5, F32), nan_aware=False)
        assert dr_mismatch(a, want), (lst, i)
        assert dr_mismatch(a, b), (lst, i)
        assert not dr_mismatch(merge_ranks(zc, zn, np.full(128, 4.25, F32)),
                               merge_ranks(zc, zn, np.full(128, 5.5, F32)))


def test_u_slots_with_a_nan():
    """Caller-supplied u's with a NaN: NaN-aware slots are a permutation with the NaN last; plain comparisons put the
    NaN u and the smallest u in one slot and leave the last slot unwritten (it keeps an earlier ray's value)."""
    u = np.random.RandomState(9).rand(64).astype(F32)
    u[20] = np.nan
    for prev in (0.25, 0.75):
        assert np.array_equal(u_slots(u, prev), np.sort(u), equal_nan=True)       # np.sort: NaN last
        old = u_slots(u, prev, nan_aware=False)
        assert old[-1] == F32(prev) and not np.array_equal(old, np.sort(u), equal_nan=True)


def dr_mismatch(a, b):
    return bool(position_mismatch({"z": a[None]}, {"z": b[None]}, slice(None), slice(None)))


def test_pattern_comparator_rejects_a_finite_nan_ray():
    """A device that returns finite values where render64 says NaN (e.g. a NaN point given a finite sigma) is
    rejected, and an exact NaN pattern is accepted."""
    ws = _ws()
    rays = np.concatenate([_ray(), _ray(o=(np.nan, 0.0, 4.0))])
    ref = render64(ws, rays, 32, 32, white_back=True)
    dev = {k: np.asarray(v, F32) for k, v in ref.items() if k in OUT_KEYS}
    assert not pattern_mismatch(dev, ref, slice(None))
    dev["rgb_fine"] = np.nan_to_num(dev["rgb_fine"])
    assert pattern_mismatch(dev, ref, [1]) == {"rgb_fine": 3}
