"""CPU checks of tests/sigma_ref.py: the encoding band covers the kernel's reduction, and each comparator of
tests/test_gpu_mesh_field.py rejects the defect it exists for."""
import numpy as np
import torch

from oracle import mesh_oracle as mo
from oracle import nerf_oracle as orc
from tests import sigma_ref as sr


def _kernel_reduction(a32):
    """fast_sincos's argument reduction (render_kernel.cuh) in exact arithmetic + fp32 rounding: the fp32 r whose
    MUFU sin / cos the kernel takes."""
    n = np.rint((a32 * np.float32(0.15915494309189535)).astype(np.float32)).astype(np.float64)
    r = (n * -6.28125 + a32.astype(np.float64)).astype(np.float32).astype(np.float64)      # both fmaf exact in float64
    return (n * -np.float64(np.float32(1.9353071795864769e-3)) + r).astype(np.float32).astype(np.float64)


def _kernel_like_encoding(xyz, rng):
    """An encoding as the kernel may form it: the reduced argument's sin / cos off by up to the MUFU error 2^-21.4,
    rounded to fp32 and then to fp16."""
    x = np.asarray(xyz, np.float32)
    cols = [x.astype(np.float16)]
    for k in range(sr.N_FREQS):
        r = _kernel_reduction((x * np.float32(2 ** k)).astype(np.float32))
        for f in (np.sin, np.cos):
            v = f(r) + rng.uniform(-1, 1, r.shape) * 2.0 ** -21.41
            cols.append(v.astype(np.float32).astype(np.float16))
    return np.concatenate(cols, 1).astype(np.float32)


def test_reduction_error_fits_the_band():
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.uniform(-61, 61, 400_000), rng.uniform(-1.5, 1.5, 100_000), [61.0, -61.0, 0.0]])
    x = x.astype(np.float32)
    worst = 0.0
    for k in range(sr.N_FREQS):
        a = (x * np.float32(2 ** k)).astype(np.float32)
        r = _kernel_reduction(a)
        worst = max(worst, float(np.abs(np.sin(r) - np.sin(a.astype(np.float64))).max()),
                    float(np.abs(np.cos(r) - np.cos(a.astype(np.float64))).max()))
    assert worst < 2.0 ** -22
    assert worst + 2.0 ** -21.41 < sr.BAND


def test_candidates_hold_kernel_like_encodings_and_reject_a_wrong_rounding():
    rng = np.random.default_rng(1)
    xyz = rng.uniform(-1.5, 1.5, (4000, 3)).astype(np.float32)
    rows, owner, choices = sr.candidate_encodings(xyz)
    n = len(xyz)
    ok = choices <= sr.MAX_ROUNDINGS
    # the first rows are e16 of the included points
    assert np.array_equal(owner[:ok.sum()], np.nonzero(ok)[0])
    assert np.array_equal(rows[:ok.sum()], sr.e16(xyz)[ok])
    frac_amb = float((choices > 1).mean())
    assert 0.3 < frac_amb < 0.7          # about half of the points have an ambiguous feature
    # a random projection stands in for the network: distinct encodings give distinct "sigma"
    proj = rng.normal(size=63)
    sig = lambda e: (e.astype(np.float64) @ proj).astype(np.float32)
    dev = _kernel_like_encoding(xyz, rng)
    hit = sr.matches_a_rounding(sig(dev), sig(rows), owner, n)
    assert hit[ok].all()
    # one feature rounded the wrong way outside the band: not among the candidates
    v = sr.embed64(xyz)
    lo, hi = sr._f16_range(v, sr.BAND)
    clear = (lo == hi)
    clear[:, :3] = False
    p, c = np.nonzero(clear & ok[:, None])
    sel = rng.choice(len(p), 300, replace=False)
    bad = dev.copy()
    h = bad[p[sel], c[sel]].astype(np.float16)
    exact = v[p[sel], c[sel]]
    wrong = np.where(exact > h.astype(np.float64), np.nextafter(h, np.float16(-np.inf)), np.nextafter(h, np.float16(np.inf)))
    bad[p[sel], c[sel]] = wrong.astype(np.float32)
    hit_bad = sr.matches_a_rounding(sig(bad), sig(rows), owner, n)
    assert not hit_bad[p[sel]].any()


def _field(p):
    """A cheap stand-in for sigma with no symmetry between the axes."""
    return (np.sin(3 * p[:, 0]) + 2 * p[:, 1] ** 2 - p[:, 2] + 0.3 * p[:, 0] * p[:, 2]).astype(np.float32)


def _chunked_grid(N, ranges, chunk, offset=0, indexing="xy"):
    """sigma_grid's chunk loop in numpy, with injectable defects."""
    axes = [np.linspace(r[0], r[1], N) for r in ranges]
    pts = np.stack(np.meshgrid(*axes, indexing=indexing), -1).reshape(-1, 3).astype(np.float32)
    out = np.empty(N ** 3, np.float32)
    for s in range(0, N ** 3, chunk):
        e = min(s + chunk, N ** 3)
        src = np.clip(np.arange(s, e) + (offset if s > 0 else 0), 0, N ** 3 - 1)
        out[s:e] = np.maximum(_field(pts[src]), 0)
    return out.reshape(N, N, N)


def test_sigma_grid_check_rejects_ij_indexing_and_a_shifted_chunk():
    N, ranges = 17, ((-1.5, 1.5), (-1.2, 1.4), (1.3, -1.5))
    q = _field(mo.grid_positions(N, *ranges))
    assert sr.grid_mismatches(_chunked_grid(N, ranges, 129), q, N) == 0
    assert sr.grid_mismatches(_chunked_grid(N, ranges, 129, indexing="ij"), q, N) > 0
    assert sr.grid_mismatches(_chunked_grid(N, ranges, 129, offset=1), q, N) > 0


def test_level_set_bar_passes_fp32_sums_and_rejects_a_dropped_relu():
    w = orc.make_weights(11)
    rng = np.random.default_rng(2)
    xyz = rng.uniform(-1.5, 1.5, (3000, 3)).astype(np.float32)
    s64 = sr.sigma64(w, xyz)
    # the float64 module is nerf_forward_torch: its float64 embedding and layers against an explicit float64 forward
    e = torch.from_numpy(sr.embed64(xyz))
    h = e
    for l in range(1, 9):
        inp = torch.cat([e, h], 1) if l == 5 else h
        h = torch.relu(inp @ torch.from_numpy(w[f"xyz_encoding_{l}.0.weight"]).double().T
                       + torch.from_numpy(w[f"xyz_encoding_{l}.0.bias"]).double())
    ref = (h @ torch.from_numpy(w["sigma.weight"][0]).double() + float(w["sigma.bias"][0])).numpy()
    assert np.abs(s64 - ref).max() < 1e-12
    rep = sr.sigma_fp16_replay(w, xyz)
    thr = float(np.median(s64))
    r = sr.field_report(sr.sigma_fp16_replay(w, xyz, acc=torch.float32), s64, rep, thr)
    assert all(r["ok"].values()), r
    assert r["replay"]["max"] > 0
    for l in (1, 5, 8):
        bad = sr.field_report(sr.sigma_fp16_replay(w, xyz, drop_relu=l), s64, rep, thr)
        assert not bad["ok"]["max"] and not bad["ok"]["p99"], (l, bad)


def test_crossings_follow_marching_cubes_vertices():
    rng = np.random.default_rng(3)
    s = rng.normal(size=(9, 10, 11)).astype(np.float32)
    pos, ends = sr.crossings(s, 0.25)
    v, _ = mo.marching_cubes(s, 0.25)
    assert np.array_equal(pos, v)
    flat = s.reshape(-1)
    assert ((flat[ends[:, 0]] > 0.25) != (flat[ends[:, 1]] > 0.25)).all()
    # axis 0 is y, axis 1 is x
    w = sr.index_to_world(np.array([[0.0, 0.0, 0.0], [8.0, 9.0, 10.0], [2.0, 0.0, 0.0]]), 11, (-1, 1), (-2, 2), (0, 5))
    assert np.allclose(w, [[-1, -2, 0], [0.8, 1.2, 5], [-1, -1.2, 0]])
