"""The Unity volume (.vol) export of extract_mesh.ipynb on the device.

A. query_rgb_sigma equals NeRF.forward on the fp16 xyz encoding followed by the embedded zero direction, bit for bit
   in all four channels (up to the fp16 roundings the in-kernel encoding may legitimately pick, tests/sigma_ref.py);
   rgb_sigma_grid equals the point query of grid_positions for every chunk size.
B. pack_volume equals the numpy restatement with the correctly rounded exp (tests/volume_ref.py) exactly: on the
   kernel's own grids and on hand-made grids at the edges of the alpha arithmetic, at every launch shape.
C. The whole path against the reference notebook's own file (tests/golden/volume_unity.part*.npz).
D. An N = 256 grid over several default-size chunks.
"""
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as mo
from tests import cases
from tests import sigma_ref as sr
from tests import volume_ref as vr

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUBE = ((-1.5, 1.5),) * 3
UNEQUAL = ((-1.5, 1.5), (-1.2, 1.4), (-1.5, 1.3))
REVERSED = ((1.5, -1.5), (-1.2, 1.4), (1.3, -1.5))
# Embedding(3, 4) of the direction (0, 0, 0)
ZERO_DIR = np.array([0, 0, 0] + [0, 0, 0, 1, 1, 1] * 4, np.float32)


def _nb():
    import nerf_pl_b200 as nb
    return nb


_MODEL = []


def _model():
    if not _MODEL:
        m = _nb().NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in cases.trained_weights()[1].items()})
        _MODEL.append(m.cuda().eval())
    return _MODEL[0]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _u32(a):
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.uint32)


# ---------------------------------------------------------------------------------------------- A
def _points(name):
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    if name == "uniform":
        return rng.uniform(-1.5, 1.5, (60000, 3)).astype(np.float32)
    if name == "wide":
        p = rng.uniform(-61, 61, (20000, 3))
        p[:6] = [[61, -61, 0], [-61, 61, 61], [60.99, -0.0, 1e-30], [0, 0, 0], [-0.0, -0.0, -0.0], [1e-7, -1e-7, 3]]
        return p.astype(np.float32)
    if name == "grid":
        parts = [mo.grid_positions(n, *r) for n, r in ((17, UNEQUAL), (17, REVERSED), (33, CUBE), (2, UNEQUAL))]
        p = np.concatenate(parts)
        neg = p.copy()
        neg[p == 0] = -0.0
        return np.concatenate([p, neg[(p == 0).any(1)]]).astype(np.float32)
    n = {"n1": 1, "n127": 127, "n129": 129, "n_sms_minus": _sms() * 128 - 1, "n_sms_plus": _sms() * 128 + 1,
         "n_two_rounds": 2 * _sms() * 128 + 77}[name]
    return rng.uniform(-1.5, 1.5, (n, 3)).astype(np.float32)


@pytest.mark.parametrize("name", ["uniform", "wide", "grid", "n1", "n127", "n129", "n_sms_minus", "n_sms_plus",
                                  "n_two_rounds"])
def test_query_rgb_sigma_equals_forward_on_the_fp16_encoding_and_zero_direction(name):
    nb = _nb()
    model = _model()
    xyz = _points(name)
    dev = nb.query_rgb_sigma(model, torch.from_numpy(xyz).cuda()).cpu().numpy()
    assert dev.shape == (len(xyz), 4)
    rows, owner, choices = sr.candidate_encodings(xyz)
    x = np.concatenate([rows, np.broadcast_to(ZERO_DIR, (len(rows), 27))], 1)
    with torch.no_grad():
        cand = model(torch.from_numpy(x).cuda()).cpu().numpy()
    n = len(xyz)
    hit = np.zeros(n, bool)
    np.logical_or.at(hit, owner, (_u32(cand) == _u32(dev)[owner]).all(1))
    included = choices <= sr.MAX_ROUNDINGS
    exact = choices == 1
    print(f"\nquery_rgb_sigma {name}: {n} points, {int(exact.sum())} unambiguous, {int((included & ~exact).sum())} "
          f"with 2-16 roundings, {int((~included).sum())} excluded")
    assert hit[exact].all(), np.nonzero(exact & ~hit)[0][:10]
    assert hit[included].all(), np.nonzero(included & ~hit)[0][:10]
    assert included.mean() > 0.8
    # the sigma channel is the sigma-only query's
    so = nb.query_sigma(model, torch.from_numpy(xyz).cuda()).cpu().numpy()
    assert np.array_equal(_u32(so), _u32(dev[:, 3]))


@pytest.mark.parametrize("ranges", [CUBE, UNEQUAL, REVERSED], ids=["cube", "unequal", "reversed"])
def test_rgb_sigma_grid_equals_the_point_query_for_every_chunk(ranges):
    nb = _nb()
    model = _model()
    N = 33
    P = N ** 3
    xyz = nb.mesh.grid_positions(N, *ranges)
    point = nb.query_rgb_sigma(model, xyz)
    for chunk in (127, 128, 129, 4999, P - 1, P):
        g = nb.rgb_sigma_grid(model, N, *ranges, chunk=chunk)
        assert g.shape == (N, N, N, 4) and g.dtype == torch.float32
        assert torch.equal(g.reshape(-1, 4).view(torch.int32), point.view(torch.int32)), chunk


# ---------------------------------------------------------------------------------------------- B
def _hand_grid(N, x_range, seed):
    """rgb with exact 0 and 1 entries; sigma < 0, -0, +0, +inf, -inf, NaN, the smallest sigma with a > 0 and its
    predecessor, tiny and huge values, and a gamma-distributed bulk."""
    rng = np.random.default_rng(seed)
    P = N ** 3
    g = np.empty((P, 4), np.float32)
    g[:, :3] = rng.uniform(0, 1, (P, 3))
    g[:, :3][rng.random((P, 3)) < 0.05] = 0.0
    g[:, :3][rng.random((P, 3)) < 0.05] = 1.0
    g[:, 3] = rng.gamma(0.7, 30.0, P)
    g[rng.random(P) < 0.3, 3] *= -1
    sm = vr.smallest_positive_alpha_sigma(x_range, N)
    special = np.float32([-1.0, -0.0, 0.0, np.inf, -np.inf, np.nan, sm, np.nextafter(sm, np.float32(0)),
                          np.nextafter(sm, np.float32(np.inf)), 1e-30, 1e30, -1e30, np.finfo(np.float32).tiny])
    pos = rng.permutation(P)[:min(P - 4, 40 * len(special))] if P > 4 else np.zeros(0, np.int64)
    g[pos, 3] = special[np.arange(len(pos)) % len(special)]
    g[:4, :3] = [[0, 0, 0], [1, 1, 1], [0, 1, 0], [1, 0, 1]]
    g[:4, 3] = np.inf
    return g.reshape(N, N, N, 4)


def _pack(grid, x_range):
    return _nb().pack_volume(torch.from_numpy(np.ascontiguousarray(grid)).cuda(), x_range).cpu().numpy()


def _check_pack(grid, x_range, label):
    dev = _pack(grid, x_range)
    ref = vr.pack_volume(grid, x_range, exp="f64")
    print(f"\n{label}: {grid.shape[0]}^3 points, {len(ref)} kept")
    assert dev.dtype == np.uint32 and dev.shape == ref.shape
    assert np.array_equal(dev, ref)
    return dev


HAND = [(20, (-1.2, 1.2)), (20, (-1.5, 1.5)), (37, (-2.0, 0.7)), (2, (-1.0, 1.0)), (64, (-1.5, 1.5))]


@pytest.mark.parametrize("N,x_range", HAND)
def test_pack_volume_on_hand_made_grids(N, x_range):
    g = _hand_grid(N, x_range, N)
    dev = _check_pack(g, x_range, f"hand-made N {N} x {x_range}")
    flat = g.reshape(-1, 4)
    sm = vr.smallest_positive_alpha_sigma(x_range, N)
    kept = set(dev[:, 0].tolist())
    assert all(i in kept for i in np.nonzero(flat[:, 3] == sm)[0])
    assert not any(i in kept for i in np.nonzero(flat[:, 3] == np.nextafter(sm, np.float32(0)))[0])
    assert not any(i in kept for i in np.nonzero(np.isnan(flat[:, 3]) | (flat[:, 3] <= 0))[0])
    inf_rows = dev[np.isin(dev[:, 0], np.nonzero(np.isinf(flat[:, 3]) & (flat[:, 3] > 0))[0])]
    assert len(inf_rows) >= 4 and ((inf_rows[:, 1] & 255) == 255).all()
    # a reversed x_range: a <= 0 everywhere
    assert len(_check_pack(g, x_range[::-1], "reversed")) == 0


def test_pack_volume_empty_grid():
    g = np.zeros((16, 16, 16, 4), np.float32)
    g[..., 3] = -np.abs(np.random.default_rng(3).normal(size=(16, 16, 16)))
    g[0, 0, 0, 3] = -0.0
    g[0, 0, 1, 3] = 0.0
    g[0, 0, 2, 3] = np.nan
    out = _check_pack(g, (-1.5, 1.5), "empty")
    assert out.shape == (0, 2)


@pytest.fixture(scope="module")
def kernel_grids():
    nb = _nb()
    return {k: nb.rgb_sigma_grid(_model(), N, *r).cpu().numpy() for k, (N, r) in
            {"cube48": (48, CUBE), "unequal33": (33, UNEQUAL), "reversed33": (33, REVERSED)}.items()}


@pytest.mark.parametrize("name", ["cube48", "unequal33", "reversed33"])
def test_pack_volume_on_the_kernels_own_grid(kernel_grids, name):
    g = kernel_grids[name]
    x_range = {"cube48": CUBE, "unequal33": UNEQUAL, "reversed33": REVERSED}[name][0]
    dev = _check_pack(g, x_range, name)
    if name != "reversed33":
        assert len(dev) > 1000
    # two runs write the same bytes
    assert vr.vol_bytes(_pack(g, x_range)) == vr.vol_bytes(dev)


_SUBPROCESS = r"""
import sys
import numpy as np
import torch
sys.path.insert(0, sys.argv[1])
import nerf_pl_b200 as nb
z = np.load(sys.argv[2])
out = {}
for name in [k for k in z.files if not k.startswith("xr_")]:
    xr = tuple(float(v) for v in z["xr_" + name])
    out[name] = nb.pack_volume(torch.from_numpy(z[name]).cuda(), xr).cpu().numpy()
np.savez(sys.argv[3], **out)
"""


def test_pack_volume_does_not_depend_on_the_launch_shape(kernel_grids, tmp_path):
    grids = {"cube48": (kernel_grids["cube48"], CUBE[0]), "hand64": (_hand_grid(64, (-1.5, 1.5), 64), (-1.5, 1.5)),
             "hand20": (_hand_grid(20, (-1.2, 1.2), 20), (-1.2, 1.2))}
    arrays = {k: g for k, (g, _) in grids.items()}
    arrays.update({"xr_" + k: np.array(xr) for k, (_, xr) in grids.items()})
    np.savez(tmp_path / "in.npz", **arrays)
    base = {k: vr.pack_volume(g, xr) for k, (g, xr) in grids.items()}
    for ctas in ("1", "3"):
        env = dict(os.environ, NERFB200_MAX_CTAS=ctas)
        out = tmp_path / f"out{ctas}.npz"
        subprocess.run([sys.executable, "-c", _SUBPROCESS, ROOT, str(tmp_path / "in.npz"), str(out)], check=True,
                       env=env, cwd=ROOT)
        got = np.load(out)
        for name, ref in base.items():
            assert vr.vol_bytes(got[name]) == vr.vol_bytes(ref), (ctas, name)


# ---------------------------------------------------------------------------------------------- C
@pytest.fixture(scope="module")
def golden(golden_dir):
    return vr.load_golden(golden_dir)[0]


@pytest.mark.parametrize("name", ["cube48", "unequal33"])
def test_volume_matches_the_reference_notebook(golden, name, tmp_path):
    nb = _nb()
    c = golden[name]
    N, ranges = c["N"], c["ranges"]
    x_range = ranges[0]
    grid = nb.rgb_sigma_grid(_model(), N, *ranges)
    dev = nb.pack_volume(grid, x_range).cpu().numpy()
    path = tmp_path / f"{name}.vol"
    nb.write_vol(str(path), dev)
    assert path.read_bytes() == vr.vol_bytes(dev)
    assert np.array_equal(dev, vr.pack_volume(grid.cpu().numpy(), x_range))
    ref = vr.unpack(c["vol"])
    # the bar: BAR_MAX times the fp16 replay's largest distance from float64 sigma on this grid
    w = cases.trained_weights()[1]
    xyz = mo.grid_positions(N, *ranges).astype(np.float32)
    s64 = sr.sigma64(w, xyz, device="cuda")
    rep = sr.sigma_fp16_replay(w, xyz, device="cuda")
    bar = sr.BAR_MAX * float(np.abs(rep - s64).max())
    cabs = abs(float(vr.scale(x_range, N)))
    thr = float(vr.smallest_positive_alpha_sigma(x_range, N))
    sig_ref = np.maximum(c["rgbsigma"][:, 3].astype(np.float64), 0)
    only = np.setxor1d(ref[:, 0], dev[:, 0])
    gap = np.abs(sig_ref[only] - thr)
    common, ir, io = np.intersect1d(ref[:, 0], dev[:, 0], return_indices=True)
    sr_, sd = ref[ir, 1].astype(np.int64), dev[io, 1].astype(np.int64)
    drgb = np.stack([np.abs(((sr_ >> s) & 255) - ((sd >> s) & 255)) for s in (24, 16, 8)], 1)
    da8 = np.abs((sr_ & 255) - (sd & 255))
    a8_bar = 1 + 255 * cabs * bar
    print(f"\n{name}: reference {len(ref)} voxels, device {len(dev)}, {len(common)} common, {len(only)} kept by one "
          f"side only (largest |sigma+ - threshold| {gap.max(initial=0):.4g}, bar {bar:.4g})")
    print(f"  rgb bytes: {np.bincount(drgb.ravel(), minlength=2).tolist()} (count by |difference|); "
          f"a8: {np.bincount(da8, minlength=2).tolist()} (bar {a8_bar:.3g}); |c| {cabs:.5g}, threshold sigma {thr:.3g}")
    assert len(common) > 0.9 * len(ref)
    assert (gap <= bar).all()
    assert drgb.max(initial=0) <= 1
    assert da8.max(initial=0) <= a8_bar


# ---------------------------------------------------------------------------------------------- D
def test_volume_at_256_over_default_chunks():
    nb = _nb()
    N = 256
    grid = nb.rgb_sigma_grid(_model(), N, *UNEQUAL)          # 2^24 points: 8 chunks of 2^21
    dev = nb.pack_volume(grid, UNEQUAL[0]).cpu().numpy()
    g = grid.cpu().numpy()
    ref = vr.pack_volume(g, UNEQUAL[0])
    print(f"\nN 256: {len(ref)} of {N ** 3} voxels kept")
    assert len(ref) > 10000
    assert np.array_equal(dev, ref)
    # the grid's chunks are the point query's
    for s in (0, (1 << 21) - 5, 7 * (1 << 21)):
        xyz = nb.mesh.grid_positions(N, *UNEQUAL, start=s, count=4096)
        q = nb.query_rgb_sigma(_model(), xyz).cpu().numpy()
        assert np.array_equal(_u32(q), _u32(g.reshape(-1, 4)[s:s + 4096]))
