"""nb.ssim and nb.visualize_depth on the device: visualize_depth bit for bit against what the unmodified reference
returned (tests/golden/depth_viz.npz) and against the numpy restatement on a full 800 x 800 trained render; ssim
against the float64 restatement (tests/ssim_ref.py), the same bits with one CTA and with the full grid, and the same
bits from strided and contiguous inputs."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import bench
from tests import cases
from tests import depth_viz_ref as dv
from tests import ssim_ref as sr

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(cases.GOLDEN, "depth_viz.npz")
# float64 kernel against float64 numpy: only the order of the window sums differs
PIXEL_TOL = 1e-12


def _nb():
    import nerf_pl_b200 as nb
    return nb


def _images(shape, seed, close=False):
    rng = np.random.default_rng(seed)
    x = rng.random(shape).astype(np.float32)
    y = np.clip(x + rng.normal(0, 0.03, shape), 0, 1).astype(np.float32) if close else \
        rng.random(shape).astype(np.float32)
    return x, y


# ---- visualize_depth ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["trained", "nan", "posinf", "neginf", "negative", "constant", "one", "odd"])
def test_visualize_depth_equals_the_reference_fixture(name):
    z = np.load(GOLDEN)
    depth = torch.from_numpy(z[f"{name}.depth"]).cuda()
    out = _nb().visualize_depth(depth)
    want = torch.from_numpy(z[f"{name}.out"]).cuda()
    assert out.dtype == torch.float32 and out.is_cuda and out.shape == want.shape
    assert torch.equal(out, want)
    # a transposed view is read through its strides
    assert torch.equal(_nb().visualize_depth(depth.t().contiguous().t()), want)


def test_visualize_depth_of_a_full_800_view():
    nb = _nb()
    models = []
    for w in cases.trained_weights():
        m = nb.NeRF()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
        models.append(m.cuda().eval())
    rays = torch.from_numpy(bench.blender_rays(0, 72, W=800, H=800, pixels="all")).cuda()
    res = nb.batched_inference(models, [nb.Embedding(3, 10), nb.Embedding(3, 4)], rays, 64, 64, False, 32768, True)
    depth = res["depth_fine"].view(800, 800)
    out = nb.visualize_depth(depth)
    want = dv.visualize_depth(depth.cpu().numpy())
    assert len(np.unique(dv.to_uint8(depth.cpu().numpy()))) > 100
    assert torch.equal(out.cpu(), torch.from_numpy(want))


# ---- ssim --------------------------------------------------------------------------------------------------------
SHAPES = [(1, 3, 1, 1), (1, 3, 2, 2), (1, 3, 37, 53), (3, 5, 16, 9), (2, 1, 64, 64), (1, 3, 400, 400),
          (1, 3, 800, 800)]


def _within_one_rounding(got, want):
    """got (float32) is the float32 rounding of a double within PIXEL_TOL of want (float64)."""
    got = np.asarray(got, np.float32)
    half_ulp = np.spacing(np.abs(got)).astype(np.float64) / 2
    return bool(np.all(np.abs(got.astype(np.float64) - want) <= half_ulp + PIXEL_TOL * np.maximum(1.0, np.abs(want))))


@pytest.mark.parametrize("close", [False, True])
@pytest.mark.parametrize("shape", SHAPES)
def test_ssim_against_the_float64_restatement(shape, close):
    nb = _nb()
    x, y = _images(shape, sum(shape), close)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    got = nb.ssim(xd, yd, "none")
    assert got.shape == shape and got.dtype == torch.float32
    assert _within_one_rounding(got.cpu().numpy(), sr.ssim(x, y, "none"))
    for red in ("mean", "sum"):
        v = nb.ssim(xd, yd, red)
        assert v.shape == () and v.dtype == torch.float32
        assert _within_one_rounding(v.cpu().numpy(), sr.ssim(x, y, red))
    assert float(nb.ssim(xd, xd)) == 1.0
    assert torch.equal(nb.ssim(xd, xd, "none"), torch.ones(shape, device="cuda"))


def test_ssim_negative_map_is_clamped():
    nb = _nb()
    rng = np.random.default_rng(3)
    x = (rng.random((1, 1, 24, 24)) > 0.5).astype(np.float32)
    y = 1 - x
    neg = sr.ssim_map(x, y) < 0
    got = nb.ssim(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), "none").cpu().numpy()
    assert neg.sum() > 50 and np.all(got[neg] == 0.0)
    assert np.array_equal(got, sr.ssim(x, y, "none").astype(np.float32))


def test_ssim_reads_the_training_scripts_layout_in_place():
    """rgb.view(H, W, 3).permute(2, 0, 1)[None], as train.py / eval.py hold their images: the same bits as the
    contiguous copy, and no copy is made (the entry reads the strides)."""
    nb = _nb()
    H, W = 123, 77
    a = torch.rand(H * W, 3, device="cuda")
    b = (a + 0.05 * torch.randn_like(a)).clamp(0, 1)
    pa, pb = a.view(H, W, 3).permute(2, 0, 1)[None], b.view(H, W, 3).permute(2, 0, 1)[None]
    assert not pa.is_contiguous()
    for red in ("mean", "sum", "none"):
        assert torch.equal(nb.ssim(pa, pb, red), nb.ssim(pa.contiguous(), pb.contiguous(), red))
    # an expanded (stride 0) batch
    e = pa.expand(4, 3, H, W)
    assert torch.equal(nb.ssim(e, pb.expand(4, 3, H, W), "none")[3], nb.ssim(pa, pb, "none")[0])


def test_ssim_is_the_same_with_one_cta():
    """NERFB200_MAX_CTAS=1 (read once per process): the same bits with one CTA as with the full grid."""
    code = (
        "import sys, torch, numpy as np\n"
        f"sys.path.insert(0, {ROOT!r})\n"
        "import nerf_pl_b200 as nb\n"
        "g = torch.Generator().manual_seed(5)\n"
        "x = torch.rand(2, 3, 400, 400, generator=g).cuda(); y = torch.rand(2, 3, 400, 400, generator=g).cuda()\n"
        "d = torch.rand(800, 800, generator=g).mul(4).add(2).cuda()\n"
        "outs = [nb.ssim(x, y, r) for r in ('mean', 'sum', 'none')] + [nb.visualize_depth(d)]\n"
        "torch.save([o.cpu() for o in outs], sys.argv[1])\n")
    res = []
    with tempfile.TemporaryDirectory() as tmp:
        for env in ("1", None):
            path = os.path.join(tmp, f"out_{env}.pt")
            e = dict(os.environ)
            e.pop("NERFB200_MAX_CTAS", None)
            if env:
                e["NERFB200_MAX_CTAS"] = env
            r = subprocess.run([sys.executable, "-c", code, path], env=e, capture_output=True, text=True, timeout=600)
            assert r.returncode == 0, r.stderr[-2000:]
            res.append(torch.load(path))
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_ssim_argument_errors_on_the_device():
    nb = _nb()
    x = torch.rand(1, 3, 8, 8, device="cuda")
    with pytest.raises(ValueError, match="same"):
        nb.ssim(x, x[:, :2])
    with pytest.raises(ValueError, match="same"):
        nb.ssim(x[0], x[0])
    with pytest.raises(ValueError, match="float32"):
        nb.ssim(x.double(), x.double())
    with pytest.raises(ValueError, match=">= 1"):
        nb.ssim(x[:, :, :0], x[:, :, :0])
    with pytest.raises(ValueError, match=r"\(H, W\)"):
        nb.visualize_depth(x[0])
    with pytest.raises(ValueError, match=">= 1"):
        nb.visualize_depth(torch.zeros(0, 5, device="cuda"))
