"""The C ABI of the density grid: the workspace sizes, the argument errors the entries return before any launch, and the
argument errors of nb.DensityGrid and CapturedTrainStep(update_every=) that need no GPU."""
import ctypes
import math

import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib

BOX = (ctypes.c_double * 6)(-1, 1, -1, 1, -1, 1)


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


def test_workspace_sizes(lib):
    ws = lib.nerfb200_density_workspace_bytes
    for N in (1, 0, -3, 1626):
        assert ws(N, 1024) == 0
    assert ws(17, 0) == 0 and ws(17, -1) == 0
    C = 16 ** 3
    assert ws(17, 1) >= 16 + 2 * C and ws(17, 100) >= 100 * 16 + 2 * C
    assert ws(17, C) == ws(17, C + 1) == ws(17, 1 << 40)       # a chunk past the grid is the grid
    assert ws(17, 1) < ws(17, 100) < ws(17, C)
    assert ws(2, 1 << 21) >= 16 + 2 and ws(1625, 1 << 21) >= 2 * 1624 ** 3 + 16 * (1 << 21)


def test_points_argument_checks(lib):
    one = ctypes.c_void_p(256)          # never dereferenced: every call below fails first
    pts = lib.nerfb200_density_points
    assert pts(1, BOX, one, 0, 1, one, None) == -1 and b"N must be in [2, 1625]" in lib.nerfb200_last_error()
    assert pts(1626, BOX, one, 0, 1, one, None) == -1
    assert pts(5, None, one, 0, 1, one, None) == -1 and b"NULL" in lib.nerfb200_last_error()
    for bad in ((-1, 1, 2, 2, -1, 1), (-1, 1, -1, 1, math.inf, 1), (math.nan, 1, -1, 1, -1, 1)):
        assert pts(5, (ctypes.c_double * 6)(*bad), one, 0, 1, one, None) == -1
        assert b"finite with min != max" in lib.nerfb200_last_error()
    for start, count in ((-1, 1), (0, -1), (0, 65), (64, 1), (65, 0), (60, 5)):
        assert pts(5, BOX, one, start, count, one, None) == -1, (start, count)
        assert b"outside the grid" in lib.nerfb200_last_error()
    assert pts(5, BOX, None, 0, 0, None, None) == 0              # nothing to do
    assert pts(5, BOX, None, 0, 4, one, None) == -1 and b"NULL" in lib.nerfb200_last_error()
    assert pts(5, BOX, one, 0, 4, None, None) == -1 and b"NULL" in lib.nerfb200_last_error()


def test_update_argument_checks(lib):
    one = ctypes.c_void_p(256)
    big = 1 << 40
    upd = lib.nerfb200_density_update

    def call(**kw):
        a = dict(packed=one, N=17, ranges=BOX, thr=1.0, decay=0.95, dilate=1, chunk=1024, key=one, density=one,
                 bits=one, ws=one, nbytes=big)
        a.update(kw)
        return upd(*a.values(), None)

    cases = [(dict(N=1), b"N must be in [2, 1625]"), (dict(N=1626), b"N must be in [2, 1625]"),
             (dict(ranges=(ctypes.c_double * 6)(0, 0, -1, 1, -1, 1)), b"min != max"),
             (dict(ranges=None), b"NULL"),
             (dict(thr=math.nan), b"NaN"), (dict(decay=-0.01), b"decay"), (dict(decay=1.01), b"decay"),
             (dict(decay=math.nan), b"decay"), (dict(dilate=-1), b"dilate"), (dict(chunk=0), b"chunk"),
             (dict(packed=None), b"NULL"), (dict(key=None), b"NULL"), (dict(density=None), b"NULL"),
             (dict(bits=None), b"NULL"), (dict(ws=None), b"NULL"),
             (dict(nbytes=lib.nerfb200_density_workspace_bytes(17, 1024) - 1), b"workspace smaller")]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert msg in lib.nerfb200_last_error(), (kw, lib.nerfb200_last_error())


def test_density_grid_argument_errors():
    box = ((-1.0, 1.0),) * 3
    for kw, msg in ((dict(N=1), "outside"), (dict(N=1626), "outside"), (dict(sigma_threshold=math.nan), "NaN"),
                    (dict(decay=-0.1), "decay"), (dict(decay=1.5), "decay"), (dict(decay=math.nan), "decay"),
                    (dict(dilate=-1), "dilate"), (dict(dilate=1.5), "dilate"), (dict(chunk=0), "chunk"),
                    (dict(x_range=(1.0, 1.0)), "min != max"), (dict(y_range=(0.0, math.inf)), "finite"),
                    (dict(z_range=(0.0,)), "min, max"), (dict(device="cpu"), "CUDA")):
        args = dict(N=8, x_range=box[0], y_range=box[1], z_range=box[2])
        args.update(kw)
        with pytest.raises((ValueError, RuntimeError), match=msg):
            nb.DensityGrid(**args)


def test_captured_step_update_every_needs_a_density_grid():
    """update_every without a DensityGrid is refused before anything touches a device."""
    sig = __import__("inspect").signature(nb.CapturedTrainStep.__init__)
    assert list(sig.parameters)[-2:] == ["occupancy", "update_every"]
    assert sig.parameters["update_every"].default is None
    from nerf_pl_b200.data import _EpochBatches

    class _Batches(_EpochBatches):
        batch_size, samples_per_rank, device = 4, 8, torch.device("meta")

        def __init__(self):
            pass

    models = [nb.NeRF(), nb.NeRF()]
    opt = nb.FusedAdam([p for m in models for p in m.parameters()], capturable=True)
    for occ in (None, "grid"):
        with pytest.raises(ValueError, match="update_every needs occupancy=DensityGrid"):
            nb.CapturedTrainStep(models, _Batches(), opt, occupancy=None if occ is None else object(),
                                 update_every=4)
