"""CPU-side checks of the view-batch entry: the argument checks that need no GPU, and DeviceViewBatches' argument
errors and its shared epoch logic."""
import ctypes
import inspect

import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib
from nerf_pl_b200 import data


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


def test_view_batch_argument_checks(lib):
    f = lib.nerfb200_view_batch
    one = ctypes.c_void_p(256)          # never dereferenced: every call below fails first, or has nothing to do
    good = dict(V=2, H=3, W=5, C=4, focal=1.5, n=8)

    def call(**kw):
        a = {**good, **kw}
        ptr = kw.get("ptr", one)
        return f(ptr, a["V"], a["H"], a["W"], a["C"], kw.get("c2w", one), a["focal"], 2.0, 6.0, 0, one, a["n"],
                 kw.get("rays", one), one, None)

    for bad, msg in ((dict(V=0), b"bad V"), (dict(H=0), b"bad V"), (dict(W=-1), b"bad V"), (dict(n=-1), b"bad V"),
                     (dict(C=1), b"C must be"), (dict(C=5), b"C must be"), (dict(focal=0.0), b"focal"),
                     (dict(focal=float("nan")), b"focal"), (dict(V=1 << 62), b"overflows"),
                     (dict(ptr=None), b"NULL"), (dict(c2w=ctypes.c_void_p(260)), b"aligned"),
                     (dict(rays=ctypes.c_void_p(264)), b"aligned")):
        assert call(**bad) == -1, bad
        assert msg in lib.nerfb200_last_error(), (bad, lib.nerfb200_last_error())
    assert call(n=0, ptr=None) == 0                      # nothing to do: no pointer is needed
    assert call(V=1, H=46341, W=46341, C=3, n=0) == 0    # V H W > 2**31 is a valid shape


def test_device_view_batches_argument_errors():
    img = torch.zeros(2, 3, 5, 4, dtype=torch.uint8)
    c2w = torch.zeros(2, 3, 4)
    for bad_img, bad_c2w in ((img.float(), c2w), (img[..., :2], c2w), (img[0], c2w), (img, c2w[:1]),
                             (img, torch.zeros(2, 4, 4))):
        with pytest.raises(ValueError):
            nb.DeviceViewBatches(bad_img, bad_c2w, 1.0, 2.0, 6.0)
    with pytest.raises(ValueError, match="batch size"):
        nb.DeviceViewBatches(img, c2w, 1.0, 2.0, 6.0, batch_size=0)
    with pytest.raises(ValueError, match="focal"):
        nb.DeviceViewBatches(img, c2w, 0.0, 2.0, 6.0)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        nb.DeviceViewBatches(img, c2w, 1.0, 2.0, 6.0, device="cpu")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        nb.DeviceRayBatches(torch.zeros(4, 8), torch.zeros(4, 3), device="cpu")


def test_one_epoch_logic_for_both_classes():
    """Both batch classes take permutation, len(), seeding and sharding from one base class, and CapturedTrainStep
    accepts either."""
    assert issubclass(nb.DeviceRayBatches, data._EpochBatches) and issubclass(nb.DeviceViewBatches, data._EpochBatches)
    for name in ("next_permutation", "__len__", "__iter__", "samples_per_rank"):
        assert name not in vars(nb.DeviceRayBatches) and name not in vars(nb.DeviceViewBatches), name
    src = inspect.getsource(nb.CapturedTrainStep.__init__)
    assert "isinstance(batches, _EpochBatches)" in src
    p = inspect.signature(nb.DeviceViewBatches).parameters
    assert list(p) == ["images", "c2w", "focal", "near", "far", "ndc", "batch_size", "shuffle", "drop_last", "seed",
                       "rank", "world_size", "device"]
    assert p["ndc"].default is False and p["batch_size"].default == 1024 and p["shuffle"].default is True
    for name in ("DeviceViewBatches", "read_blender_views", "read_llff_views"):
        assert name in nb.__all__ and hasattr(nb, name)
