"""Training batches generated on the device from the views (pytest -m gpu): view_batch_kernel and DeviceViewBatches.

- The kernel equals the float32 emulation (tests/views_ref.py) bit for bit: RGB and RGBA, NDC on and off, odd H and
  W, ids in any order; one 256 x 256 RGBA image holds every (value, alpha) pair.
- DeviceViewBatches yields, bit for bit, the batches of a DeviceRayBatches built from nb.generate_rays per view and
  the same colours, with the same seed: shuffled or not, drop_last, and every rank of a world of 3.
- CapturedTrainStep over 50 replays leaves identical parameters and Adam state with either class.
- view(v) equals generate_rays plus the colours (and alpha > 0 as valid_mask).
- A dataset of V H W > 2**31 pixels (6.45 GB of uint8): ids near the end and around 2**31 decode in 64 bits.
"""
import numpy as np
import pytest
import torch

import nerf_pl_b200 as nb
from nerf_pl_b200 import _lib
from tests import cases
from tests import units_ref as ur
from tests import views_ref as vr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _poses(V, seed, radius=4.0):
    """Cameras on a sphere looking at the origin (Blender-style, "right up back")."""
    rng = np.random.default_rng(seed)
    out = np.zeros((V, 3, 4))
    for v in range(V):
        z = rng.normal(size=3)
        z[2] = abs(z[2]) + 0.3
        z /= np.linalg.norm(z)
        x = np.cross([0.0, 0.0, 1.0], z)
        x /= np.linalg.norm(x)
        out[v] = np.stack([x, np.cross(z, x), z, radius * z], 1)
    return out


def _forward_poses(V, seed):
    """Forward-facing cameras near the identity (LLFF-style, for NDC)."""
    rng = np.random.default_rng(seed)
    out = np.zeros((V, 3, 4))
    for v in range(V):
        out[v, :, :3] = vr._rotation(rng, 0.08)
        out[v, :, 3] = rng.uniform(-0.3, 0.3, 3)
    return out


def _images(V, H, W, C, seed):
    return np.random.default_rng(seed).integers(0, 256, (V, H, W, C), dtype=np.uint8)


def _same(a, b):
    a = a.cpu().numpy() if torch.is_tensor(a) else a
    b = b.cpu().numpy() if torch.is_tensor(b) else b
    return a.shape == b.shape and ur.bitwise_differ(a, b) == 0


def _scene(C, ndc, V=3, H=17, W=23, seed=0):
    images = _images(V, H, W, C, seed)
    c2w = _forward_poses(V, seed) if ndc else _poses(V, seed)
    return images, c2w, 0.9 * W, (0.0, 1.0) if ndc else (2.0, 6.0)


# ------------------------------------------------------------------------------------------------- the kernel
@pytest.mark.parametrize("ndc", [False, True])
@pytest.mark.parametrize("C", [3, 4])
def test_kernel_equals_the_emulation(C, ndc, dev):
    images, c2w, focal, (near, far) = _scene(C, ndc)
    b = nb.DeviceViewBatches(images, c2w, focal, near, far, ndc=ndc, seed=1)
    n = b.n_rays
    for ids in (np.arange(n), np.random.default_rng(2).permutation(n)[:1000], np.array([n - 1, 0, n - 1, 17])):
        got = b.gather(torch.from_numpy(ids).to(dev))
        rays, rgbs = vr.view_batch32(images, c2w, focal, near, far, ndc, ids)
        assert _same(got["rays"], rays) and _same(got["rgbs"], rgbs)
    empty = b.gather(torch.zeros(0, dtype=torch.int64, device=dev))
    assert empty["rays"].shape == (0, 8) and empty["rgbs"].shape == (0, 3)


def test_every_value_and_alpha_pair(dev):
    val, alpha = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8), indexing="ij")
    img = np.stack([val, 255 - val, val[::-1], alpha], -1)[None]
    b = nb.DeviceViewBatches(img, _poses(1, 3), 300.0, 2.0, 6.0, shuffle=False)
    got = b.gather(torch.arange(256 * 256, device=dev))
    assert _same(got["rgbs"], vr.colours32(img.reshape(-1, 4)))
    rgb = nb.DeviceViewBatches(np.ascontiguousarray(img[..., :3]), _poses(1, 3), 300.0, 2.0, 6.0, shuffle=False)
    assert _same(rgb.gather(torch.arange(256 * 256, device=dev))["rgbs"], vr.colours32(img[0, ..., :3].reshape(-1, 3)))


def test_out_of_range_ids_give_nan_rows(dev):
    images, c2w, focal, (near, far) = _scene(4, False)
    b = nb.DeviceViewBatches(images, c2w, focal, near, far)
    got = b.gather(torch.tensor([-1, b.n_rays, 5], device=dev))
    assert torch.isnan(got["rays"][:2]).all() and torch.isnan(got["rgbs"][:2]).all()
    assert torch.isfinite(got["rays"][2]).all()
    torch.cuda.synchronize()
    assert _lib.load().nerfb200_check_status() == 0


# -------------------------------------------------------------------------------- against DeviceRayBatches
def _ray_batches_equivalent(images, c2w, focal, near, far, ndc, dev, **kw):
    V, H, W, C = images.shape
    rays = torch.cat([nb.generate_rays(H, W, focal, c2w[v], near, far, ndc=ndc, device=dev) for v in range(V)])
    rgbs = torch.from_numpy(vr.colours32(images.reshape(-1, C)))
    return nb.DeviceRayBatches(rays, rgbs, **kw)


@pytest.mark.parametrize("shuffle,drop_last,world", [(True, False, 1), (False, False, 1), (True, True, 1),
                                                      (True, False, 3), (True, True, 3)])
@pytest.mark.parametrize("C,ndc", [(4, False), (3, True)])
def test_same_batches_as_device_ray_batches(C, ndc, shuffle, drop_last, world, dev):
    images, c2w, focal, (near, far) = _scene(C, ndc, V=4, H=19, W=21, seed=5)
    for rank in range(world):
        kw = dict(batch_size=256, shuffle=shuffle, drop_last=drop_last, seed=7, rank=rank, world_size=world)
        a = nb.DeviceViewBatches(images, c2w, focal, near, far, ndc=ndc, **kw)
        b = _ray_batches_equivalent(images, c2w, focal, near, far, ndc, dev, **kw)
        assert len(a) == len(b) and a.samples_per_rank == b.samples_per_rank
        for _ in range(2):
            ea, eb = list(a), list(b)
            assert len(ea) == len(eb) == len(a)
            for x, y in zip(ea, eb):
                assert _same(x["rays"], y["rays"]) and _same(x["rgbs"], y["rgbs"])


def test_captured_step_is_the_same_with_either_class(dev):
    """50 replays (16 full batches per epoch: three reshuffles), in-kernel random numbers: parameters and Adam state
    bit for bit."""
    images, c2w, focal, (near, far) = _scene(4, False, V=4, H=64, W=64, seed=9)
    runs = []
    for kind in ("views", "rays"):
        kw = dict(batch_size=1024, seed=21)
        if kind == "views":
            batches = nb.DeviceViewBatches(images, c2w, focal, near, far, **kw)
        else:
            batches = _ray_batches_equivalent(images, c2w, focal, near, far, False, dev, **kw)
        models = []
        for w in cases.weights():
            m = nb.NeRF()
            m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in w.items()})
            models.append(m.to(dev))
        opt = nb.FusedAdam([p for m in models for p in m.parameters()], capturable=True, lr=5e-4, eps=1e-8)
        step = nb.CapturedTrainStep(models, batches, opt, 64, False, 1.0, 0.0, 64, True, randoms={"seed": 4000})
        assert step.per_epoch == 16
        losses = torch.stack([step.step()[0].clone() for _ in range(50)])
        assert step.epoch == 3
        runs.append((losses, step.params, opt))
    torch.cuda.synchronize()
    assert _lib.load().nerfb200_check_status() == 0
    (la, pa, oa), (lb, pb, ob) = runs
    assert torch.equal(la, lb) and torch.isfinite(la).all()
    for p, q in zip(pa, pb):
        assert torch.equal(p, q)
        for key in ("exp_avg", "exp_avg_sq", "step"):
            assert torch.equal(oa.state[p][key], ob.state[q][key]), key


@pytest.mark.parametrize("C,ndc", [(4, False), (3, True), (3, False)])
def test_view_equals_generate_rays_and_colours(C, ndc, dev):
    images, c2w, focal, (near, far) = _scene(C, ndc, V=3, H=15, W=9, seed=11)
    b = nb.DeviceViewBatches(images, c2w, focal, near, far, ndc=ndc)
    V, H, W, _ = images.shape
    for v in range(V):
        out = b.view(v)
        assert _same(out["rays"], nb.generate_rays(H, W, focal, c2w[v], near, far, ndc=ndc, device=dev))
        assert _same(out["rgbs"], vr.colours32(images[v].reshape(-1, C)))
        if C == 4:
            assert torch.equal(out["valid_mask"].cpu(), torch.from_numpy(images[v, ..., 3].reshape(-1) > 0))
        else:
            assert "valid_mask" not in out
    with pytest.raises(IndexError):
        b.view(V)


# ------------------------------------------------------------------------------------------------ 64-bit decode
def test_ids_beyond_two_to_the_31(dev):
    """V = 5 views of 20736 x 20736 RGB: 2,149,908,480 pixels (> 2**31), 6.45 GB.  Only the pixels the ids name are
    written; each row equals the emulation."""
    V, H, W, C = 5, 20736, 20736, 3
    total = V * H * W
    assert total > 2 ** 31
    images = torch.empty((V, H, W, C), dtype=torch.uint8, device=dev)
    ids = np.array([total - 1, total - 2, total - W, (V - 1) * H * W, (V - 1) * H * W - 1, 2 ** 31 - 1, 2 ** 31,
                    2 ** 31 + 1, 3 * H * W + 7, H * W, 12345], np.int64)
    v, rem = np.divmod(ids, H * W)
    j, i = np.divmod(rem, W)
    px = np.random.default_rng(13).integers(0, 256, (len(ids), C), dtype=np.uint8)
    images[torch.from_numpy(v).to(dev), torch.from_numpy(j).to(dev), torch.from_numpy(i).to(dev)] = \
        torch.from_numpy(px).to(dev)
    c2w = _poses(V, 14)
    focal = 0.7 * W
    b = nb.DeviceViewBatches(images, c2w, focal, 2.0, 6.0, batch_size=4096)
    assert b.images.data_ptr() == images.data_ptr()                 # a device uint8 tensor is not copied
    assert b.n_rays == total and len(b) == -(-total // 4096)
    got = b.gather(torch.from_numpy(ids).to(dev))
    rays = vr.pixel_rays32(i, j, H, W, focal, c2w.astype(np.float32)[v], 2.0, 6.0)
    assert _same(got["rays"], rays) and _same(got["rgbs"], vr.colours32(px))
    del b, images
    torch.cuda.empty_cache()
