"""DeviceRayBatches (pytest -m gpu): device-resident shuffled batches as the training DataLoader's replacement.

Every epoch is exactly a permutation of the dataset, batch sizes and len() are DataLoader's, epochs differ and a seed
repeats, DDP rank shards are disjoint and cover the epoch, and a short training loop fed by it equals, bit for bit,
the same loop fed the same index lists from host tensors."""
import numpy as np
import pytest
import torch
from torch.utils.data import DataLoader

import nerf_pl_b200 as nb
from oracle import nerf_oracle as orc
from tests import cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _dataset(n, seed=0):
    """Host rays / colours whose first two columns carry the row index (exact in fp32), so rows can be traced."""
    g = torch.Generator().manual_seed(seed)
    rays = torch.rand(n, 8, generator=g)
    rgbs = torch.rand(n, 3, generator=g)
    rays[:, 0] = torch.arange(n, dtype=torch.float32)
    rgbs[:, 0] = torch.arange(n, dtype=torch.float32)
    return rays, rgbs


def _epoch_indices(batches, rays, rgbs):
    """The row indices of one epoch, batch by batch, checked row for row against the source."""
    out = []
    for b in batches:
        assert b["rays"].is_cuda and b["rgbs"].is_cuda and b["rays"].dtype == torch.float32
        idx = b["rays"][:, 0].long().cpu()
        assert torch.equal(b["rays"].cpu(), rays[idx]) and torch.equal(b["rgbs"].cpu(), rgbs[idx])
        out.append(idx)
    return out


@pytest.mark.parametrize("n,bs", [(5000, 1024), (4096, 1024), (7, 3), (1, 4)])
@pytest.mark.parametrize("drop_last", [False, True])
def test_epochs_are_permutations_with_dataloader_batches(n, bs, drop_last, dev):
    rays, rgbs = _dataset(n, n)
    batches = nb.DeviceRayBatches(rays, rgbs, batch_size=bs, drop_last=drop_last, seed=11)
    ref = [len(b) for b in DataLoader(range(n), batch_size=bs, drop_last=drop_last)]
    assert len(batches) == len(ref)
    epochs = []
    for _ in range(3):
        ep = _epoch_indices(batches, rays, rgbs)
        assert [len(i) for i in ep] == ref
        flat = torch.cat(ep) if ep else torch.zeros(0, dtype=torch.long)
        if drop_last:
            assert flat.unique().numel() == flat.numel() == n // bs * bs
        else:
            assert torch.equal(flat.sort().values, torch.arange(n))
        epochs.append(flat)
    if n > 3 and len(ref):
        assert not torch.equal(epochs[0], epochs[1]) and not torch.equal(epochs[1], epochs[2])
    again = nb.DeviceRayBatches(rays, rgbs, batch_size=bs, drop_last=drop_last, seed=11)
    for e in epochs:
        ep = _epoch_indices(again, rays, rgbs)
        assert torch.equal(torch.cat(ep) if ep else torch.zeros(0, dtype=torch.long), e)


def test_unshuffled_is_in_order(dev):
    rays, rgbs = _dataset(10)
    ep = _epoch_indices(nb.DeviceRayBatches(rays, rgbs, batch_size=4, shuffle=False), rays, rgbs)
    assert [i.tolist() for i in ep] == [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9]]


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("n", [3001, 3000])
def test_rank_shards(world, n, dev):
    """Simulated worlds of 2 and 3: per epoch the ranks' rows are disjoint apart from DistributedSampler's padding,
    cover the dataset, and every rank has the same number of samples and batches."""
    rays, rgbs = _dataset(n, 5)
    ranks = [nb.DeviceRayBatches(rays, rgbs, batch_size=256, seed=3, rank=r, world_size=world) for r in range(world)]
    assert len({len(b) for b in ranks}) == 1
    per_rank = -(-n // world)
    for _ in range(2):
        parts = [torch.cat(_epoch_indices(b, rays, rgbs)) for b in ranks]
        assert all(p.numel() == per_rank for p in parts)
        allidx = torch.cat(parts)
        assert set(allidx.tolist()) == set(range(n))
        assert allidx.numel() - allidx.unique().numel() == per_rank * world - n


def test_unseeded_ranks_share_the_permutation(dev):
    """Ranks whose processes were seeded differently (torch.initial_seed() differs), built with seed=None: their
    shards still come from one permutation per epoch, so they are disjoint and cover the dataset."""
    n, world = 3001, 2
    rays, rgbs = _dataset(n, 6)
    ranks = []
    with torch.random.fork_rng(devices=[dev]):
        for r, s in enumerate((4676324892963314700, 11435171766610437433)):
            torch.manual_seed(s)
            ranks.append(nb.DeviceRayBatches(rays, rgbs, batch_size=256, rank=r, world_size=world))
    for _ in range(2):
        parts = [torch.cat(_epoch_indices(b, rays, rgbs)) for b in ranks]
        allidx = torch.cat(parts)
        assert set(allidx.tolist()) == set(range(n))
        assert allidx.numel() - allidx.unique().numel() == -(-n // world) * world - n


def test_eager_loop_equals_host_fed_loop(dev):
    """20 steps of render_rays_loss -> backward -> FusedAdam on DeviceRayBatches (5 epochs of 4 full batches and a
    partial one) == the same loop fed the same index lists from host tensors moved per batch: losses, the 48
    parameters and the Adam state bit for bit."""
    n, bs, seed = 4 * 1024 + 300, 1024, 77
    emb = [nb.Embedding(3, 10), nb.Embedding(3, 4)]
    rays = torch.from_numpy(orc.make_rays(n, 90))
    rgbs = torch.rand(n, 3, generator=torch.Generator().manual_seed(91))
    batches = nb.DeviceRayBatches(rays, rgbs, batch_size=bs, seed=seed)
    g = torch.Generator(device=dev).manual_seed(seed)
    host_batches = []
    while len(host_batches) < 20:
        perm = torch.randperm(n, device=dev, generator=g).cpu()
        host_batches += [perm[i:i + bs] for i in range(0, n, bs)]
    runs = []
    for feed in ("device", "host"):
        models = [nb.NeRF(), nb.NeRF()]
        for m, w in zip(models, cases.weights()):
            m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in w.items()})
        models = [m.to(dev) for m in models]
        params = [p for m in models for p in m.parameters()]
        opt = nb.FusedAdam(params, lr=5e-4, eps=1e-8)
        losses, step = [], 0
        it = None
        while step < 20:
            if feed == "device":
                if it is None:
                    it = iter(batches)
                b = next(it, None)
                if b is None:
                    it = None
                    continue
                r, c = b["rays"], b["rgbs"]
            else:
                idx = host_batches[step]
                r, c = rays[idx].to(dev), rgbs[idx].to(dev)
            opt.zero_grad(set_to_none=True)
            out = nb.render_rays_loss(models, emb, r, c, 64, False, 1.0, 0.0, 64, 32768, True,
                                      randoms={"seed": 500 + step})
            out["loss"].backward()
            opt.step()
            losses.append(out["loss"].detach().clone())
            step += 1
        runs.append((torch.stack(losses), params, opt))
    (la, pa, oa), (lb, pb, ob) = runs
    assert torch.equal(la, lb)
    for x, y in zip(pa, pb):
        assert torch.equal(x, y)
        for k in ("exp_avg", "exp_avg_sq", "step"):
            assert torch.equal(oa.state[x][k], ob.state[y][k]), k
