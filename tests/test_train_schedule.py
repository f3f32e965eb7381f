"""Host-side arithmetic of the device-resident training loop (no GPU): batches per epoch as ``DataLoader`` counts
them, rank shards as ``DistributedSampler`` makes them, and the epoch / offset schedule of ``CapturedTrainStep``."""
import pytest
import torch
from torch.utils.data import DataLoader, DistributedSampler

from nerf_pl_b200.data import default_seed, next_step_schedule, num_batches, shard_indices, shard_size


@pytest.mark.parametrize("n", [1, 5, 1023, 1024, 1025, 4096, 5000])
@pytest.mark.parametrize("bs", [1, 7, 1024])
@pytest.mark.parametrize("drop_last", [False, True])
def test_num_batches_is_dataloader_len(n, bs, drop_last):
    assert num_batches(n, bs, drop_last) == len(DataLoader(range(n), batch_size=bs, drop_last=drop_last))


@pytest.mark.parametrize("n", [1, 2, 3, 10, 11, 1000, 1001])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_shards_are_distributed_sampler_shards(n, world):
    """shard_indices of an epoch permutation == DistributedSampler's indices of that permutation (its padding
    included), for every rank; the shards have equal length, cover the permutation and overlap only in the padding."""
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(n * 31 + world))
    shards = [shard_indices(perm, r, world) for r in range(world)]
    for r, sh in enumerate(shards):
        ref = list(DistributedSampler(range(n), num_replicas=world, rank=r, shuffle=False))
        assert sh.tolist() == [int(perm[i]) for i in ref]
        assert sh.shape[0] == shard_size(n, world)
    allidx = torch.cat(shards)
    assert set(allidx.tolist()) == set(range(n))
    assert allidx.shape[0] - n == shard_size(n, world) * world - n          # the padding is the only repetition
    if shard_size(n, world) * world == n:
        assert torch.equal(allidx.sort().values, torch.arange(n))


def test_shard_rank_out_of_range():
    with pytest.raises(ValueError):
        shard_indices(torch.arange(4), 2, 2)


@pytest.mark.parametrize("per_epoch", [1, 3, 7])
def test_epoch_schedule(per_epoch):
    """CapturedTrainStep.step()'s schedule (next_step_schedule): step k takes batch k mod per_epoch of epoch
    k // per_epoch; the permutation is redrawn exactly before the first step of every epoch after the first, so the
    device offset (batch * B) is reset there and never passes the last full batch."""
    B, samples = 4, per_epoch * 4 + 3            # a partial batch at the end is never used
    redraws, offset = 0, 0
    for k in range(5 * per_epoch + 2):
        redraw, epoch, batch = next_step_schedule(k, per_epoch)
        assert (epoch, batch) == (k // per_epoch, k % per_epoch)
        assert redraw == (k > 0 and k % per_epoch == 0)
        if redraw:
            redraws += 1
            offset = 0
        assert offset == batch * B and offset + B <= samples
        assert redraws == epoch
        offset += B
    with pytest.raises(ValueError):
        next_step_schedule(0, 0)


def test_default_seed_is_rank_independent_under_ddp():
    """Processes that were never seeded have different torch.initial_seed(); under DDP the default seed must not
    depend on it, or the ranks would shard different permutations."""
    seeds = []
    with torch.random.fork_rng(devices=[]):
        for s in (4676324892963314700, 11435171766610437433):
            torch.manual_seed(s)
            seeds.append((default_seed(None, 2), default_seed(None, 1), default_seed(9, 2)))
    assert seeds[0][0] == seeds[1][0] == 0
    assert seeds[0][1] != seeds[1][1]                  # one process: follows torch.manual_seed
    assert seeds[0][2] == seeds[1][2] == 9
