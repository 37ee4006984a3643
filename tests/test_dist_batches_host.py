"""CPU: the per-rank batches of sam_road_b200.dataset under torch.distributed -- evaluation shards equal
DistributedSampler's (shuffle=False, drop_last=False), per-rank lengths, and the per-rank seed derivation shared
by the batches and the dropout masks (sam_road_b200.ranks)."""
import numpy as np
import pytest
import torch.utils.data

from sam_road_b200 import dataset as D
from sam_road_b200 import ranks

WORLDS = (1, 2, 3, 8)
SIZES = ("1", "5", "W", "W+1", "97")


def _n(size, world):
    return {"1": 1, "5": 5, "W": world, "W+1": world + 1, "97": 97}[size]


def _sampler(n, rank, world):
    return list(torch.utils.data.DistributedSampler(range(n), num_replicas=world, rank=rank, shuffle=False,
                                                    drop_last=False))


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("size", SIZES)
def test_eval_shard_equals_distributed_sampler(size, world):
    n = _n(size, world)
    for rank in range(world):
        assert D.eval_shard(n, rank, world).tolist() == _sampler(n, rank, world), (n, rank, world)
    with pytest.raises(ValueError, match="rank"):
        D.eval_shard(n, world, world)


class _Scenes:
    """Stands in for LabelScenes: a batch is the patch rows it was asked for, or the drawn count."""

    def batch(self, B, patches=None, seed=None):
        return patches if patches is not None else B


def _dataset(is_train, n_eval=0):
    ds = D.SatMapDataset.__new__(D.SatMapDataset)
    ds.is_train, ds.dataset, ds._scenes = is_train, "spacenet", _Scenes()
    ds.eval_patches = [(i, (3 * i, 5 * i), None) for i in range(n_eval)]
    return ds


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("B", [1, 4])
def test_eval_loader_serves_this_ranks_shard(size, world, B, monkeypatch):
    n = _n(size, world)
    ds = _dataset(False, n)
    for rank in range(world):
        monkeypatch.setattr(ranks, "rank_and_world", lambda: (rank, world))
        loader = ds.loader(B)
        batches = list(loader)
        want = _sampler(n, rank, world)
        assert len(loader) == len(batches) == -(-len(want) // B)
        assert all(b.shape[0] == B for b in batches[:-1]) and 1 <= batches[-1].shape[0] <= B
        rows = np.concatenate(batches)
        assert rows[:, 0].tolist() == want
        assert rows[:, 1].tolist() == [3 * i for i in want] and rows[:, 2].tolist() == [5 * i for i in want]
        assert not rows[:, 3].any()


@pytest.mark.parametrize("world", WORLDS)
def test_train_loader_length_per_rank(world, monkeypatch):
    ds = _dataset(True)
    n = len(ds)                                   # spacenet: 84667 training samples per epoch
    B = 16
    for rank in range(world):
        monkeypatch.setattr(ranks, "rank_and_world", lambda: (rank, world))
        loader = ds.loader(B)
        sizes = list(loader)
        per_rank = -(-n // world)
        assert len(loader) == len(sizes) == -(-per_rank // B)
        assert sum(sizes) == per_rank and all(s == B for s in sizes[:-1])


def test_single_process_is_world_one():
    assert ranks.rank_and_world() == (0, 1)


def test_rank_seed_keeps_rank0_and_separates_ranks():
    rng = np.random.RandomState(0)
    seeds = [0, 1, 2 ** 62 - 1] + [int(s) for s in rng.randint(0, 2 ** 62, 20, dtype=np.int64)]
    for s in seeds:
        assert ranks.rank_seed(s, 0) == s
        derived = [ranks.rank_seed(s, r) for r in range(8)]
        assert len(set(derived)) == 8, s
        assert all(0 <= d < 2 ** 64 for d in derived)
        assert derived == [ranks.rank_seed(s, r) for r in range(8)]
    # the same rank never maps two seeds to one
    assert len({ranks.rank_seed(s, 5) for s in seeds}) == len(seeds)
    with pytest.raises(ValueError, match="rank"):
        ranks.rank_seed(1, -1)
