"""The process's place among the ranks of torch.distributed, and the per-rank seeds derived from it.

Under DDP every rank usually starts from the same torch.manual_seed, so a seed drawn from torch's default
generator is the same on every rank.  The training batches, the evaluation batches and the dropout masks
therefore key their Philox streams with `rank_seed(drawn, rank)`: rank 0 (and a single process) keeps the
drawn seed, every other rank gets a different one (DESIGN.md §12).
"""
from __future__ import annotations

from typing import Tuple

_M64 = (1 << 64) - 1
_GOLDEN = 0x9E3779B97F4A7C15      # odd, so rank -> rank * _GOLDEN is a bijection of the 64-bit integers


def rank_and_world() -> Tuple[int, int]:
    """(rank, world size) of the default process group when torch.distributed is initialised, else (0, 1)."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def _mix64(z: int) -> int:
    """SplitMix64's finaliser: a bijection of the 64-bit integers that maps 0 to 0."""
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def rank_seed(seed: int, rank: int) -> int:
    """The 64-bit Philox seed rank `rank` uses for the drawn `seed`: seed itself on rank 0, and for a fixed seed
    a different value on every rank (the XOR mask is a bijection of the rank)."""
    if rank < 0:
        raise ValueError(f"rank must be >= 0 (got {rank})")
    return (int(seed) ^ _mix64((int(rank) * _GOLDEN) & _M64)) & _M64


def draw_seed() -> int:
    """A seed drawn from torch's default generator (62 bits), made per rank with rank_seed."""
    import torch
    return rank_seed(int(torch.randint(0, 2 ** 62, (), dtype=torch.int64).item()), rank_and_world()[0])
