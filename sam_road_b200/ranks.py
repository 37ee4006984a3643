"""The process's place among the ranks of torch.distributed, and the per-rank seeds derived from it.

Under DDP every rank usually starts from the same torch.manual_seed, so a seed drawn from torch's default
generator is the same on every rank.  The training batches, the evaluation batches and the dropout masks
therefore key their Philox streams with `rank_seed(drawn, rank)`: rank 0 (and a single process) keeps the
drawn seed, every other rank gets a different one (DESIGN.md §12).

The command-line tools (`inferencer`, `topo_metric`, `apls_metric`) run one process per GPU under torchrun with
`process_group` and `local_gpu`, split their work with `shard`, and end their ranks' shares with `run_checked`, so
that a failure on one rank stops every rank with its message instead of leaving the others at a barrier
(DESIGN.md §17).
"""
from __future__ import annotations

import contextlib
import os
from typing import Iterator, Tuple

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


def local_gpu() -> int:
    """The GPU of this rank on its box: LOCAL_RANK as torchrun sets it, else the rank."""
    return int(os.environ.get("LOCAL_RANK", rank_and_world()[0]))


@contextlib.contextmanager
def process_group() -> Iterator[Tuple[int, int]]:
    """Yields (rank, world size) for a command started by a launcher.  When the launcher set WORLD_SIZE > 1 (with
    RANK, MASTER_ADDR and MASTER_PORT, as torchrun does) and no default process group exists yet, one is initialised
    from that environment: NCCL on this rank's GPU when CUDA is available, else gloo.  A group made here is destroyed
    on exit; one that existed before is left to its owner.  Without a launcher, or with one rank, nothing is
    initialised and this yields (0, 1)."""
    import torch
    import torch.distributed as dist
    made = False
    if int(os.environ.get("WORLD_SIZE", "1")) > 1 and dist.is_available() and not dist.is_initialized():
        if torch.cuda.is_available():
            dev = torch.device("cuda", local_gpu())
            torch.cuda.set_device(dev)
            dist.init_process_group("nccl", device_id=dev)
        else:
            dist.init_process_group("gloo")
        made = True
    try:
        yield rank_and_world()
    finally:
        if made:
            dist.destroy_process_group()


def shard(n: int, rank: int, world: int) -> range:
    """The items of rank `rank` among n: every world-th one from the rank's own index (items rank::world)."""
    if not 0 <= rank < world:
        raise ValueError(f"rank must be in [0, {world}) (got {rank})")
    return range(rank, n, world)


def _collective_device():
    import torch
    import torch.distributed as dist
    return torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")


def broadcast(obj):
    """Rank 0's `obj` on every rank (the object itself in one process).  The others return once rank 0 has called
    this, so what rank 0 did before the call is done when they continue."""
    import torch.distributed as dist
    if rank_and_world()[1] == 1:
        return obj
    box = [obj]
    dist.broadcast_object_list(box, src=0)
    return box[0]


def max_over_ranks(x: float) -> float:
    """The largest of every rank's x (x itself in one process)."""
    import torch
    import torch.distributed as dist
    if rank_and_world()[1] == 1:
        return x
    t = torch.tensor([float(x)], dtype=torch.float64, device=_collective_device())
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def run_checked(fn, *args, **kwargs):
    """fn(*args, **kwargs) as this rank's share of a run, then a status check every rank takes part in.

    In one process an exception from fn propagates unchanged.  With several ranks every rank first finishes its
    share, then one all-reduce finds the lowest rank whose share raised; if there is one, every rank raises a
    RuntimeError with that rank's message (chained to the exception on the rank itself).  So one rank's failure
    fails the run on all of them and no rank is left waiting.  When this returns on any rank, every rank's share
    has returned: the all-reduce is also the barrier after which rank 0 may read what the others wrote."""
    import torch
    import torch.distributed as dist
    rank, world = rank_and_world()
    if world == 1:
        return fn(*args, **kwargs)
    error, out = None, None
    try:
        out = fn(*args, **kwargs)
    except Exception as e:      # reported to every rank below
        error = e
    first = torch.tensor([rank if error is not None else world], dtype=torch.int64, device=_collective_device())
    dist.all_reduce(first, op=dist.ReduceOp.MIN)
    first = int(first.item())
    if first == world:
        return out
    msg = [f"{type(error).__name__}: {error}" if rank == first else None]
    dist.broadcast_object_list(msg, src=first)
    raise RuntimeError(f"rank {first} of {world} failed: {msg[0]}") from error
