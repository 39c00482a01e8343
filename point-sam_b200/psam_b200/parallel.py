"""Data-parallel plumbing: clouds are independent units, so the path shards by contiguous ranges of clouds per
rank (weights replicated) and needs exactly one collective - the all_gather of per-cloud metrics at the end
Works with any torch.distributed backend (NCCL on GPUs, gloo in CPU tests)."""
from __future__ import annotations

from typing import List, Tuple

import torch


def shard_range(total: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous split b in [rank*total/world, (rank+1)*total/world); remainders go to the first ranks."""
    base, rem = divmod(total, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def gather_metric(local: torch.Tensor, total: int) -> torch.Tensor:
    """all_gather of per-cloud metric rows [n_local, ...] from every rank -> [total, ...] in cloud order."""
    import torch.distributed as dist

    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return local
    world = dist.get_world_size()
    sizes = [shard_range(total, r, world) for r in range(world)]
    nmax = max(b - a for a, b in sizes)
    pad = torch.zeros((nmax,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    out: List[torch.Tensor] = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(out, pad)
    return torch.cat([o[: b - a] for o, (a, b) in zip(out, sizes)], dim=0)


def plan_graph_chunks(n_local: int, lanes: int, max_chunk: int) -> Tuple[int, int]:
    """Clouds per CUDA graph and number of graphs for a rank's shard of a fixed batch (bench.py config c3): at most
    `max_chunk` clouds per graph, fewer when the shard is small so that `lanes` graphs stay in flight on every rank count
    (8 ranks x 4 clouds: four 1-cloud graphs overlap instead of one 4-cloud graph running alone); the chunk divides the shard."""
    chunk = max(1, min(max_chunk, n_local // max(1, lanes)))
    while chunk > 1 and n_local % chunk:
        chunk -= 1
    return chunk, n_local // max(1, chunk)
