"""Data-parallel plumbing: clouds are independent units, so the path shards by contiguous ranges of clouds per
rank (weights replicated) and needs exactly one collective - the all_gather of per-cloud metrics at the end
Works with any torch.distributed backend (NCCL on GPUs, gloo in CPU tests).  Also the plan that cuts clouds of different
sizes into padded batches (plan_eval_batches)."""
from __future__ import annotations

from typing import Dict, Hashable, List, Sequence, Tuple

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


def plan_eval_batches(sizes: Sequence[int], keys: Sequence[Hashable], batch_size: int,
                      max_batch_points: int) -> List[List[int]]:
    """Batches of crop indices for forward_varlen (evaluation/eval_kitti.py) and for the crop batches of
    PointCloudMaskGenerator.generate_packed_batch_crops.  Crops are grouped by key (their group shape: crops of different
    shapes need different G / K and never share a batch), each group is sorted by size so that the padding stays small,
    and runs of at most batch_size crops with len(batch) * N_max <= max_batch_points are cut from it (a crop larger than
    the cap runs alone).  The cap bounds the decoder's upscaling input, B * M * N_max * Du * 4 bytes.  Groups come in
    order of first appearance; every crop appears exactly once."""
    if batch_size < 1 or max_batch_points < 1:
        raise ValueError(f"batch_size ({batch_size}) and max_batch_points ({max_batch_points}) must be >= 1")
    if len(sizes) != len(keys):
        raise ValueError(f"{len(sizes)} sizes and {len(keys)} keys")
    groups: Dict[Hashable, List[int]] = {}
    for i, k in enumerate(keys):
        groups.setdefault(k, []).append(i)
    batches: List[List[int]] = []
    for idx in groups.values():
        cur: List[int] = []
        for i in sorted(idx, key=lambda j: (sizes[j], j)):
            if cur and (len(cur) + 1 > batch_size or (len(cur) + 1) * sizes[i] > max_batch_points):
                batches.append(cur)
                cur = []
            cur.append(i)
        batches.append(cur)
    return batches
