"""Data-parallel plumbing of the hot path: the batch (independent sequences / images) is sharded
across one-process-per-GPU ranks, weights are replicated, and ONE collective per step gathers the
per-rank results -- replacing the reference's rank-file + barrier gather
(utils/caption_collect.py:7-37, utils/misc.py:277-280).  There is no collective inside the forward."""
from __future__ import annotations

from typing import List

import torch


def shard_range(n_items: int, rank: int, world: int) -> List[int]:
    """Indices of the global batch owned by ``rank``: ``i::world`` -- what ``accelerator.prepare(DataLoader)``
    gives the reference (engine/lmm_trainer.py:1315)."""
    return list(range(rank, n_items, world))


def gather_results(local: torch.Tensor, n_items: int, rank: int, world: int, group=None) -> torch.Tensor:
    """All-gather the per-rank result rows (same trailing shape on every rank) and put them back in global
    batch order.  Ranks may own different numbers of rows (n_items not divisible by world): rows are padded
    to the maximum for the collective.  NCCL on GPUs (NVLink / NVSwitch), gloo in the CPU tests."""
    import torch.distributed as dist
    if world == 1:
        return local
    per_rank = [len(shard_range(n_items, r, world)) for r in range(world)]
    width = max(per_rank)
    pad = local.new_zeros((width,) + tuple(local.shape[1:]))
    pad[: local.shape[0]] = local
    bufs = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(bufs, pad, group=group)
    out = local.new_empty((n_items,) + tuple(local.shape[1:]))
    for r in range(world):
        out[r::world] = bufs[r][: per_rank[r]]
    return out
