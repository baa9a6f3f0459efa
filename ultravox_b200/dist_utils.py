"""Multi-GPU helpers (one process per GPU; env-var rank discovery like ref:ultravox/utils/device_helpers.py:7-45).

Inference shards clips across ranks with NO data-path collective (``shard_indices``, the reference's
``sharded_batch_iterator`` rule i % world == rank, ref:ultravox/training/ddp_utils.py:57-69); adapter training has exactly
one exchange, ``allreduce_mean_`` on the flat projector gradient (SURVEY.md 8e)."""
from __future__ import annotations

import os

import torch
import torch.distributed as dist


def world_size() -> int:
    return int(os.environ.get("WORLD_SIZE", "1"))


def rank() -> int:
    return int(os.environ.get("RANK", "0"))


def local_rank() -> int:
    return int(os.environ.get("LOCAL_RANK", "0"))


def shard_indices(n_items: int, shard: int, n_shards: int) -> list[int]:
    return [i for i in range(n_items) if i % n_shards == shard]


def group_world_size(group=None) -> int:
    """Ranks in the data-parallel group (1 without an initialised process group)."""
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(group)
    return 1


def allreduce_sum_(flat: torch.Tensor, group=None) -> float:
    """In-place SUM over the data-parallel group; returns 1 / world for the caller to fold into its next kernel (the optimizer
    step reads the gradient anyway: a separate x 1/world pass over the flat buffer is a wasted HBM round trip)."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
        return 1.0 / dist.get_world_size(group)
    return 1.0


def allreduce_mean_(flat: torch.Tensor, group=None) -> torch.Tensor:
    """In-place mean over the data-parallel group (sum all-reduce, then 1/world)."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
        flat.mul_(1.0 / dist.get_world_size(group))
    return flat


def max_over_ranks(value: float, device=None, group=None) -> float:
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return value
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return float(t)
