"""Multi-GPU plumbing for the attention hot path: independent (batch x head) problems are the only unit that
shards (the reference is single-head; multi-head is a stride change, AttentionKernelDescriptor.swift:36-42).

Every rank runs the SAME single-GPU kernels on its contiguous block of heads; the computation itself has no
exchange step, so there is no data-path collective.  torch.distributed (NCCL over NVLink on GPUs, gloo in the
CPU tests) is used only for the trivial "inputs start on rank 0 / outputs end on rank 0" scatter and gather.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
import torch.distributed as dist


def head_partition(total_heads: int, world_size: int, rank: int, kv_group: int = 1) -> Tuple[int, int]:
    """Contiguous block partition [start, start + count) of `total_heads` problems for `rank`; the first
    (total % world) ranks take one extra so counts differ by at most one.

    Grouped K/V (kv_group query heads share one K/V head): the partition is in whole groups, so a rank's query heads
    [start, start + count) read exactly the K/V heads [start / kv_group, (start + count) / kv_group), which is
    head_partition(total_heads / kv_group, world_size, rank) -- the partition to shard K and V (and dK, dV) with."""
    if total_heads < 0 or world_size <= 0 or not 0 <= rank < world_size or kv_group < 1:
        raise ValueError("invalid partition request")
    if total_heads % kv_group:
        raise ValueError(f"{total_heads} heads are not a whole number of groups of {kv_group}")
    base, extra = divmod(total_heads // kv_group, world_size)
    start = rank * base + min(rank, extra)
    return start * kv_group, (base + (1 if rank < extra else 0)) * kv_group


def scatter_heads(full: Optional[torch.Tensor], total_heads: int, tail_shape, dtype, device, src: int = 0,
                  group=None, kv_group: int = 1) -> torch.Tensor:
    """Rank `src` holds `full` = [total_heads, *tail_shape]; every rank returns its [count, *tail_shape] shard
    (head_partition with `kv_group`; `group` is the process group).
    Point-to-point sends (ncclSend/ncclRecv under NCCL, posted as ONE batch so that the transfers to all peers run
    concurrently over NVSwitch instead of one after the other), no collective on the compute path."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    start, count = head_partition(total_heads, world, rank, kv_group)
    if rank == src:
        assert full is not None and full.shape[0] == total_heads
        ops = []
        for peer in range(world):
            if peer == src:
                continue
            ps, pc = head_partition(total_heads, world, peer, kv_group)
            if pc:
                ops.append(dist.P2POp(dist.isend, full[ps:ps + pc], peer, group))
        requests = dist.batch_isend_irecv(ops) if ops else []
        shard = full[start:start + count].clone()
        for r in requests:
            r.wait()
        return shard
    shard = torch.empty((count, *tail_shape), dtype=dtype, device=device)
    if count:
        for r in dist.batch_isend_irecv([dist.P2POp(dist.irecv, shard, src, group)]):
            r.wait()
    return shard


def gather_heads(shard: torch.Tensor, total_heads: int, dst: int = 0, group=None,
                 out: Optional[torch.Tensor] = None, kv_group: int = 1) -> Optional[torch.Tensor]:
    """Inverse of scatter_heads: rank `dst` returns [total_heads, ...] (written into `out` when given, so that a caller
    timing the transfer does not time a multi-gigabyte allocation), the others None.  All receives are posted as one
    batch."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    if rank != dst:
        if shard.shape[0]:
            for r in dist.batch_isend_irecv([dist.P2POp(dist.isend, shard.contiguous(), dst, group)]):
                r.wait()
        return None
    full = out if out is not None else torch.empty((total_heads, *shard.shape[1:]), dtype=shard.dtype,
                                                   device=shard.device)
    assert full.shape[0] == total_heads and full.shape[1:] == shard.shape[1:]
    ops = []
    for peer in range(world):
        ps, pc = head_partition(total_heads, world, peer, kv_group)
        if pc == 0:
            continue
        if peer == dst:
            full[ps:ps + pc] = shard
        else:
            ops.append(dist.P2POp(dist.irecv, full[ps:ps + pc], peer, group))
    for r in (dist.batch_isend_irecv(ops) if ops else []):
        r.wait()
    return full


def max_over_ranks(value: float, device, group=None) -> float:
    """Device-timed durations are reduced with MAX over ranks (the slowest rank defines the step)."""
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return float(t.item())
