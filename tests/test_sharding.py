"""Multi-GPU host logic on CPU: world_size-2 (and 3) gloo process groups exercise the head partition and the
scatter/gather plumbing bench.py and clients use around the single-GPU kernels."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def test_head_partition_covers_every_head_exactly_once():
    from mfa_b200.sharding import head_partition
    for total in (0, 1, 7, 64, 2048, 2049):
        for world in (1, 2, 3, 4, 8):
            owned = []
            counts = []
            for rank in range(world):
                start, count = head_partition(total, world, rank)
                owned.extend(range(start, start + count))
                counts.append(count)
            assert owned == list(range(total))
            assert max(counts) - min(counts) <= 1
    # BASELINE.json configs[4]: batch 64 x heads 32 = 2048 problems over 8 GPUs -> 256 each
    assert head_partition(2048, 8, 3) == (768, 256)
    with pytest.raises(ValueError):
        head_partition(8, 2, 2)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, total_heads, results):
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import mfa_b200  # noqa: F401
    from mfa_b200.sharding import gather_heads, head_partition, max_over_ranks, scatter_heads

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        gen = torch.Generator().manual_seed(0)
        full_q = torch.randn(total_heads, 16, 8, generator=gen) if rank == 0 else None
        shard = scatter_heads(full_q, total_heads, (16, 8), torch.float32, "cpu")
        start, count = head_partition(total_heads, world, rank)
        assert shard.shape == (count, 16, 8)
        # stand-in for the per-rank kernel: something head-local and rank-dependent
        out = shard * 2.0 + float(start)
        gathered = gather_heads(out, total_heads)
        slowest = max_over_ranks(float(rank + 1), "cpu")
        assert slowest == float(world)
        if rank == 0:
            expected = full_q * 2.0
            for r in range(world):
                s, c = head_partition(total_heads, world, r)
                expected[s:s + c] += float(s)
            results.put(bool(torch.equal(gathered, expected)))
        else:
            assert gathered is None
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,total_heads", [(2, 6), (2, 5), (3, 4)])
def test_scatter_compute_gather_round_trip_gloo(world, total_heads):
    ctx = mp.get_context("spawn")
    results = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, total_heads, results)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert results.get(timeout=10) is True
