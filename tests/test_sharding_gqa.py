"""Grouped K/V on the multi-GPU plumbing, over world-size 2 and 3 gloo process groups on CPU: query heads are scattered
in whole groups (sharding.scatter_heads(kv_group=G)), each rank's K/V shard is the plain partition of the total / G K/V
heads, and the per-rank results (query heads, and dK / dV already summed per group) gather back in order.

(Kept apart from tests/test_kv_group.py, like tests/test_sharding.py: the spawned gloo workers run after the tests that
trace kernels with torch.profiler.)"""
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sharding_worker(rank, world, port, total, G, results):
    import sys
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    from mfa_b200.sharding import gather_heads, head_partition, scatter_heads

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        gen = torch.Generator().manual_seed(0)
        full_q = torch.randn(total, 6, 4, generator=gen) if rank == 0 else None
        full_k = torch.randn(total // G, 5, 4, generator=gen) if rank == 0 else None
        q = scatter_heads(full_q, total, (6, 4), torch.float32, "cpu", kv_group=G)
        k = scatter_heads(full_k, total // G, (5, 4), torch.float32, "cpu")
        start, count = head_partition(total, world, rank, kv_group=G)
        assert q.shape[0] == count and k.shape[0] == count // G
        # stand-in for the grouped kernel: each query head plus the sum of its K/V head, and dK summed per group
        out = q + k.repeat_interleave(G, dim=0).sum(dim=(1, 2), keepdim=True)
        dk = k * float(G)
        gathered = gather_heads(out, total, kv_group=G)
        gathered_k = gather_heads(dk, total // G)
        if rank == 0:
            expected = full_q + full_k.repeat_interleave(G, dim=0).sum(dim=(1, 2), keepdim=True)
            results.put(bool(torch.equal(gathered, expected)) and bool(torch.equal(gathered_k, full_k * float(G))))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,total,G", [(2, 8, 4), (3, 12, 2), (2, 6, 3)])
def test_grouped_scatter_gather_round_trip_gloo(world, total, G):
    import torch.multiprocessing as mp
    from tests.test_sharding import _free_port
    ctx = mp.get_context("spawn")
    results = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_sharding_worker, args=(r, world, port, total, G, results)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert results.get(timeout=10) is True
