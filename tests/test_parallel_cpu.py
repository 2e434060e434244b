"""world_size-2 gloo tests (CPU) of the N>1 host logic: shard layout covers every unit exactly once, the optional
row gather reassembles the matrix, and the timing reduction is a max over ranks."""
import os

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from builders import free_port


def _worker(rank, world, port, n_total):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from rotate_yolov3_b200 import parallel as P
    lo, hi = P.shard_range(n_total, rank, world)
    full = torch.arange(n_total * 3, dtype=torch.float32).view(n_total, 3)
    got = P.all_gather_rows(full[lo:hi].clone(), n_total)
    assert torch.equal(got, full)
    m = P.max_over_ranks(10.0 + rank, torch.device("cpu"))
    assert m == 10.0 + world - 1
    # every unit owned exactly once
    owner = torch.zeros(n_total, dtype=torch.int32)
    owner[lo:hi] += 1
    dist.all_reduce(owner)
    assert bool((owner == 1).all())
    # data-parallel gradient averaging: one flat all-reduce, parameters without a gradient are skipped
    params = [torch.nn.Parameter(torch.zeros(3, 2)), torch.nn.Parameter(torch.zeros(5)), torch.nn.Parameter(torch.zeros(1))]
    params[0].grad = torch.full((3, 2), float(rank + 1))
    params[1].grad = torch.arange(5, dtype=torch.float32) * (rank + 1)
    P.allreduce_gradients(params)
    mean = sum(range(1, world + 1)) / world
    assert torch.allclose(params[0].grad, torch.full((3, 2), mean))
    assert torch.allclose(params[1].grad, torch.arange(5, dtype=torch.float32) * mean)
    assert params[2].grad is None
    # bucketed all-reduce over a flat arena (what Darknet's backward drives on the GPU with NCCL): buckets are cut at
    # block boundaries, launched as soon as their last gradient is final, and the result is the SUM (finish() returns
    # the 1/world factor the caller applies)
    arena = torch.arange(1000, dtype=torch.float32) * (rank + 1)
    bounds = [100, 130, 400, 410, 900, 1000]
    gb = P.GradBuckets(arena, bounds, bucket_bytes=4 * 250)
    assert gb.buckets == [(0, 400), (400, 900), (900, 1000)] and gb.world == world
    gb.ready(130)
    assert gb.next == 0
    gb.ready(410)
    assert gb.next == 1 and len(gb.works) == 1
    inv = gb.finish()
    assert inv == 1.0 / world and gb.next == 0 and not gb.works
    assert torch.allclose(arena * inv, torch.arange(1000, dtype=torch.float32) * mean)
    dist.destroy_process_group()


def test_shard_range_properties():
    from rotate_yolov3_b200 import parallel as P
    for n in (0, 1, 7, 32, 10000):
        for w in (1, 2, 3, 8):
            spans = [P.shard_range(n, r, w) for r in range(w)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            assert all(spans[i][1] == spans[i + 1][0] for i in range(w - 1))
            sizes = [hi - lo for lo, hi in spans]
            assert max(sizes) - min(sizes) <= 1


def test_two_rank_gloo():
    mp.spawn(_worker, args=(2, free_port(), 37), nprocs=2, join=True)
