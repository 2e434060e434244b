"""Data-parallel training over NCCL (rows a11 / 8e): two ranks, one process per GPU, `parallel.DistributedDataParallel`
(bucketed all-reduce overlapped with backward, CUDA-graph segments) -- the gradients every rank ends up with must equal
the mean of the two ranks' local gradients computed WITHOUT the wrapper (per-replica BatchNorm like the reference,
model/models.py:62).  Needs >= 2 GPUs (skipped otherwise)."""
import os

import pytest
import torch

import helpers
from builders import free_port

pytestmark = pytest.mark.gpu


def _local_grads(rank, use_graph, steps=1):
    import rotate_yolov3_b200 as pkg
    m = pkg.Darknet(helpers.mini_cfg(64, 48), {"context_factor": 1.0})
    helpers.init_darknet_weights(m, seed=5)
    m = m.cuda().train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.momentum = 0.0                                   # identical forwards across repetitions
    m.use_cuda_graph = use_graph
    x = torch.rand(4, 3, 48, 64, generator=torch.Generator().manual_seed(100 + rank)).cuda()
    return m, x


def _worker(rank, world, port, use_graph, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    import torch.distributed as dist
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from rotate_yolov3_b200 import parallel
    # reference: each rank's own gradients, no wrapper
    m, x = _local_grads(rank, False)
    sum(p.float().pow(2).mean() for p in m(x)).backward()
    local = torch.cat([p.grad.reshape(-1) for p in m.parameters()])
    want = local.clone()
    dist.all_reduce(want)
    want /= world
    # wrapped: bucketed overlapped all-reduce inside backward (tiny buckets so that several are in flight)
    m2, x2 = _local_grads(rank, use_graph)
    ddp = parallel.DistributedDataParallel(m2, bucket_mb=0)
    m2._ddp["bucket_bytes"] = 64 << 10
    got = None
    for _ in range(3 if use_graph else 1):                       # graph mode: eager+capture step, then replayed steps
        for p in m2.parameters():
            p.grad = None
        sum(p.float().pow(2).mean() for p in ddp(x2)).backward()
        got = torch.cat([p.grad.reshape(-1) for p in m2.parameters()])
    nb = len(m2._tplan.buckets.buckets)
    err = float((got - want).abs().max() / want.abs().max())
    q.put((rank, err, nb))
    dist.destroy_process_group()


@pytest.mark.parametrize("use_graph", [False, True])
def test_two_rank_nccl_gradients_equal_mean_of_local_gradients(use_graph):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, use_graph, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    res = sorted(q.get() for _ in range(2))
    for rank, err, nb in res:
        assert nb >= 3, nb                                       # several buckets were all-reduced during backward
        # split-K atomics reorder fp32 sums between two runs of the same backward: rounding-level differences only
        assert err <= 2e-2, (rank, err)
