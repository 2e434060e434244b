"""Sharding helpers for the multi-GPU form of the hot path (SURVEY.md 8e): every unit of work is independent
(row blocks of the IoU matrix, images for NMS / detection), so ranks take contiguous shards and NO data-path
collective is needed; results are gathered only when a caller wants the whole thing on every rank."""
import torch
import torch.distributed as dist


def shard_range(n, rank, world):
    """contiguous [lo, hi) of n units for `rank`; sizes differ by at most one, earlier ranks take the remainder"""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def all_gather_rows(local, n_total):
    """gather row shards [n_r, ...] (shard_range layout) into [n_total, ...] on every rank (optional epilogue)"""
    world = dist.get_world_size()
    rank = dist.get_rank()
    sizes = [shard_range(n_total, r, world) for r in range(world)]
    maxn = max(hi - lo for lo, hi in sizes)
    pad = torch.zeros((maxn,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    bufs = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(bufs, pad)
    return torch.cat([b[: hi - lo] for b, (lo, hi) in zip(bufs, sizes)], 0)


def max_over_ranks(value, device):
    """timing convention of bench.py: the job takes as long as its slowest rank"""
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def allreduce_gradients(params):
    """Data-parallel training (train.py:168-176 wraps the model in DistributedDataParallel): average the gradients of
    `params` over the ranks with ONE all-reduce of the flattened buffer (NCCL on GPUs, gloo in the CPU tests).  Every rank
    must call it the same number of times.  No-op without an initialised process group / with world size 1."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return
    grads = [p.grad for p in params if p.grad is not None]
    if not grads:
        return
    flat = torch._utils._flatten_dense_tensors(grads)
    dist.all_reduce(flat)
    flat.div_(dist.get_world_size())
    for g, f in zip(grads, torch._utils._unflatten_dense_tensors(flat, grads)):
        g.copy_(f)


class GradBuckets:
    """Bucketed, overlapped gradient all-reduce over one flat fp32 arena (reference: train.py:169-175 wraps the model in
    DistributedDataParallel, whose reducer does the same thing for the reference's modules).

    The training plan lays its parameter gradients out in ONE flat tensor in the order backward produces them
    (last block first); ``boundaries`` are the arena offsets where a block's gradients end.  Buckets are contiguous
    arena ranges of at least ``bucket_bytes`` cut at block boundaries.  ``ready(offset)`` is called by backward when every
    gradient below ``offset`` has been produced: each bucket that became complete is all-reduced asynchronously on a side
    stream (NCCL) -- overlapping the rest of backward -- and ``finish()`` makes the caller's stream wait for all of them.
    ``ranges`` (default: the whole arena) are the sorted, disjoint parts of the arena that hold trainable parameters'
    gradients; buckets never leave them, so frozen parameters are not all-reduced (like torch DDP's reducer).
    Device-agnostic (gloo on CPU in the tests: streams are skipped there)."""

    def __init__(self, arena, boundaries, bucket_bytes=32 << 20, group=None, ranges=None):
        self.arena, self.group = arena, group
        self.world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
        cap = max(1, bucket_bytes // arena.element_size())
        self.buckets = []                      # (lo, hi) element ranges
        for r_lo, r_hi in (ranges if ranges is not None else [(0, arena.numel())]):
            lo = r_lo
            for b in boundaries:
                if lo < b < r_hi and b - lo >= cap:
                    self.buckets.append((lo, b))
                    lo = b
            if lo < r_hi:
                self.buckets.append((lo, r_hi))
        self.cuda = arena.is_cuda
        self.stream = torch.cuda.Stream(device=arena.device) if self.cuda else None
        self.reset()

    def reset(self):
        self.next = 0
        self.works = []

    def ready(self, offset):
        """every gradient in arena[:offset] is final (as far as the caller's stream is concerned)"""
        if self.world == 1:
            return
        while self.next < len(self.buckets) and self.buckets[self.next][1] <= offset:
            lo, hi = self.buckets[self.next]
            self.next += 1
            view = self.arena[lo:hi]
            if self.cuda:
                ev = torch.cuda.Event()
                ev.record(torch.cuda.current_stream(self.arena.device))
                self.stream.wait_event(ev)
                with torch.cuda.stream(self.stream):
                    self.works.append(dist.all_reduce(view, group=self.group, async_op=True))
            else:
                self.works.append(dist.all_reduce(view, group=self.group, async_op=True))

    def finish(self):
        """flush the remaining buckets and make the current stream wait for every all-reduce; returns 1 / world"""
        self.ready(self.arena.numel())
        if self.cuda and self.works:
            # the collectives were enqueued from the side stream; work.wait() orders them before the CURRENT stream
            for w in self.works:
                w.wait()
            torch.cuda.current_stream(self.arena.device).wait_stream(self.stream)
        else:
            for w in self.works:
                w.wait()
        self.works = []
        self.next = 0
        return 1.0 / self.world


class DistributedDataParallel(torch.nn.Module):
    """Drop-in for the ``torch.nn.parallel.DistributedDataParallel(model)`` wrap of train.py:175: ``.module`` is the
    wrapped Darknet, forward is delegated.  Instead of autograd hooks, the Darknet's own backward (train_path.py) hands
    finished gradient buckets to GradBuckets, so the NCCL all-reduce of bucket k overlaps the backward kernels of the
    blocks before it; the gradients autograd receives are already averaged over the ranks."""

    def __init__(self, module, bucket_mb=32, process_group=None, reserved_sms=0):
        super().__init__()
        self.module = module
        # reserved_sms: SMs the backward GEMMs leave to the concurrent NCCL kernels.  The default leaves every SM to the
        # GEMMs; the argument is for rank counts where the all-reduce competes with them
        module._ddp = {"bucket_bytes": int(bucket_mb * (1 << 20)), "group": process_group, "reserved_sms": int(reserved_sms)}
        module.drop_training_plans()  # the plans build their buckets at construction
        module._pplan = None

    def forward(self, *a, **k):
        return self.module(*a, **k)


class DevicePrefetcher:
    """Host -> device double buffering for the training loop (the reference copies each batch synchronously,
    train.py:262-263 `imgs = imgs.to(device)`): the pinned host tensors of step i+1 are copied on a side stream while
    step i computes; `get()` makes the compute stream wait for the copy it hands out.

        pf = DevicePrefetcher(device)
        pf.put(imgs_h, targets_h)                # start copying batch 0
        for ...:
            imgs, targets = pf.get()             # batch i on the device
            pf.put(next_imgs_h, next_targets_h)  # batch i+1 copies while the step below runs
            loss = ...; loss.backward(); opt.step()
    """

    def __init__(self, device):
        self.device = torch.device(device)
        self.stream = torch.cuda.Stream(device=self.device)
        self._pending = None

    def put(self, *host_tensors):
        with torch.cuda.stream(self.stream):
            dev = [t.to(self.device, non_blocking=True) for t in host_tensors]
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self._pending = (dev, ev)

    def get(self):
        if self._pending is None:
            raise RuntimeError("DevicePrefetcher.get() without a pending batch: call put(...) first")
        dev, ev = self._pending
        self._pending = None
        cur = torch.cuda.current_stream(self.device)
        cur.wait_event(ev)
        for t in dev:
            t.record_stream(cur)        # the caching allocator must not recycle it under the consumer
        return dev
