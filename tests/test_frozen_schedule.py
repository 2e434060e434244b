"""The backward schedules of trainable masks (train_path.Schedule), on CPU plans: with every parameter trainable the
schedule is the full plan; the reference's --prebias / --transfer / frozen-backbone masks (train.py:120-135, :215-220)
run only what their trainable parameters need; for random masks every writer of a needed gradient range runs with its
full-plan accumulate flag and no launch runs whose whole output is unused.  "Needed" is restated here from the parameter
sets upstream of every tensor, not from the schedule's own walk.  The arena ranges and the DDP buckets of a mask cover
exactly its trainable parameters."""
import os
import random

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from builders import free_port, graph_model, m_model


CPU = torch.device("cpu")
CFGS = ["cfg/yolov3.cfg", "cfg/HRSC+/yolov3_512_se.cfg", "cfg/yolov3-m.cfg"]


def _plan(name):
    from rotate_yolov3_b200.train_path import TrainPlan
    m, h, w = (m_model(), 64, 64) if name.endswith("yolov3-m.cfg") else graph_model(name)
    return m, TrainPlan(m, 1, h, w, CPU)


def masks(m):
    nf = int(m.module_defs[m.yolo_layers[0] - 1]["filters"])
    named = list(m.named_parameters())
    return {"prebias": tuple(p.numel() == nf for _, p in named),
            "transfer": tuple(p.shape[0] == nf for _, p in named),
            "cutoff75": tuple(int(n.split(".")[1]) >= 75 for n, _ in named)}


def _full_ops(plan):
    """every launch the plan has, restated from the block structure"""
    out = [("head", b.i, None) for b in plan.blocks if b.is_head]
    for b in reversed(plan.blocks):
        if b.se is not None:
            out.append(("se", b.se.i, b.se.gx_acc))
        if not b.is_head:
            out.append(("bnact", b.i, b.gres_acc if b.gres is not None else None))
        out.append(("wgrad", b.i, None))
        if b.gsrc is not None:
            out.append(("dgrad", b.i, (b.gsrc_acc, b.dxs_direct)))
    return out


def _upstream(plan):
    """per gradient view: the parameters its tensor depends on (a forward walk over the gradient twins of the activation
    views and their channel ranges)"""
    written = {}

    def params_of(v):
        if v is None or v.buf is None:
            return frozenset()
        lo, hi = v.ch_off, v.ch_off + v.c
        return frozenset().union(*[s for a, b, s in written.get(id(v.buf), []) if a < hi and lo < b])

    for b in plan.blocks:
        own = {k for k in plan.param_slots if k[0] == (b.owner if b.owner is not None else b.i)
               and (b.owner is None or k[1] == "Conv2d.weight")}
        if b.is_head:
            continue
        s = own | params_of(b.gsrc) | params_of(b.gres)
        written.setdefault(id(b.gy.buf), []).append((b.gy.ch_off, b.gy.ch_off + b.gy.c, s))
        if b.se is not None:
            s = s | {k for k in plan.param_slots if k[0] == b.se.i}
            written.setdefault(id(b.se.gu.buf), []).append((b.se.gu.ch_off, b.se.gu.ch_off + b.se.gu.c, s))
    return params_of, written


def _check(plan, sch):
    from rotate_yolov3_b200 import graph as G
    tr = sch.trainable
    params_of, producers = _upstream(plan)
    need = lambda v: bool(params_of(v) & tr)           # noqa: E731
    ops = sch.ops(plan)
    ran = {(k, i) for k, i, _ in ops}
    written = {}
    for b in reversed(plan.blocks):
        wi = b.owner if b.owner is not None else b.i
        writes = [("se", b.se.i if b.se is not None else None, b.se.gx if b.se is not None else None),
                  ("bnact", b.i, b.gres), ("dgrad", b.i, b.gsrc)]
        for kind, i, v in writes:
            if v is None:
                continue
            if need(v):
                assert (kind, i) in ran, ("needed range not written", kind, i)
            if (kind, i) in ran:
                acc = G.claim(written, v)
                full = {"se": getattr(b.se, "gx_acc", None), "bnact": b.gres_acc, "dgrad": b.gsrc_acc}[kind]
                if need(v):
                    assert acc == full, ("accumulate flag", kind, i)
        # nothing runs whose whole output is unused
        own = {k for k in tr if k[0] == b.i}
        if ("wgrad", b.i) in ran:
            assert (wi, "Conv2d.weight") in tr
        if ("dgrad", b.i) in ran:
            assert need(b.gsrc)
            if not all(params_of(G.View(b.gsrc.buf, b.gsrc.ch_off + c, 8, 1, 1)) & tr for c in range(0, b.gsrc.c, 8)):
                # the allowed partial case: a concat consumer's dgrad also writes a frozen producer's range
                lo, hi = b.gsrc.ch_off, b.gsrc.ch_off + b.gsrc.c
                assert len({(a, b_) for a, b_, _ in producers[id(b.gsrc.buf)] if a < hi and lo < b_}) > 1, b.i
        if ("bnact", b.i) in ran:
            assert (("wgrad", b.i) in ran or ("dgrad", b.i) in ran or (b.gres is not None and need(b.gres))
                    or (b.owner is None and own - {(b.i, "Conv2d.weight")}))
        if b.se is not None and ("se", b.se.i) in ran:
            assert need(b.se.gx) or any(k[0] == b.se.i for k in tr)
        if ("head", b.i) in ran:
            assert (wi, "Conv2d.weight") in tr or need(b.gsrc)
        if ("head_bias", b.i) in ran:
            assert (b.i, "Conv2d.bias") in tr and ("head", b.i) not in ran
    # the ranges handed back: exactly the pieces holding a trainable parameter
    for lo, hi, keys in plan.pieces:
        inside = any(a <= lo and hi <= b_ for a, b_ in sch.ranges)
        assert inside == any(k in tr for k in keys), (lo, hi, keys)
    return ops


@pytest.mark.parametrize("name", CFGS)
def test_all_trainable_is_the_full_plan(name):
    m, plan = _plan(name)
    sch = plan._schedule((True,) * len(plan.names))
    assert sch is plan.sched
    assert sch.ops(plan) == _full_ops(plan)
    assert sch.ranges == [(0, plan.garena.numel())] and sch.dw_ranges == [(0, plan.dw_arena.numel())]
    assert len(sch.segments) == 1 and sch.segments[0] == list(reversed(plan.blocks))
    assert sch.pwd_used == {b.i for b in plan.blocks if b.owner is None and b.i > 0}


@pytest.mark.parametrize("name", CFGS)
def test_reference_masks(name):
    m, plan = _plan(name)
    ms = masks(m)
    heads = [b for b in plan.blocks if b.is_head]
    owners = [b for b in heads if b.owner is None]
    pre = _check(plan, plan._schedule(ms["prebias"]))
    assert sorted(pre) == sorted(("head_bias", b.i, None) for b in owners)
    tra = _check(plan, plan._schedule(ms["transfer"]))
    assert sorted(k for k, _, _ in tra) == sorted(["head"] * len(heads) + ["wgrad"] * len(heads))
    cut = _check(plan, plan._schedule(ms["cutoff75"]))
    assert all(i >= 75 for _, i, _ in cut)
    dg = {i for k, i, _ in cut if k == "dgrad"}
    for i, d in enumerate(m.module_defs):
        if i >= 75 and d["type"] == "route" and "," in d["layers"]:
            assert i + 1 in dg, i                    # the concat's consumer still runs its dgrad
    assert 75 not in dg
    # a switch back selects the cached schedule; nothing is rebuilt
    assert plan._schedule(ms["prebias"]) is plan._schedule(ms["prebias"])


@pytest.mark.parametrize("name", CFGS)
def test_random_masks(name):
    m, plan = _plan(name)
    rng = random.Random(1234)
    n = len(plan.names)
    for trial in range(12):
        p = [0.02, 0.1, 0.5, 0.9][trial % 4]
        mask = tuple(rng.random() < p for _ in range(n))
        _check(plan, plan._schedule(mask))


def _bucket_worker(rank, world, port):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from rotate_yolov3_b200.train_path import TrainPlan
    m, h, w = graph_model("cfg/yolov3.cfg")
    m._ddp = {"bucket_bytes": 1 << 20, "group": None, "reserved_sms": 0}
    plan = TrainPlan(m, 1, h, w, CPU)
    full = plan.sched
    assert [b for b in full.buckets.buckets] == [b for b in full.buckets.buckets if b[1] in plan.bounds]
    for name, mask in masks(m).items():
        sch = plan._schedule(mask)
        bk = sch.buckets.buckets
        # buckets tile the trainable ranges exactly
        assert sorted(bk) == bk and all(any(a <= lo and hi <= b for a, b in sch.ranges) for lo, hi in bk)
        assert sum(hi - lo for lo, hi in bk) == sum(hi - lo for lo, hi in sch.ranges)
        # every bucket is complete at its segment's ready offset
        done = set()
        for seg, ready in zip(sch.segments, sch.ready):
            done |= {b for b in bk if b[1] <= ready}
        assert done == set(bk)
        base = (torch.arange(plan.garena.numel()) % 1000).float()
        plan.garena.copy_(base * (rank + 1))
        for ready in sch.ready:
            sch.buckets.ready(ready)
        inv = sch.buckets.finish()
        inside = torch.zeros(plan.garena.numel(), dtype=torch.bool)
        for lo, hi in sch.ranges:
            inside[lo:hi] = True
        assert torch.equal(plan.garena[inside] * inv, base[inside] * 1.5), name       # mean over ranks 1 and 2
        assert torch.equal(plan.garena[~inside], base[~inside] * (rank + 1)), name    # frozen: not all-reduced
    dist.destroy_process_group()


def test_buckets_of_a_mask_two_rank_gloo():
    mp.spawn(_bucket_worker, args=(2, free_port()), nprocs=2, join=True)
