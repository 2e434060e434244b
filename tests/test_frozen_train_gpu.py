"""Training with frozen parameters on the GPU: a step under a trainable mask gives the trainable parameters the same bits
as the step with every parameter trainable, the frozen ones no gradient at all, and runs none of the launches whose
results only frozen parameters would use.  Masks: the reference's --prebias (head biases), --transfer (head convs) and
frozen backbone (blocks >= 75 train) of train.py:120-135 / :215-220, one SE's fc weights, one yolov3-m owner weight.
BatchNorm momentum is 0, so that every forward is the same and the running statistics do not move."""
import math
import os

import pytest
import torch

import helpers
from builders import free_port, transfer_mask
from helpers import GOLDEN, SMALL_ANCHORS

pytestmark = pytest.mark.gpu
REF = os.path.join(GOLDEN, "reference_cfg")


def _prep(m, seed):
    helpers.init_darknet_weights(m, seed=seed)
    m = m.cuda().train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.momentum = 0.0
    return m


def yolov3(width=160, height=128):
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import cfgs
    text = cfgs.yolov3_cfg(width=width, height=height, classes=1, anchors=SMALL_ANCHORS, n_anchors=6)
    return _prep(pkg.Darknet(text, {"context_factor": 1.0}, arc="default"), 321)


def se_model():
    import rotate_yolov3_b200 as pkg
    old = os.getcwd()
    os.chdir(REF)                   # the SE cfg names its anchor file relative to the reference root
    try:
        m = pkg.Darknet("cfg/HRSC+/yolov3_512_se.cfg", {"context_factor": 1.0}, arc="default")
    finally:
        os.chdir(old)
    return _prep(m, 5)


def m_graph():
    from builders import m_model
    return _prep(m_model(), 7)


def prebias(m):
    nf = int(m.module_defs[m.yolo_layers[0] - 1]["filters"])
    return [p.numel() == nf for p in m.parameters()]          # train.py:129-130


def cutoff75(m):
    return [int(n.split(".")[1]) >= 75 for n, _ in m.named_parameters()]     # train.py:218-220


def only(names):
    return lambda m: [n in names for n, _ in m.named_parameters()]


def _set(m, mask):
    for p, t in zip(m.parameters(), mask):
        p.requires_grad_(bool(t))
        p.grad = None


def _step(m, x, gs, mask):
    """one forward + backward under `mask`: (gradients by name, head outputs, running statistics)"""
    _set(m, mask)
    ps = m(x)
    sum((p * g).sum() for p, g in zip(ps, gs)).backward()
    grads = {n: (p.grad.clone() if p.grad is not None else None) for n, p in m.named_parameters()}
    return grads, [p.detach().clone() for p in ps], [b.clone() for n, b in m.named_buffers()
                                                     if not n.endswith("num_batches_tracked")]


def _cotangents(m, x):
    with torch.no_grad():
        _set(m, [True] * len(list(m.parameters())))
        ps = m(x)
    g = torch.Generator(device="cuda").manual_seed(9)
    return [torch.randn(p.shape, device="cuda", generator=g) / math.sqrt(p.numel()) for p in ps]


def _check_mask(m, x, mask_fn):
    gs = _cotangents(m, x)
    full = _step(m, x, gs, [True] * len(list(m.parameters())))
    mask = mask_fn(m)
    assert any(mask) and not all(mask)
    got = _step(m, x, gs, mask)
    for (n, p), t in zip(m.named_parameters(), mask):
        if not t:
            assert got[0][n] is None, n
        elif full[0][n] is None:                 # a weight_from block's own, unused modules
            assert got[0][n] is None, n
        else:
            assert torch.equal(got[0][n], full[0][n]), n
    for a, b in zip(got[1], full[1]):
        assert torch.equal(a, b)
    for a, b in zip(got[2], full[2]):
        assert torch.equal(a, b)
    return m._tplan.sched


@pytest.mark.parametrize("mask", ["prebias", "transfer", "cutoff75"])
def test_masked_step_equals_the_full_step(mask):
    m = yolov3()
    x = torch.rand(2, 3, 128, 160, generator=torch.Generator().manual_seed(1)).cuda()
    sch = _check_mask(m, x, {"prebias": prebias, "transfer": transfer_mask, "cutoff75": cutoff75}[mask])
    kinds = {k for k, _, _ in sch.ops(m._tplan)}
    assert kinds == {"prebias": {"head_bias"}, "transfer": {"head", "wgrad"},
                     "cutoff75": {"head", "bnact", "wgrad", "dgrad"}}[mask]


def test_masked_step_at_608():
    m = yolov3(608, 608)
    x = torch.rand(2, 3, 608, 608, generator=torch.Generator().manual_seed(2)).cuda()
    _check_mask(m, x, cutoff75)


def test_se_fc_only():
    m = se_model()
    se = [i for i, d in enumerate(m.module_defs) if d["type"] == "se"][3]
    x = torch.rand(2, 3, 128, 160, generator=torch.Generator().manual_seed(3)).cuda()
    sch = _check_mask(m, x, only({"module_list.%d.fc.0.weight" % se, "module_list.%d.fc.2.weight" % se}))
    ops = sch.ops(m._tplan)
    assert ("se", se, True) in ops or ("se", se, False) in ops
    assert not any(k in ("wgrad", "head_bias") for k, _, _ in ops)


def test_yolov3m_owner_weight_only():
    m = m_graph()
    owners = sorted({int(d["weight_from"]) for d in m.module_defs if "weight_from" in d})
    x = torch.rand(2, 3, 128, 160, generator=torch.Generator().manual_seed(4)).cuda()
    sch = _check_mask(m, x, only({"module_list.%d.Conv2d.weight" % owners[0]}))
    users = [i for i, d in enumerate(m.module_defs) if "weight_from" in d and int(d["weight_from"]) == owners[0]]
    wg = [i for k, i, _ in sch.ops(m._tplan) if k == "wgrad"]
    assert sorted(wg) == sorted(users + [owners[0]])


def test_prebias_backward_launches_only_the_bias_reductions():
    """the loss here is plain PyTorch (no library kernels), so the launch-count delta over backward is the plan's alone:
    per head the bias-only reduction and its ordered row sum, nothing else"""
    import rotate_yolov3_b200 as pkg
    m = yolov3()
    x = torch.rand(2, 3, 128, 160).cuda()
    _set(m, prebias(m))
    ps = m(x)
    loss = sum((p * p).mean() for p in ps)
    torch.cuda.synchronize()
    c0 = pkg._lib.lib.ryolo_launch_count()
    loss.backward()
    torch.cuda.synchronize()
    assert pkg._lib.lib.ryolo_launch_count() - c0 == 2 * len(m.yolo_layers)
    assert sum(p.grad is not None for p in m.parameters()) == len(m.yolo_layers)


@pytest.mark.parametrize("n", [19, 38, 76])
def test_head_bias_grad_equals_the_sums_of_the_full_conversion(n):
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import layout as L
    lib, P, st = pkg._lib.lib, pkg._lib.ptr, pkg._lib.stream_ptr()
    b, c = 64, 504
    g = torch.randn(b, c, n, n, generator=torch.Generator(device="cuda").manual_seed(n), device="cuda")
    dst = L.alloc_padded(b, n, n, 512, torch.device("cuda"))
    want, got = torch.full((c,), 0.5, device="cuda"), torch.full((c,), 0.5, device="cuda")
    pkg._lib.check(lib.ryolo_head_grad_nchw_to_padded(P(g), b, c, n, n, P(dst), 512, P(want), st), "hg")
    pkg._lib.check(lib.ryolo_head_bias_grad(P(g), b, c, n, n, P(got), st), "hb")
    assert torch.equal(got, want)                      # both ADD to the output
    assert torch.allclose(got.double() - 0.5, g.double().sum((0, 2, 3)), rtol=1e-4, atol=2e-2)
    assert lib.ryolo_head_bias_grad(P(g), b, c, n, n, None, st) != 0


def test_cuda_graph_mask_switch_equals_eager():
    """frozen backbone at epoch 0, unfrozen at epoch 1 (train.py:215-220): the switch re-captures the graphs"""
    m = yolov3()
    x = torch.rand(2, 3, 128, 160, generator=torch.Generator().manual_seed(5)).cuda()
    gs = _cotangents(m, x)
    full_mask, frozen = [True] * len(list(m.parameters())), cutoff75(m)
    eager = {k: _step(m, x, gs, mk)[0] for k, mk in (("frozen", frozen), ("full", full_mask))}
    m.use_cuda_graph = True
    for k, mk in (("frozen", frozen), ("frozen", frozen), ("frozen", frozen), ("full", full_mask), ("full", full_mask),
                  ("full", full_mask)):
        got = _step(m, x, gs, mk)[0]
        for n in got:
            assert (got[n] is None) == (eager[k][n] is None), (k, n)
            assert got[n] is None or torch.equal(got[n], eager[k][n]), (k, n)
    assert m._tplan.replayed_kernels > 0


def test_reference_prebias_and_transfer_loops(tmp_path):
    """train.py:120-135 then the inner loop train.py:268-287, through the reference's import line"""
    from rotate_yolov3_b200 import dropin
    dropin.install()
    from model.models import Darknet
    from rotate_yolov3_b200.loss import compute_loss
    hyp = {"giou": 0.1, "cls": 27.76, "cls_pw": 1.0, "obj": 20.35, "obj_pw": 1.0, "iou_t": 0.5, "ang_t": math.pi / 12,
           "reg": 1.0, "context_factor": 1.0}
    imgs = torch.rand(4, 3, 48, 64).cuda()
    targets = torch.tensor([[0, 0, 0.5, 0.5, 0.4, 0.1, 0.3], [2, 0, 0.3, 0.6, 0.5, 0.12, -0.7]]).cuda()
    for opt_prebias, opt_transfer in ((True, False), (False, True)):
        model = Darknet(helpers.mini_cfg(64, 48), {"context_factor": 1.0}, arc="default")
        helpers.init_darknet_weights(model, seed=11)
        model = model.cuda().train()
        model.nc, model.hyp, model.arc = 1, hyp, "default"
        pg0, pg1 = [], []
        for k, v in dict(model.named_parameters()).items():
            (pg1 if "Conv2d.weight" in k else pg0).append(v)
        optimizer = torch.optim.SGD(pg0, lr=1e-3, momentum=0.9, nesterov=True)
        optimizer.add_param_group({"params": pg1, "weight_decay": 5e-4})
        nf = int(model.module_defs[model.yolo_layers[0] - 1]["filters"])
        for p in model.parameters():
            if opt_prebias and p.numel() == nf:
                p.requires_grad = True
            elif opt_transfer and p.shape[0] == nf:
                p.requires_grad = True
            else:
                p.requires_grad = False
        before = {n: p.detach().clone() for n, p in model.named_parameters()}
        for i in range(4):
            pred = model(imgs)
            loss, loss_items = compute_loss(pred, targets.clone(), model, hyp)
            assert torch.isfinite(loss).all()
            loss.backward()
            optimizer.step()
            optimizer.zero_grad()
        for n, p in model.named_parameters():
            assert torch.equal(p.detach(), before[n]) != p.requires_grad, n


def _ddp_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    import torch.distributed as dist
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import parallel

    def make():
        m = pkg.Darknet(helpers.mini_cfg(64, 48), {"context_factor": 1.0})
        m = _prep(m, 5)
        _set(m, transfer_mask(m))
        return m
    x = torch.rand(4, 3, 48, 64, generator=torch.Generator().manual_seed(100 + rank)).cuda()
    m = make()
    sum(p.float().pow(2).mean() for p in m(x)).backward()
    want = torch.cat([p.grad.reshape(-1) for p in m.parameters() if p.requires_grad])
    dist.all_reduce(want)
    want /= world
    m2 = make()
    ddp = parallel.DistributedDataParallel(m2, bucket_mb=0)
    m2._ddp["bucket_bytes"] = 1 << 10
    sum(p.float().pow(2).mean() for p in ddp(x)).backward()
    got = torch.cat([p.grad.reshape(-1) for p in m2.parameters() if p.requires_grad])
    frozen_none = all(p.grad is None for p in m2.parameters() if not p.requires_grad)
    sch = m2._tplan.sched
    inside = all(any(a <= lo and hi <= b for a, b in sch.ranges) for lo, hi in sch.buckets.buckets)
    q.put((rank, float((got - want).abs().max() / want.abs().max()), frozen_none, inside))
    dist.destroy_process_group()


def test_two_rank_nccl_transfer_mask():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_ddp_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    for rank, err, frozen_none, inside in sorted(q.get() for _ in range(2)):
        assert frozen_none and inside
        assert err <= 2e-2, (rank, err)
