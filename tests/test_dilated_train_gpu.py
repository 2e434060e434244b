"""Training the multi-branch dilated graph (cfg/yolov3-m.cfg) on the GPU in bf16, against the REFERENCE's own autograd
(tests/golden/darknet_m_golden.npz, make_golden_m.py: reference Darknet + compute_loss on the CPU in fp32, batch 2 at
160 x 128, arcs default and Fdefault), plus the repeatability of the step and the post-processing of the 16-head io.

What the graph adds to the training step: `weight_from` blocks (linear convs on another block's weight, whose own
Conv2d / BatchNorm2d the reference never uses: their gradients are None), dilated convs as ordinary convs on phase
images with ryolo_dilate_split / ryolo_dilate_merge as each other's adjoint, owners whose weight gradient sums their own
use and every branch use, a bias + PReLU conv without BatchNorm (block 109) and a 3x3 / stride-2 conv on an odd grid
(block 108: 5 x 4 -> 3 x 2 here).  The gradient bounds are the statistical ones of test_train_gpu.py /
test_se_train_gpu.py (bf16 activations through ~100 blocks against fp32)."""
import json

import numpy as np
import pytest
import torch

from builders import cosine, golden_text, m_golden, m_model
from helpers import init_darknet_weights

pytestmark = pytest.mark.gpu

HYP = {"giou": 0.1, "cls": 27.76, "cls_pw": 1.0, "obj": 20.35, "obj_pw": 1.0, "iou_t": 0.5, "ang_t": 3.1415926 / 12,
       "reg": 1.0, "context_factor": 1.0, "fl_gamma": 1.5}
TARGETS = [[0, 0, 0.30, 0.40, 57.5 / 160, 13.8 / 128, 0.5],
           [0, 0, 0.70, 0.60, 60.0 / 160, 14.5 / 128, -0.9],
           [1, 0, 0.50, 0.50, 55.0 / 160, 13.0 / 128, 1.2],
           [1, 0, 0.20, 0.80, 58.0 / 160, 14.0 / 128, -0.3]]


def _sample_idx(numel, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, numel, (n,), generator=g)


def _step(arc, seed_w, seed_x):
    from rotate_yolov3_b200.loss import compute_loss
    m = m_model(arc=arc)
    m.hyp, m.nc = HYP, 1                # train.py sets both before compute_loss
    init_darknet_weights(m, seed=seed_w)
    m = m.cuda().train()
    x = torch.rand(2, 3, 128, 160, generator=torch.Generator().manual_seed(seed_x)).cuda()
    ps = m(x)
    loss, items = compute_loss(ps, torch.tensor(TARGETS).cuda(), m, HYP)
    loss.backward()
    return m, ps, float(loss), items.detach().cpu().numpy()


@pytest.mark.parametrize("arc", ["default", "Fdefault"])
def test_training_step_vs_reference_autograd(arc):
    g = m_golden()
    sd = json.loads(golden_text(g, "seeds"))
    m, ps, loss, items = _step(arc, sd["train_w"], sd["train_x"])
    assert len(ps) == 16
    for k in (0, 4, 12):
        want = g["%s_p%d" % (arc, k)]
        got = ps[k].detach().reshape(-1)[_sample_idx(ps[k].numel(), len(want), 200 + k).cuda()].float().cpu().numpy()
        err, scale = np.abs(got - want), float(g["%s_p%d_absmax" % (arc, k)])
        assert err.max() <= 0.2 * scale and np.sqrt((err ** 2).mean()) <= 4e-2 * scale, (k, err.max(), scale)
    want_items = g[arc + "_items"]
    print("\n[%s] loss %.4f (reference %.4f), items %s / %s" % (arc, loss, float(g[arc + "_loss"]), items, want_items))
    assert abs(loss - float(g[arc + "_loss"])) <= 0.05 * abs(float(g[arc + "_loss"]))
    assert np.all(np.abs(items - want_items) <= 0.05 * np.abs(want_items) + 1e-3), (items, want_items)

    names = [n for n, _ in m.named_parameters()]
    assert names == [str(n) for n in g[arc + "_names"]]
    has = [p.grad is not None for _, p in m.named_parameters()]
    # None exactly where the reference has None: the weight_from blocks' own Conv2d / BatchNorm2d, the d-convs' BN
    assert has == [bool(h) for h in g[arc + "_has_grad"]]
    cos, ratio = {}, {}
    for j, (name, prm) in enumerate(m.named_parameters()):
        if prm.grad is None:
            continue
        want = g[arc + "_samples"][j].astype(np.float64)
        gflat = prm.grad.reshape(-1)
        got = gflat[_sample_idx(gflat.numel(), len(want), 1000 + j).cuda()].double().cpu().numpy()
        cos[name] = cosine(got, want)
        ratio[name] = float(gflat.double().norm()) / (float(g[arc + "_norms"][j]) + 1e-30)
    big = [n for n in cos if n.endswith("Conv2d.weight")]
    cb, rb = np.array([cos[n] for n in big]), np.array([ratio[n] for n in big])
    print("[%s] conv weights: cos min %.4f median %.4f, |ratio - 1| max %.4f median %.4f" % (
        arc, cb.min(), np.median(cb), np.abs(rb - 1).max(), np.median(np.abs(rb - 1))))
    assert cb.min() >= 0.65 and np.median(cb) >= 0.75
    assert np.all(np.abs(rb - 1) <= 0.15) and np.median(np.abs(rb - 1)) <= 0.02
    # the shared owners' gradients include every branch use: against the reference's sum, like any conv weight, and far
    # from what the owner's own use alone gives (the branches carry most of it)
    owners = sorted({int(d["weight_from"]) for d in m.module_defs if "weight_from" in d})
    assert owners == [75, 76, 77, 78, 79, 80, 81, 87, 88, 89, 90, 91, 92, 93, 99, 100, 101, 102, 103, 104, 105]
    for o in owners:
        n = "module_list.%d.Conv2d.weight" % o
        assert abs(ratio[n] - 1) <= 0.15 and cos[n] >= 0.65, (n, ratio[n], cos[n])
    small = [n for n in cos if not n.endswith("Conv2d.weight") and not n.endswith("activation.weight")]
    cs, rs = np.array([cos[n] for n in small]), np.array([ratio[n] for n in small])
    assert np.median(cs) >= 0.75 and np.all(np.abs(rs - 1) <= 1.0) and np.median(np.abs(rs - 1)) <= 0.05
    # the bias + PReLU conv without BatchNorm: its bias gradient (d-beta of bn_act_bwd) like a conv weight's; its slope
    # gradient, one sum over every pixel with heavy cancellation (the other blocks' slopes reach ratios of 2 against
    # fp32 and are not bounded), with the per-vector bound of the BN / bias vectors above
    assert abs(ratio["module_list.109.Conv2d.bias"] - 1) <= 0.15, ratio["module_list.109.Conv2d.bias"]
    assert abs(ratio["module_list.109.activation.weight"] - 1) <= 1.0, ratio["module_list.109.activation.weight"]


def _grads(m):
    return [p.grad.clone() if p.grad is not None else None for p in m.parameters()]


def test_training_step_is_bitwise_repeatable():
    m, _, l1, _ = _step("default", 31, 32)
    g1 = _grads(m)
    from rotate_yolov3_b200.loss import compute_loss
    m.zero_grad(set_to_none=True)
    x = torch.rand(2, 3, 128, 160, generator=torch.Generator().manual_seed(32)).cuda()
    # the BN running statistics moved in the first step; they do not enter a training forward
    ps = m(x)
    loss, _ = compute_loss(ps, torch.tensor(TARGETS).cuda(), m, HYP)
    loss.backward()
    assert float(loss) == l1
    for (name, _), a, b in zip(m.named_parameters(), g1, _grads(m)):
        assert (a is None) == (b is None), name
        if a is not None:
            assert torch.equal(a.view(-1).view(torch.int32), b.view(-1).view(torch.int32)), name


def test_cuda_graph_training_step_equals_eager():
    m, _, _, _ = _step("default", 41, 42)
    eager = _grads(m)
    from rotate_yolov3_b200.loss import compute_loss
    m.use_cuda_graph = True
    x = torch.rand(2, 3, 128, 160, generator=torch.Generator().manual_seed(42)).cuda()
    for _ in range(3):                   # capture, then replays
        m.zero_grad(set_to_none=True)
        ps = m(x)
        loss, _ = compute_loss(ps, torch.tensor(TARGETS).cuda(), m, HYP)
        loss.backward()
        for (name, _), a, b in zip(m.named_parameters(), eager, _grads(m)):
            assert (a is None) == (b is None), name
            if a is not None:
                assert torch.equal(a, b), name


def test_detect_postprocess_on_the_16_head_io():
    """detect_postprocess on yolov3-m's io (16 heads, 72 anchors each) == the per-image pipeline, bit for bit"""
    import helpers
    m = init_darknet_weights(m_model(), seed=51).cuda().eval()
    x = torch.rand(2, 3, 416, 416, generator=torch.Generator().manual_seed(52)).cuda()
    with torch.no_grad():
        io, _ = m(x)
    assert io.shape == (2, 1646208, 7)
    helpers.check_postprocess_equals_per_image(io.contiguous(), 0.5, 0.4, 4000, 2.0)
