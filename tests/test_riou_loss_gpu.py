"""Rotated-IoU loss (SURVEY.md 8f item 4): value vs the float64 convex-clip oracle (1e-4 relative, the north_star IoU
tolerance) and analytic gradient vs central differences of that float64 oracle -- the extension has no reference
counterpart (model/loss.py never calls a rotated IoU, SURVEY D1), so the oracle is the only checker."""
import ctypes

import numpy as np
import pytest
import torch

import helpers
from builders import overlapping_pairs

pytestmark = pytest.mark.gpu
DP = ctypes.POINTER(ctypes.c_double)


def _oracle_iou(a, b):
    orc = helpers.oracle()
    a = np.ascontiguousarray(a, dtype=np.float64)
    b = np.ascontiguousarray(b, dtype=np.float64)
    return orc.orc_skew_iou(a.ctypes.data_as(DP), b.ctypes.data_as(DP), 0)


def test_value_and_gradient_vs_float64_oracle():
    from rotate_yolov3_b200.iou import riou_loss, rotated_iou
    n = 400
    a, b = overlapping_pairs(n, 3)
    # fp32-representable inputs on both sides
    ad = a.cuda().requires_grad_(True)
    bd = b.cuda().requires_grad_(True)
    iou = rotated_iou(ad, bd)
    want = np.array([_oracle_iou(a[i].numpy(), b[i].numpy()) for i in range(n)])
    got = iou.detach().cpu().numpy()
    assert np.all(np.abs(got - want) <= 1e-4 * np.abs(want) + 1e-6), np.abs(got - want).max()
    assert (want > 0.05).mean() > 0.8                       # the set actually overlaps
    w = torch.linspace(0.5, 1.5, n).cuda()
    (iou * w).sum().backward()
    ga, gb = ad.grad.cpu().numpy(), bd.grad.cpu().numpy()
    worst = 0.0
    for i in range(0, n, 4):
        for which, base, grad in (("a", a, ga), ("b", b, gb)):
            num = np.zeros(5)
            for k in range(5):
                h = 1e-4 * (1.0 if k == 4 else 10.0)
                p = base[i].numpy().astype(np.float64).copy()
                m = p.copy()
                p[k] += h
                m[k] -= h
                other = (b if which == "a" else a)[i].numpy().astype(np.float64)
                fp = _oracle_iou(p, other) if which == "a" else _oracle_iou(other, p)
                fm = _oracle_iou(m, other) if which == "a" else _oracle_iou(other, m)
                num[k] = (fp - fm) / (2 * h) * float(w[i])
            scale = np.abs(num).max() + 1e-6
            err = np.abs(grad[i] - num).max() / scale
            worst = max(worst, err)
            # kinks (a corner of one box crossing an edge of the other inside the finite-difference stencil) are rare but exist
            assert err <= 5e-2, (i, which, grad[i], num)
    print("riou gradient: worst error / max component = %.2e" % worst)
    assert worst <= 5e-2
    # loss wrapper and degenerate inputs: zero-area and disjoint boxes give IoU 0 and zero gradients, never NaN
    z = a.clone().cuda()
    z[:5, 2] = 0.0
    far = b.clone().cuda()
    far[5:10, 0] += 1e4
    zz = z.requires_grad_(True)
    loss = riou_loss(zz, far)
    loss.backward()
    assert torch.isfinite(loss) and torch.isfinite(zz.grad).all()
    assert float(zz.grad[:10].abs().max()) == 0.0


def test_gradient_descent_on_riou_loss_aligns_boxes():
    from rotate_yolov3_b200.iou import riou_loss
    a, b = overlapping_pairs(64, 9)
    pred = a.cuda().clone().requires_grad_(True)
    target = b.cuda()
    opt = torch.optim.Adam([pred], lr=0.05)          # scale-free steps: pixels and radians have very different gradients
    first = None
    for _ in range(300):
        opt.zero_grad()
        loss = riou_loss(pred, target)
        if first is None:
            first = float(loss)
        loss.backward()
        opt.step()
    assert float(loss) < 0.6 * first, (first, float(loss))


def test_axis_aligned_boxes_with_collinear_edges_have_the_right_value():
    """boxes whose edges lie ON each other's edges (axis-aligned, equal height / same centre line: what detection labels are
    full of): the value must be the true IoU.  An edge-clipping evaluation counts such a shared run twice; the kernel takes the
    value from the clamp integral instead."""
    from rotate_yolov3_b200.iou import rotated_iou
    a = torch.tensor([[100.0, 100.0, 40.0, 20.0, 0.0], [100.0, 100.0, 40.0, 20.0, 0.0], [50.0, 60.0, 30.0, 30.0, 0.0],
                      [100.0, 100.0, 40.0, 20.0, np.pi / 2], [10.0, 10.0, 8.0, 4.0, 0.0]])
    b = torch.tensor([[120.0, 100.0, 40.0, 20.0, 0.0], [100.0, 100.0, 40.0, 20.0, 0.0], [65.0, 60.0, 30.0, 30.0, 0.0],
                      [100.0, 120.0, 40.0, 20.0, np.pi / 2], [10.0, 12.0, 8.0, 4.0, 0.0]])
    want = np.array([_oracle_iou(a[i].numpy(), b[i].numpy()) for i in range(len(a))])
    assert abs(want[0] - 1.0 / 3.0) < 1e-9 and abs(want[1] - 1.0) < 1e-9
    ad, bd = a.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
    iou = rotated_iou(ad, bd)
    got = iou.detach().cpu().numpy()
    assert np.all(np.abs(got - want) <= 1e-4 * np.abs(want) + 1e-6), (got, want)
    iou.sum().backward()
    assert torch.isfinite(ad.grad).all() and torch.isfinite(bd.grad).all()
