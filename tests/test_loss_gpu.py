"""compute_loss on CUDA tensors = the fused path (loss._FusedLoss, csrc/loss.cu): the objectness term over every cell
and the whole head cotangent come from two hand-written kernels that read the head tensors through their strides.
Checked against (1) the reference's own outputs (tests/golden/loss_golden.npz, generated from /root/reference by
tests/golden/make_golden.py section 9) and (2) the masked PyTorch formulation on the CPU, for contiguous inputs and for
permuted views of NCHW buffers (what Darknet.forward returns in training), nc = 1 and nc > 1, with and without targets."""
import os

import numpy as np
import pytest
import torch

from builders import fake_loss_model
from helpers import GOLDEN

pytestmark = pytest.mark.gpu


def _golden():
    g = np.load(os.path.join(GOLDEN, "loss_golden.npz"))
    hyp = {str(k): float(v) for k, v in zip(g["hyp_keys"], g["hyp_vals"])}
    return g, hyp


def _as_nchw_view(t):
    """[B, na, ny, nx, no] values stored as a contiguous NCHW [B, na*no, ny, nx] buffer, returned as the permuted view"""
    B, na, ny, nx, no = t.shape
    base = t.permute(0, 1, 4, 2, 3).contiguous().view(B, na * no, ny, nx)
    return base, base.view(B, na, no, ny, nx).permute(0, 1, 3, 4, 2)


@pytest.mark.parametrize("layout", ["contiguous", "nchw_view"])
def test_fused_loss_vs_reference_golden(layout):
    from rotate_yolov3_b200.loss import compute_loss
    g, hyp = _golden()
    dev = torch.device("cuda", 0)
    leaves, ps = [], []
    for k in range(3):
        t = torch.from_numpy(g["p%d" % k]).to(dev)
        if layout == "contiguous":
            leaf = t.clone().requires_grad_(True)
            leaves.append(leaf), ps.append(leaf)
        else:
            base, view = _as_nchw_view(t)
            base.requires_grad_(True)
            leaves.append(base)
            ps.append(base.view(t.shape[0], t.shape[1], t.shape[4], t.shape[2], t.shape[3]).permute(0, 1, 3, 4, 2))
    m = fake_loss_model([torch.from_numpy(g["p%d" % k]) for k in range(3)], hyp)
    loss, items = compute_loss(ps, torch.from_numpy(g["targets"]).to(dev), m, hyp)
    assert np.allclose(loss.detach().cpu().numpy(), g["loss"], rtol=1e-5, atol=1e-6)
    assert np.allclose(items.cpu().numpy(), g["items"], rtol=1e-5, atol=1e-6)
    (loss * 1.0).backward()
    for k in range(3):
        got = leaves[k].grad
        if layout == "nchw_view":
            assert got.is_contiguous()           # the cotangent arrives in the head buffer's own layout: no copy
            B, na, ny, nx, no = g["p%d" % k].shape
            got = got.view(B, na, no, ny, nx).permute(0, 1, 3, 4, 2)
        assert np.allclose(got.cpu().numpy(), g["dp%d" % k], rtol=1e-4, atol=1e-7), k


@pytest.mark.parametrize("nc,nt", [(1, 40), (3, 17), (1, 1), (1, 0)])
def test_fused_loss_equals_masked_cpu(nc, nt):
    from rotate_yolov3_b200 import loss as L
    g, hyp = _golden()
    dev = torch.device("cuda", 0)
    gen = torch.Generator().manual_seed(5 + nc + nt)
    shapes = [(2, 2, 4, 5, nc + 6), (2, 2, 8, 10, nc + 6), (2, 2, 16, 20, nc + 6)]
    base = [torch.randn(s, generator=gen) for s in shapes]
    t = torch.rand(nt, 7, generator=gen)
    if nt:
        t[:, 0] = torch.randint(0, 2, (nt,), generator=gen).float()
        t[:, 1] = torch.randint(0, nc, (nt,), generator=gen).float()
        t[:, 2:4] = t[:, 2:4] * 0.98 + 0.01
        t[:, 4:6] = t[:, 4:6] * 0.6 + 0.005
        t[:, 6] = (t[:, 6] - 0.5) * 3.0
        t[nt // 2] = t[0]
    m = fake_loss_model(base, hyp)
    m.nc = nc
    cpu = [b.clone().requires_grad_(True) for b in base]
    if nt:
        want, want_items = L._compute_loss_masked(cpu, t.clone(), m, hyp)
    else:
        want, want_items = L._compute_loss_no_targets(cpu, m)
    (want * 3.0).sum().backward()
    gpu_leaves = [b.to(dev).requires_grad_(True) for b in base]
    got, got_items = L.compute_loss(gpu_leaves, t.clone().to(dev), m, hyp)
    assert got.shape == want.shape
    assert np.allclose(got.detach().cpu().numpy(), want.detach().numpy(), rtol=2e-5, atol=1e-6)
    assert np.allclose(got_items.cpu().numpy(), want_items.numpy(), rtol=2e-5, atol=1e-6)
    (got * 3.0).sum().backward()
    for a, b in zip(gpu_leaves, cpu):
        assert np.allclose(a.grad.cpu().numpy(), b.grad.numpy(), rtol=1e-4, atol=1e-7)


def test_head_grad_nchw_to_padded_matches_layout():
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import layout as Lm
    lib, P = pkg._lib.lib, pkg._lib.ptr
    dev = torch.device("cuda", 0)
    # the last shape has more than 2048 image rows: several rows per block (the kernel keeps ~2k blocks in the grid)
    for (B, C, ny, nx) in ((2, 504, 19, 19), (3, 21, 5, 37), (1, 14, 8, 64), (30, 24, 80, 40)):
        g = torch.randn(B, C, ny, nx, device=dev)
        cs = Lm.round_up(C, 32)
        dst = torch.full((B, ny + 2, nx + 2, cs), 7.0, dtype=torch.bfloat16, device=dev)
        bias = torch.full((C,), 2.0, device=dev)
        pkg._lib.check(lib.ryolo_head_grad_nchw_to_padded(P(g), B, C, ny, nx, P(dst), cs, P(bias), pkg._lib.stream_ptr(dev)), "hg")
        want = g.permute(0, 2, 3, 1).to(torch.bfloat16)
        assert torch.equal(dst[:, 1:-1, 1:-1, :C], want)
        assert torch.allclose(bias - 2.0, g.sum((0, 2, 3)), rtol=1e-4, atol=1e-3)     # added to what was there
        assert bool((dst[:, 0] == 7.0).all()) and bool((dst[:, 1:-1, 1:-1, C:] == 7.0).all())


def test_fused_loss_under_no_grad_and_with_detached_heads():
    """test.py:96-98 evaluates compute_loss on the training-mode output under torch.no_grad(): same value, no graph"""
    from rotate_yolov3_b200.loss import compute_loss
    g, hyp = _golden()
    dev = torch.device("cuda", 0)
    ps = [torch.from_numpy(g["p%d" % k]).to(dev) for k in range(3)]
    m = fake_loss_model([torch.from_numpy(g["p%d" % k]) for k in range(3)], hyp)
    with torch.no_grad():
        loss, items = compute_loss(ps, torch.from_numpy(g["targets"]).to(dev), m, hyp)
    assert not loss.requires_grad
    assert np.allclose(loss.cpu().numpy(), g["loss"], rtol=1e-5, atol=1e-6)
    assert np.allclose(items.cpu().numpy(), g["items"], rtol=1e-5, atol=1e-6)
