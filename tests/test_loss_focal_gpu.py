"""Focal arcs of compute_loss on CUDA tensors: the fused path (loss._FusedLoss) with the focal instantiations of the
objectness kernels (csrc/loss.cu, ryolo_obj_focal_fwd / _bwd) and the focal matched-row terms.

  * against the reference's own compute_loss (tests/golden/loss_focal_golden.npz, cases a-c) for contiguous heads and
    for permuted views of NCHW buffers, and against the masked CPU form for nc in {1, 3};
  * the kernels against float64 of their own inputs at the batch-64 608 x 608 heads, logits out to +-40;
  * bitwise repeatability, and gamma = 0 == the BCE kernels bit for bit;
  * the Darknet-53 graph at 160 x 128 in parity precision trained with the Fdefault loss against the reference (case d);
  * a bf16 training step with Fdefault under CUDA graphs is bitwise repeatable."""
import ctypes

import numpy as np
import pytest
import torch

import focal_cases as FC
from builders import (STEP_HYP, assert_same, fake_loss_model, repeat, report_and_check_gradients, small_train_model,
                      step_targets)
from helpers import SMALL_ANCHORS, init_darknet_weights

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


def _nchw_leaf(t):
    """[B, na, ny, nx, no] values stored as a contiguous NCHW [B, na*no, ny, nx] leaf, and the permuted view of it"""
    B, na, ny, nx, no = t.shape
    base = t.permute(0, 1, 4, 2, 3).contiguous().view(B, na * no, ny, nx).requires_grad_(True)
    return base, base.view(B, na, no, ny, nx).permute(0, 1, 3, 4, 2)


def _fmodel(heads, hyp, nc=1):
    m = fake_loss_model(heads, hyp)
    m.arc, m.nc = "Fdefault", nc
    return m


@pytest.mark.parametrize("layout", ["contiguous", "nchw_view"])
@pytest.mark.parametrize("case", range(6))
def test_fused_focal_loss_vs_reference_golden(case, layout):
    from rotate_yolov3_b200.loss import compute_loss
    g = FC.golden()
    tag, heads, tg, hyp = FC.cases()[case]
    leaves, ps = [], []
    for h in heads:
        if layout == "contiguous":
            leaf = h.cuda().requires_grad_(True)
            leaves.append(leaf), ps.append(leaf)
        else:
            leaf, view = _nchw_leaf(h.cuda())
            leaves.append(leaf), ps.append(view)
    loss, items = compute_loss(ps, tg.cuda(), _fmodel(heads, hyp), hyp)
    assert np.allclose(loss.detach().cpu().numpy(), g[tag + "_loss"], rtol=1e-5, atol=1e-6), tag
    assert np.allclose(items.cpu().numpy(), g[tag + "_items"], rtol=1e-5, atol=1e-6), tag
    loss.backward()
    for k, h in enumerate(heads):
        got = leaves[k].grad
        if layout == "nchw_view":
            assert got.is_contiguous()           # the cotangent arrives in the head buffer's own layout
            B, na, ny, nx, no = h.shape
            got = got.view(B, na, no, ny, nx).permute(0, 1, 3, 4, 2)
        assert np.allclose(got.cpu().numpy(), g[tag + "_dp%d" % k], rtol=1e-4, atol=1e-7), (tag, k)


@pytest.mark.parametrize("gamma", FC.GAMMAS)
@pytest.mark.parametrize("nt", [40, 17, 1, 0])
@pytest.mark.parametrize("nc", [1, 3])
def test_fused_focal_loss_equals_masked_cpu(nc, nt, gamma):
    from rotate_yolov3_b200 import loss as L
    _, _, hyp0 = FC.base_inputs()
    hyp = FC.focal_hyp(hyp0, gamma, 1.6)
    gen = torch.Generator().manual_seed(7 + nc + nt)
    shapes = [(2, 2, 4, 5, nc + 6), (2, 2, 8, 10, nc + 6), (2, 2, 16, 20, nc + 6)]
    base = [torch.randn(s, generator=gen) * 2.0 for s in shapes]
    t = torch.rand(nt, 7, generator=gen)
    if nt:
        t[:, 0] = torch.randint(0, 2, (nt,), generator=gen).float()
        t[:, 1] = torch.randint(0, nc, (nt,), generator=gen).float()
        t[:, 2:4] = t[:, 2:4] * 0.98 + 0.01
        t[:, 4:6] = t[:, 4:6] * 0.6 + 0.005
        t[:, 6] = (t[:, 6] - 0.5) * 3.0
        t[nt // 2] = t[0]
    m = _fmodel(base, hyp, nc)
    cpu = [b.clone().requires_grad_(True) for b in base]
    if nt:
        want, want_items = L._compute_loss_masked(cpu, t.clone(), m, hyp)
    else:
        want, want_items = L._compute_loss_no_targets(cpu, m)
    (want * 3.0).sum().backward()
    gpu = [b.cuda().requires_grad_(True) for b in base]
    got, got_items = L.compute_loss(gpu, t.clone().cuda(), m, hyp)
    assert got.shape == want.shape
    assert np.allclose(got.detach().cpu().numpy(), want.detach().numpy(), rtol=2e-5, atol=1e-6)
    assert np.allclose(got_items.cpu().numpy(), want_items.numpy(), rtol=2e-5, atol=1e-6)
    if nt:
        assert float(got_items[2]) > 0 and (nc == 1 or float(got_items[1]) > 0)
    (got * 3.0).sum().backward()
    for a, b in zip(gpu, cpu):
        assert np.allclose(a.grad.cpu().numpy(), b.grad.numpy(), rtol=1e-4, atol=1e-7)


# ---------------------------------------------------------------------------------------------------------------
# the kernels against float64 of their own inputs at the training shapes
NA, NO, B64 = 72, 7, 64


def _head608(ny, seed):
    """NCHW [64, 72 * 7, ny, ny] buffer as the [64, 72, ny, ny, 7] view Darknet returns; logits uniform in [-40, 40]
    with one cell in eight exactly 0, 5 % positive cells"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = (torch.rand(B64, NA * NO, ny, ny, generator=g, device="cuda") * 2.0 - 1.0) * FC.EXTREME
    buf[torch.rand(buf.shape, generator=g, device="cuda") < 0.125] = 0.0
    x = buf.view(B64, NA, NO, ny, ny).permute(0, 1, 3, 4, 2)
    tobj = (torch.rand(B64, NA, ny, ny, generator=g, device="cuda") < 0.05).float()
    return x, tobj


def _kernel_call(x, tobj, pw, gamma, scale, focal=True):
    import rotate_yolov3_b200 as pkg
    L = pkg._lib
    B, na, ny, nx, no = x.shape
    strides = (ctypes.c_longlong * 5)(*x.stride())
    s = torch.zeros(1, dtype=torch.float64, device="cuda")
    g = torch.empty_strided(x.shape, x.stride(), dtype=torch.float32, device="cuda")
    sc = torch.full((1,), scale, device="cuda")
    st = L.stream_ptr()
    if focal:
        L.check(L.lib.ryolo_obj_focal_fwd(L.ptr(x), strides, B, na, ny, nx, no, 5, L.ptr(tobj), pw, gamma, L.ptr(s), st), "f")
        L.check(L.lib.ryolo_obj_focal_bwd(L.ptr(x), strides, B, na, ny, nx, no, 5, L.ptr(tobj), pw, gamma, L.ptr(sc),
                                          L.ptr(g), st), "b")
    else:
        L.check(L.lib.ryolo_obj_bce_fwd(L.ptr(x), strides, B, na, ny, nx, no, 5, L.ptr(tobj), pw, L.ptr(s), st), "f")
        L.check(L.lib.ryolo_obj_bce_bwd(L.ptr(x), strides, B, na, ny, nx, no, 5, L.ptr(tobj), pw, L.ptr(sc), L.ptr(g), st), "b")
    return s, g


def focal_f64_and_bounds(x, t, pw, gamma, scale):
    """float64 value of the focal objectness terms of the fp32 inputs x (logits), t (targets), and bounds on the fp32
    evaluation.  u = 2^-24; per cell, with lw = 1 + (pw - 1) t:

      l = (1 - t) x + lw (log1p(exp(-|x|)) + max(-x, 0)),   |l~ - l| <= dl = 8 u m_l,
          m_l = |(1 - t) x| + lw (log1p(exp(-|x|)) + max(-x, 0))   (the magnitudes of the terms of l; expf / log1pf
          within 2 ulp, a handful of roundings; the same per-cell bound as the BCE sum in test_determinism_gpu)
      b(l) = 2^-20 + 1 - exp(-l)  (increasing, >= 2^-20),   lf = l b^g,
      F(l) = dlf/dl = b^g + g l e^-l b^(g-1)  <=  (1 + g) b^g   because l e^-l <= 1 - e^-l <= b,
    so over [l - dl, l + dl] the error carried from l is at most dl (1 + g) b(l + dl)^g.  The rest is rounding of
    expm1f (1 ulp), the subtraction, powf (<= 4 ulp, relative error of the base times g) and the product:
      |lf~ - lf| <= dl (1 + g) b(l + dl)^g + 8 u (1 + g) lf.
    The forward sum adds these in double: its bound is the sum of the per-cell bounds plus n 2^-53 sum(lf).

    Cotangent: d = s dl/dx F(l), dl/dx = (1 - t) + lw (sigmoid(x) - 1).  dl/dx is within 4 u m_g of its value,
    m_g = (1 - t) + lw (sigmoid(x) + 1) (its terms: sigmoid(x) - 1 cancels for large x).  F carries the error of l
    through |F'(l)| <= g e^-l b^(g-1) (2 + l + |g - 1|) (the same l e^-l <= b), evaluated at the worst end of
    [l - dl, l + dl] (e^-l and, for g < 1, b^(g-1) at the low end; b^(g-1) at the high end for g >= 1), and its own
    roundings (powf, expf, the division b^g / b, three products, one add) within 16 u (1 + g) F.  With dF the sum:
      |d~ - d| <= s (4 u m_g (F + dF) + |dl/dx| dF + 2 u |dl/dx| F)."""
    x, t = x.double(), t.double()
    lw = 1.0 + (pw - 1.0) * t
    sp = torch.log1p(torch.exp(-x.abs())) + (-x).clamp(min=0)
    l = (1.0 - t) * x + lw * sp
    m_l = ((1.0 - t) * x).abs() + lw * sp
    dl = 8 * U * m_l
    eps = 2.0 ** -20

    def b(v):
        return eps - torch.expm1(-v.clamp(min=0.0))
    bl = b(l)
    lf = l * bl ** gamma
    F = bl ** gamma + gamma * l * torch.exp(-l) * bl ** (gamma - 1)
    lo, hi = (l - dl).clamp(min=0.0), l + dl
    cell_f = dl * (1 + gamma) * b(hi) ** gamma + 8 * U * (1 + gamma) * lf
    sg = torch.sigmoid(x)
    dldx = (1.0 - t) + lw * (sg - 1.0)
    m_g = (1.0 - t) + lw * (sg + 1.0)
    bpow = b(lo) ** (gamma - 1) if gamma < 1 else b(hi) ** (gamma - 1)
    dF = dl * gamma * torch.exp(-lo) * bpow * (2.0 + hi + abs(gamma - 1.0)) + 16 * U * (1 + gamma) * F
    cell_b = scale * (4 * U * m_g * (F + dF) + dldx.abs() * dF + 2 * U * dldx.abs() * F)
    return lf, cell_f, scale * dldx * F, cell_b


@pytest.mark.parametrize("gamma", FC.GAMMAS)
@pytest.mark.parametrize("ny", [19, 38, 76])
def test_focal_kernels_vs_float64_at_608(ny, gamma):
    pw, scale = 1.7, 20.35 / (B64 * NA * ny * ny)
    x, tobj = _head608(ny, 100 + ny)
    s, g = _kernel_call(x, tobj, pw, gamma, scale)
    xo = x[..., 5]
    lf, cell_f, d64, cell_b = focal_f64_and_bounds(xo, tobj, pw, gamma, scale)
    n = lf.numel()
    want = float(lf.sum())
    bound = float(cell_f.sum()) + n * 2.0 ** -53 * float(lf.abs().sum())
    err = abs(float(s) - want)
    print("[focal %d g=%g] sum %.6e |err| %.3e bound %.3e" % (ny, gamma, want, err, bound))
    assert err <= bound, (err, bound)
    ratio = ((g[..., 5].double() - d64).abs() / (cell_b + 1e-300)).max()
    print("[focal %d g=%g] cotangent: worst |err| / bound %.3e" % (ny, gamma, float(ratio)))
    assert float(ratio) <= 1.0
    others = torch.cat([g[..., :5], g[..., 6:]], -1)
    assert bool((others == 0).all()) and not bool(torch.signbit(others).any())     # exactly +0


@pytest.mark.parametrize("ny", [19, 38, 76])
def test_focal_kernels_repeatable_and_gamma0_is_bce(ny):
    x, tobj = _head608(ny, 200 + ny)
    scale = 20.35 / (B64 * NA * ny * ny)
    s, g = repeat(lambda: _kernel_call(x, tobj, 1.0, 0.5, scale))
    assert torch.isfinite(s).all() and bool(torch.isfinite(g).all())
    s0, g0 = _kernel_call(x, tobj, 1.7, 0.0, scale)
    sb, gb = _kernel_call(x, tobj, 1.7, 0.0, scale, focal=False)
    torch.cuda.synchronize()
    assert torch.equal(s0, sb) and torch.equal(g0, gb)


def test_focal_kernels_reject_bad_gamma():
    import rotate_yolov3_b200 as pkg
    L = pkg._lib
    x, tobj = torch.zeros(1, 1, 2, 2, 7, device="cuda"), torch.zeros(1, 1, 2, 2, device="cuda")
    strides = (ctypes.c_longlong * 5)(*x.stride())
    s = torch.zeros(1, dtype=torch.float64, device="cuda")
    for gm in (-0.5, float("nan"), float("inf")):
        assert L.lib.ryolo_obj_focal_fwd(L.ptr(x), strides, 1, 1, 2, 2, 7, 5, L.ptr(tobj), 1.0, gm, L.ptr(s), L.stream_ptr()) != 0


# ---------------------------------------------------------------------------------------------------------------
def test_darknet53_parity_trained_with_fdefault_vs_reference():
    """case (d): parity precision, Fdefault loss, against the reference's autograd of the same graph and loss"""
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import cfgs
    from rotate_yolov3_b200.loss import compute_loss
    g = FC.golden()
    x, tg, hyp = FC.darknet_case()
    m = pkg.Darknet(cfgs.yolov3_cfg(width=160, height=128, classes=1, anchors=SMALL_ANCHORS, n_anchors=6),
                    {"context_factor": 1.0}, arc="Fdefault", precision="parity")
    init_darknet_weights(m, seed=321)
    m = m.cuda().train()
    m.hyp, m.nc = hyp, 1
    ps = m(x.cuda())
    loss, items = compute_loss(ps, tg.cuda(), m, hyp)
    assert abs(float(loss) - float(g["d_loss"][0])) <= 1e-4 * abs(float(g["d_loss"][0])), (float(loss), g["d_loss"])
    assert np.allclose(items.cpu().numpy(), g["d_items"], rtol=1e-4, atol=1e-6), (items, g["d_items"])
    loss.backward()
    grads = dict(m.named_parameters())
    rows = []
    for name, norm, idx, smp in zip(g["d_names"], g["d_norms"], g["d_sample_idx"], g["d_samples"]):
        name = str(name)
        gr = grads[name].grad.reshape(-1)
        got = gr[torch.from_numpy(np.asarray(idx, dtype=np.int64)).cuda()].cpu().numpy()
        scale = max(float(np.abs(smp).max()), float(norm) / gr.numel() ** 0.5)
        if name.endswith("activation.weight"):
            sscale = max(float(nn_) for nm_, nn_ in zip(g["d_names"], g["d_norms"]) if str(nm_).endswith("activation.weight"))
            e = abs(float(gr[0]) - float(np.asarray(smp).reshape(-1)[0])) / sscale
            rows.append((int(name.split(".")[1]), name, e, e))
            continue
        rows.append((int(name.split(".")[1]), name, float(np.abs(got - smp).max()) / scale,
                     abs(float(gr.norm()) - float(norm)) / float(norm)))
    report_and_check_gradients("darknet-53 160x128 trained with Fdefault", rows)


def test_bf16_fdefault_training_step_with_cuda_graphs_is_bitwise_repeatable():
    from rotate_yolov3_b200.loss import compute_loss
    hyp = dict(STEP_HYP, fl_gamma=0.5)

    def setup(m):
        m.nc, m.hyp, m.arc = 1, hyp, "Fdefault"
        return m

    def step(m, x, t):
        for p in m.parameters():
            p.grad = None
        ps = m(x)
        loss, items = compute_loss(ps, t.clone(), m, hyp)
        loss.backward()
        out = {"loss": loss.detach().clone(), "items": items.detach().clone()}
        for n, p in m.named_parameters():
            out["grad:" + n] = p.grad.clone()
        torch.cuda.synchronize()
        return out
    m = setup(small_train_model())
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    x = torch.rand(2, 3, 128, 160, generator=torch.Generator().manual_seed(17)).cuda()
    t = step_targets()
    ref = step(m, x, t)
    assert float(ref["items"][2]) > 0 and all(torch.isfinite(v).all() for v in ref.values())
    m.load_state_dict(sd0)
    assert_same(ref, step(m, x, t), "rerun")
    m3 = setup(small_train_model())
    m3.load_state_dict(sd0)
    m3.use_cuda_graph = True
    assert_same(ref, step(m3, x, t), "graph capture step")
    m3.load_state_dict(sd0)                      # in place: the captured graphs stay valid
    assert_same(ref, step(m3, x, t), "graph replay")
    assert m3._tplan.replayed_kernels > 0
