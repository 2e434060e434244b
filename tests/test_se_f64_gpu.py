"""Every SE kernel of one bf16 training step of the reference's SE graphs, at their native sizes (yolov3_512_se.cfg at
512 x 512, yolov3_608_se.cfg at 608 x 608), batch 2, against float64 of the inputs it actually received.  A dense random
cotangent per head (loss = sum (p * G)) reaches every SE.

Forward (post hoc: the plan keeps x, u, m, p, s):  m = mean_hw x, p = W1 m, s = sigmoid(W2 relu(p)), u = bf16(x s).
Backward: plan._backward_block is wrapped (instance attribute) so that the production order and accumulate flags run
unchanged; gu, x and the prior gx are snapshotted before the block and its SE run, and ds, dm, gx, gW1, gW2 are checked
right after.  Bounds (U = 2^-24, the fp32 unit roundoff):
  m, ds     L U sum|terms| (+ U |m| for the division), L = the longest fp32 addition chain of the launch: the pixels one
            thread adds in its span, the lanes of a channel, the spans (se_chain mirrors se_nsplit in csrc/se.cu)
  p, dhid   (n + 1) U |W| |v|, n terms; dhid also carries da's 3 U relative error; dm carries dhid's error through W1^T
  s         s (1 - s) (cr + 1) U |W2| |relu(p)| + 4 U s   (expf, the add and the division)
  gW1, gW2  (B + 1) U sum_b |a||b| plus the propagated error of da / dhid
  u, gx     half a bf16 ulp of the float64 result + the fp32 terms (3 U each), and no rounding bias:
            |mean((got - want) sign(want))| <= 2^-12 rms(want)
Every ratio |err| / bound must be <= 1.  Wiring is checked through the plan's pointers: the 1x1 conv after each SE reads u,
each `from=-4` shortcut adds x, the concat routes' sources 36 / 61 are the unscaled x (and have three gradient writers:
the concat consumer's dgrad, the unit's shortcut gradient, the SE), and the halos of u and gu are zero.  A last test puts
plausible bugs into the stored tensors and requires a check to fail on each."""
import os
import types

import pytest
import torch

from builders import REF_CFG
from checked_step import Step, backward, dense_loss
from f64_refs import TINY, U, bf16_check, halo_zero, rtz_bf16, se_chain, vint
from helpers import init_darknet_weights

pytestmark = pytest.mark.gpu

BATCH = 2


def ratio(got, want, bound):
    return float(((got.double() - want).abs() / (bound + TINY)).max())


def fwd_refs(se, x, w1, w2):
    """float64 references of the forward outputs from the kernels' own inputs; returns (refs, bounds)"""
    B, hw = x.shape[0], se.h * se.w
    c, cr = se.c, se.cr
    m, p, s = se.m.view(B, c).double(), se.p.view(B, cr).double(), se.s.view(B, c).double()
    xd = x.double()
    m64 = xd.sum((1, 2)) / hw
    m_b = se_chain(se.h, se.w, c) * U * xd.abs().sum((1, 2)) / hw + U * m64.abs()
    p64 = m @ w1.t()
    p_b = (c + 1) * U * (m.abs() @ w1.abs().t())
    hid = p.clamp(min=0)
    a64 = hid @ w2.t()
    s64 = torch.sigmoid(a64)
    s_b = s64 * (1 - s64) * (cr + 1) * U * (hid @ w2.abs().t()) + 4 * U * s64
    u64 = xd * s.view(B, 1, 1, c)
    return dict(m=(m64, m_b), p=(p64, p_b), s=(s64, s_b), u=(u64, 3 * U * u64.abs()))


def bwd_refs(se, gu, x, gx_old, w1, w2, gw1, gw2):
    B, hw = x.shape[0], se.h * se.w
    c, cr = se.c, se.cr
    m, p, s = se.m.view(B, c).double(), se.p.view(B, cr).double(), se.s.view(B, c).double()
    ds, dm = se.ds.view(B, c).double(), se.dm.view(B, c).double()
    prod = gu.double() * x.double()
    ds64 = prod.sum((1, 2))
    ds_b = se_chain(se.h, se.w, c) * U * prod.abs().sum((1, 2))
    da = ds * s * (1 - s)
    mask = (p > 0).double()
    dh_mag = da.abs() @ w2.abs()
    dhid = (da @ w2) * mask
    dh_err = (c + 4) * U * dh_mag * mask
    dm64 = dhid @ w1
    dm_b = (cr + 1) * U * (dhid.abs() @ w1.abs()) + dh_err @ w1.abs()
    hid = p.clamp(min=0)
    gw2_64 = da.t() @ hid
    gw2_b = (B + 4) * U * (da.abs().t() @ hid)
    gw1_64 = dhid.t() @ m
    gw1_b = (B + 1) * U * (dhid.abs().t() @ m.abs()) + dh_err.t() @ m.abs()
    gus = gu.double() * s.view(B, 1, 1, c)
    dmh = (dm / hw).view(B, 1, 1, c)
    gx64 = gus + dmh + (gx_old.double() if gx_old is not None else 0.0)
    gx_e = 3 * U * (gus.abs() + dmh.abs() + (gx_old.double().abs() if gx_old is not None else 0.0))
    return dict(ds=(ds64, ds_b), dm=(dm64, dm_b), gw1=(gw1_64, gw1_b), gw2=(gw2_64, gw2_b), gx=(gx64, gx_e))


def _run(cfg, size, seed):
    import rotate_yolov3_b200 as pkg
    cwd = os.getcwd()
    os.chdir(REF_CFG)
    try:
        model = pkg.Darknet(cfg, {"context_factor": 1.0}, arc="default")
    finally:
        os.chdir(cwd)
    init_darknet_weights(model, seed=seed)
    model = model.cuda().train()
    x = torch.rand(BATCH, 3, size, size, generator=torch.Generator().manual_seed(seed + 1)).cuda()
    st = Step(model, x)
    ps = model(x)
    torch.cuda.synchronize()
    plan = model._tplan
    st.plan = plan
    st.ses = [b.se for b in plan.blocks if b.se is not None]
    st.fwd, st.keep = {}, {}
    for se in st.ses:
        fc = model.module_list[se.i].fc
        w1, w2 = fc[0].weight.detach().double(), fc[2].weight.detach().double()
        xv = vint(se.x)
        refs = fwd_refs(se, xv, w1, w2)
        r = {}
        B = BATCH
        r["m"] = ratio(se.m.view(B, se.c), *refs["m"])
        r["p"] = ratio(se.p.view(B, se.cr), *refs["p"])
        r["s"] = ratio(se.s.view(B, se.c), *refs["s"])
        r.update({"u_" + k: v for k, v in bf16_check(vint(se.u), *refs["u"]).items()})
        r["halo_u"] = halo_zero(se.u.buf)
        st.fwd[se.i] = r
    loss = dense_loss(st, ps, seed + 2)

    def check(st, blk, orig):
        """the SE of the block: gu, x and the prior gx snapshotted, the block and its SE run, then checked (recorded
        under the SE's layer index)"""
        se = blk.se
        if se is None:
            orig(blk)
            return None
        gu, xv = vint(se.gu).clone(), vint(se.x).clone()
        gx_old = vint(se.gx).clone() if se.gx_acc else None
        orig(blk)
        fc = model.module_list[se.i].fc
        refs = bwd_refs(se, gu, xv, gx_old, fc[0].weight.detach().double(), fc[2].weight.detach().double(), se.gw1, se.gw2)
        B = BATCH
        r = {"acc": bool(se.gx_acc)}
        r["ds"] = ratio(se.ds.view(B, se.c), *refs["ds"])
        r["dm"] = ratio(se.dm.view(B, se.c), *refs["dm"])
        r["gw1"] = ratio(se.gw1.view(se.cr, se.c), *refs["gw1"])
        r["gw2"] = ratio(se.gw2.view(se.c, se.cr), *refs["gw2"])
        r.update({"gx_" + k: v for k, v in bf16_check(vint(se.gx), *refs["gx"]).items()})
        r["halo_gu"] = halo_zero(se.gu.buf)
        st.bwd[se.i] = r
        if se.i == st.ses[0].i:
            st.keep = dict(se=se, gu=gu, x=xv, gx_old=gx_old, refs=refs,
                           fwd=fwd_refs(se, xv, fc[0].weight.detach().double(), fc[2].weight.detach().double()))
    backward(st, loss, check)
    return st


@pytest.fixture(scope="module", params=[("cfg/HRSC+/yolov3_512_se.cfg", 512), ("cfg/ICDAR/yolov3_608_se.cfg", 608)],
                ids=["se512", "se608"])
def step(request):
    cfg, size = request.param
    st = _run(cfg, size, 11)
    worst = {}
    for d in (st.fwd, st.bwd):
        for i, r in d.items():
            for k, v in r.items():
                if isinstance(v, float) and v > worst.get(k, (-1, 0))[0]:
                    worst[k] = (v, i)
    print("\n[%s] worst |err| / bound per quantity (SE block): %s" % (
        request.node.callspec.id if hasattr(request.node, "callspec") else size,
        ", ".join("%s %.3f (%d)" % (k, v, i) for k, (v, i) in sorted(worst.items()))))
    return st


def _passed(r):
    return all((v <= 1.0) if isinstance(v, float) else v for k, v in r.items() if k != "acc")


def test_se_wiring(step):
    plan = step.plan
    assert len(step.ses) == 20
    by_i = {b.i: b for b in plan.blocks}
    for se in step.ses:
        conv1 = by_i[se.i + 1]
        assert conv1.k == 1 and conv1.src is se.u and conv1.gsrc is se.gu, se.i
        conv3 = by_i[se.i + 2]
        assert conv3.fuse_res and conv3.res is se.x and conv3.gres is se.gx, se.i
        assert se.u.buf.data_ptr() != se.x.buf.data_ptr()
    for i in (37, 62):
        se = next(s_ for s_ in step.ses if s_.i == i)
        assert se.x.buf.shape[-1] > se.x.c                       # x lives in the concat buffer of route 118 / 106
        concat = [b for b in plan.blocks if b.gsrc is not None and b.gsrc.buf is se.gx.buf and b.gsrc.c > se.x.c]
        assert len(concat) == 1                                  # the concat consumer's dgrad writes gx first ...
        assert by_i[i + 2].gres_acc and se.gx_acc                # ... the shortcut gradient and the SE accumulate
    # every SE input is also a shortcut source, whose gradient (the 3x3 block's bn_act_bwd) comes first: the SE accumulates
    assert all(s_.gx_acc for s_ in step.ses)


def test_se_forward_kernels_vs_float64(step):
    bad = {i: r for i, r in step.fwd.items() if not _passed(r)}
    assert not bad, bad


def test_se_backward_kernels_vs_float64(step):
    assert set(step.bwd) == {se.i for se in step.ses}
    bad = {i: r for i, r in step.bwd.items() if not _passed(r)}
    assert not bad, bad
    assert all(r["acc"] for r in step.bwd.values())


def test_bounds_reject_plausible_bugs(step):
    """each bug, put into the stored tensors, fails its check; the factors are printed with -s"""
    out = {}
    k = step.keep
    se, hw = k["se"], k["se"].h * k["se"].w
    B, c = BATCH, se.c
    s_ = se.s.view(B, c)
    m_pad = se.m.view(B, c) * hw / ((se.h + 2) * (se.w + 2))
    out["mean over the padded grid"] = ratio(m_pad, *k["fwd"]["m"])
    u_img0 = (k["x"].float() * s_[0].view(1, 1, 1, c)).to(torch.bfloat16)
    out["image 1 scaled by image 0's s"] = bf16_check(u_img0, *k["fwd"]["u"])["max"]
    out["u rounded toward zero (bias)"] = bf16_check(rtz_bf16(k["x"].float() * s_.view(B, 1, 1, c)), *k["fwd"]["u"])["bias"]
    gx_nodm = (k["gx_old"].float() + k["gu"].float() * s_.view(B, 1, 1, c)).to(torch.bfloat16)
    out["dm / hw dropped"] = bf16_check(gx_nodm, *k["refs"]["gx"])["max"]
    gx_over = (k["gu"].float() * s_.view(B, 1, 1, c) + (se.dm.view(B, c) / hw).view(B, 1, 1, c)).to(torch.bfloat16)
    out["gx overwritten instead of accumulated"] = bf16_check(gx_over, *k["refs"]["gx"])["max"]
    p = se.p.view(B, se.cr).double()
    da = se.ds.view(B, c).double() * s_.double() * (1 - s_.double())
    dh_last = (da[-1] @ step.model.module_list[se.i].fc[2].weight.detach().double()) * (p[-1] > 0).double()
    gw1 = se.gw1.view(se.cr, c).double() - torch.outer(dh_last, se.m.view(B, c)[-1].double())
    out["gW1 missing the last image"] = ratio(gw1, *k["refs"]["gw1"])
    print("\n[se bugs] |err| / bound: " + ", ".join("%s %.3g" % kv for kv in out.items()))
    assert all(v > 1.0 for v in out.values()), out


def test_se_kernels_first_writer_accumulate_and_relu_at_zero():
    """ryolo_se_bwd alone: gx as the first writer and accumulating (the reference graphs only accumulate), and hidden units
    with p == 0 exactly (a zero row of W1) pass no gradient, like torch's relu backward"""
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import layout as L
    lib, dev = pkg._lib.lib, torch.device("cuda")
    B, h, w, c, cr = 3, 19, 19, 256, 16
    g = torch.Generator().manual_seed(5)
    x = L.to_padded_nhwc(torch.randn(B, c, h, w, generator=g).to(dev), 256)
    gu = L.to_padded_nhwc(torch.randn(B, c, h, w, generator=g).to(dev), 256)
    u, gx = torch.zeros_like(x), torch.zeros_like(x)
    w1 = (torch.randn(cr, c, generator=g) * 0.1).to(dev)
    w1[3] = 0
    w2 = (torch.randn(c, cr, generator=g) * 0.1).to(dev)
    f = lambda n: torch.zeros(n, dtype=torch.float32, device=dev)     # noqa: E731
    m, p, s, ds, dm, gw1, gw2 = f(B * c), f(B * cr), f(B * c), f(B * c), f(B * c), f(cr * c), f(c * cr)
    ws = torch.empty(lib.ryolo_se_workspace_bytes(B, h, w, c, cr), dtype=torch.uint8, device=dev)
    P, st = pkg._lib.ptr, pkg._lib.stream_ptr(dev)
    assert lib.ryolo_se_fwd(P(x), 256, P(u), 256, B, h, w, c, P(w1), P(w2), cr, P(m), P(p), P(s), P(ws), ws.numel(), st) == 0
    assert lib.ryolo_se_bwd(P(gu), 256, P(x), 256, P(gx), 256, 0, B, h, w, c, P(w1), P(w2), cr, P(m), P(p), P(s), P(ds), P(dm),
                            P(gw1), P(gw2), P(ws), ws.numel(), st) == 0
    torch.cuda.synchronize()
    se = types.SimpleNamespace(h=h, w=w, c=c, cr=cr, m=m, p=p, s=s, ds=ds, dm=dm)
    xi, gui = x[:, 1:-1, 1:-1], gu[:, 1:-1, 1:-1]
    r = bf16_check(gx[:, 1:-1, 1:-1], *bwd_refs(se, gui, xi, None, w1.double(), w2.double(), gw1, gw2)["gx"])
    assert r["max"] <= 1 and r["bias"] <= 1, r                     # first writer
    gx_old = gx.clone()
    assert lib.ryolo_se_bwd(P(gu), 256, P(x), 256, P(gx), 256, 1, B, h, w, c, P(w1), P(w2), cr, P(m), P(p), P(s), P(ds), P(dm),
                            P(gw1), P(gw2), P(ws), ws.numel(), st) == 0
    torch.cuda.synchronize()
    r = bf16_check(gx[:, 1:-1, 1:-1], *bwd_refs(se, gui, xi, gx_old[:, 1:-1, 1:-1], w1.double(), w2.double(), gw1, gw2)["gx"])
    assert r["max"] <= 1 and r["bias"] <= 1, r                     # accumulating
    assert halo_zero(gx) and halo_zero(u)
    assert bool((p.view(B, cr)[:, 3] == 0).all())
    assert bool((gw1.view(cr, c)[3] == 0).all()) and bool((gw2.view(c, cr)[:, 3] == 0).all())
    assert float(gw1.view(cr, c).abs().sum()) > 0
