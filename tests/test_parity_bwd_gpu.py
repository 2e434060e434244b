"""Parity-precision backward, kernel by kernel, against float64 at the shapes parity training runs.

The end-to-end gradient tests (test_parity_gpu.py) cannot bound the layers below the heads tightly: a PReLU kink
crossing flips whole channels.  Here every backward kernel gets the same fp32 inputs as a float64 reference, with no
graph in between, so no crossing can happen and the bounds can be those of the forward test (test_px_conv_vs_float64):

    max |got - want| <= 5e-6 * max |want|,   rms(got - want) <= 2e-6 * rms(want),
    |mean((got - want) * sign(want))| <= 1e-6 * rms(want)                                     (no truncation bias)

Operands are arbitrary fp32 values, split into three bf16 planes by ryolo_px_split_from_nchw.

  1. weight gradient: ryolo_px_wgrad over all planes of dz and x + ryolo_px_unpack_wgrad, buffers built as ParityPlan
     builds them (first layer on the im2col columns, space-to-depth layers on the xs buffer, a slice of a concat buffer).
     The bf16 path's ryolo_conv_wgrad keeps ONE wgmma accumulator over the whole pixel range of a split, and the tensor
     pipe's accumulator does not round to nearest.  On parity operands its bias grows with the chain length: measured
     on an H100 SXM (132 SMs, 400 W), bias/rms -9.0e-6 (708 updates per chain) .. -2.1e-5 (1676) at batch 2 and
     -7.5e-5 (5640) .. -1.7e-4 (13380) at batch 16, max error up to 2.7e-4 of scale.  ryolo_px_wgrad restarts the
     accumulator every 8 k-steps (32 updates) and folds it into round-to-nearest fp32 sums, as px_conv does: bias/rms
     -2.3e-7 .. -3.4e-7 and max error <= 7.8e-7 of scale on every case, whatever the chain length.  The test runs both
     and requires the old path to fail the bias bound on the 608 x 608 layers, so the cases keep showing the defect the
     segmented accumulation removes.
  2. input gradient: px_pack_weights modes 1 / 3 + px_conv (ksize 3, 1, -2; accumulate 0 / 1) + px_depth_to_space.
  3. px_bn_act_bwd: BatchNorm backward (batch / running statistics) through PReLU, the PReLU branch decided on the host
     with the kernel's own fp32 arithmetic.
  4. px_bn_stats + px_bn_finalize: two-pass float64 statistics, running-statistics update, eval mode.
  5. elementwise and layout kernels with one rounding each: bit for bit against a torch fp32 emulation.
  6. each bound fails on a reference with one plausible kernel bug put in."""
import pytest
import torch
import torch.nn.functional as F

from builders import ryolo_lib
from f64_refs import (NP, PX_BIAS_TOL, PX_MAX_TOL, PX_RMS_TOL, U, BnCase, bn_errors, f32_buf, gemm_sms, measure, merge3,
                      planes_of, px_call, rup, split3, stream, ulps_f32, vp)
from helpers import wgrad_plan

pytestmark = pytest.mark.gpu

H100_SXM_SMS = 132


def _PP():
    from rotate_yolov3_b200 import parity_path as PP
    return PP


# ---------------------------------------------------------------------------------------------------------------
# split operands
def split_buf(x, plane, ch_off=0, cs=None):
    """fp32 NCHW -> split padded NHWC [B, H+2, W+2, NP*plane] (or cs channels): x at channels ch_off.. of every plane"""
    b, c, h, w = x.shape
    cs = NP * plane if cs is None else cs
    buf = torch.zeros((b, h + 2, w + 2, cs), dtype=torch.bfloat16, device=x.device)
    px_call("ryolo_px_split_from_nchw", vp(x.contiguous()), b, c, h, w, vp(buf, 2 * ch_off), cs, plane, NP, stream())
    return buf


def nchw(buf, c, ch_off=0):
    return buf[:, 1:-1, 1:-1, ch_off:ch_off + c].permute(0, 3, 1, 2)


# ---------------------------------------------------------------------------------------------------------------
# the three bounds
def within(m):
    return m["max"] <= PX_MAX_TOL and m["rms"] <= PX_RMS_TOL and abs(m["bias"]) <= PX_BIAS_TOL


def fmt(m):
    return "max/scale %.2e  rms/rms %.2e  bias/rms %+.2e" % (m["max"], m["rms"], m["bias"])


# ---------------------------------------------------------------------------------------------------------------
# 1. weight gradient
class WgradCase:
    """One parity weight gradient as ParityPlan.backward runs it: dz [B, H+2, W+2, 3 po] with cout_pad = 3 po, x = the
    whole split source buffer (im2col columns, space-to-depth xs, or a concat buffer with x in a slice)."""

    def __init__(self, kind, batch, h, w, cin, cout, ksize=3, ch_off=0, ctot=None, seed=0):
        dev = torch.device("cuda")
        g = torch.Generator().manual_seed(seed)
        self.kind, self.b, self.cin, self.cout, self.ch_off = kind, batch, cin, cout, ch_off
        self.po = rup(cout, 64)
        if kind == "first":              # 3x3 conv on the image through its im2col columns (27 of 64 per plane)
            img = torch.randn(batch, 3, h, w, generator=g).to(dev)
            self.x = img
            self.xw = torch.zeros((batch, h + 2, w + 2, NP * 64), dtype=torch.bfloat16, device=dev)
            px_call("ryolo_px_im2col_first", vp(img), batch, h, w, vp(self.xw), NP * 64, 64, NP, stream())
            self.gh, self.gw, self.k = h, w, 1
            self.dz = torch.randn(batch, cout, h, w, generator=g).to(dev)
        elif kind == "s2d":              # 3x3 / stride 2 on [B, cin, h, w]: 2x2 taps on the space-to-depth buffer
            self.x = torch.randn(batch, cin, h, w, generator=g).to(dev)
            plane = rup(cin, 64)
            src = split_buf(self.x, plane)
            self.p4 = rup(4 * cin, 64)
            self.xw = torch.zeros((batch, h // 2 + 2, w // 2 + 2, NP * self.p4), dtype=torch.bfloat16, device=dev)
            for k in range(NP):
                px_call("ryolo_space_to_depth", vp(src, 2 * k * plane), NP * plane, batch, h, w, cin,
                      vp(self.xw, 2 * k * self.p4), NP * self.p4, stream())
            self.gh, self.gw, self.k = h // 2, w // 2, 2
            self.dz = torch.randn(batch, cout, h // 2, w // 2, generator=g).to(dev)
        else:                            # k x k stride 1, x at channel ch_off of a ctot-channel buffer
            ctot = cin if ctot is None else ctot
            full = torch.randn(batch, ctot, h, w, generator=g).to(dev) * 4.0 + 3.0     # sentinels around the slice
            self.x = torch.randn(batch, cin, h, w, generator=g).to(dev)
            full[:, ch_off:ch_off + cin] = self.x
            self.xw = split_buf(full, rup(ctot, 64))
            self.gh, self.gw, self.k = h, w, ksize
            self.dz = torch.randn(batch, cout, h, w, generator=g).to(dev)
        self.dzb = split_buf(self.dz, self.po)
        self.xcs = self.xw.shape[-1]

    def plan(self, segmented=True):
        return wgrad_plan(self.k, self.xcs, NP * self.po, self.b, self.gh, self.gw, gemm_sms(), segmented=segmented)

    def run(self, entry="ryolo_px_wgrad"):
        dev = self.dz.device
        dw = torch.zeros((self.k * self.k, NP * self.po, self.xcs), dtype=torch.float32, device=dev)
        px_call(entry, vp(self.dzb), NP * self.po, NP * self.po, vp(self.xw), self.xcs, self.xcs, self.b, self.gh, self.gw,
              self.k, vp(dw), stream())
        return dw

    def unpack(self, dw):
        pi = self.xcs // NP
        if self.kind == "first":
            gw = torch.full((self.cout, 27, 1, 1), float("nan"), device=dw.device)
            px_call("ryolo_px_unpack_wgrad", vp(dw), self.po, pi, NP, 0, self.cout, 27, 1, 0, vp(gw), stream())
            return gw.view(self.cout, 3, 3, 3)
        if self.kind == "s2d":
            gw = torch.full((self.cout, self.cin, 3, 3), float("nan"), device=dw.device)
            px_call("ryolo_px_unpack_wgrad", vp(dw), self.po, pi, NP, 2, self.cout, self.cin, 3, 0, vp(gw), stream())
            return gw
        gw = torch.full((self.cout, self.cin, self.k, self.k), float("nan"), device=dw.device)
        px_call("ryolo_px_unpack_wgrad", vp(dw), self.po, pi, NP, 0, self.cout, self.cin, self.k, self.ch_off, vp(gw), stream())
        return gw

    def ref_fn(self):
        if self.kind == "first":
            return lambda x, dz: torch.nn.grad.conv2d_weight(x, (self.cout, 3, 3, 3), dz, padding=1)
        if self.kind == "s2d":
            return lambda x, dz: torch.nn.grad.conv2d_weight(x, (self.cout, self.cin, 3, 3), dz, stride=2, padding=1)
        return lambda x, dz: torch.nn.grad.conv2d_weight(x, (self.cout, self.cin, self.k, self.k), dz,
                                                         padding=(self.k - 1) // 2)

    def ref(self):
        return self.ref_fn()(self.x.double(), self.dz.double())


# name -> (WgradCase kwargs, (ksplit, updates per chain) of ryolo_px_wgrad, of ryolo_conv_wgrad; on a 132-SM H100 SXM)
WGRAD_CASES = {
    "l0_first_b2": (dict(kind="first", batch=2, h=608, w=608, cin=3, cout=32), (22, 2116), (66, 708)),
    "l1_s2d_b2": (dict(kind="s2d", batch=2, h=608, w=608, cin=32, cout=64), (5, 2344), (8, 1464)),
    "l3_k3_b2": (dict(kind="k3", batch=2, h=304, w=304, cin=32, cout=64), (7, 1676), (7, 1676)),
    "k3_128_256_b2": (dict(kind="k3", batch=2, h=76, w=76, cin=128, cout=256), (3, 256), (1, 764)),
    "concat_slice": (dict(kind="k3", batch=2, h=38, w=38, cin=64, cout=64, ch_off=64, ctot=192), (3, 68), (4, 52)),
    "k1_1024_512": (dict(kind="k1", batch=2, h=19, w=19, cin=1024, cout=512, ksize=1), (1, 56), (1, 56)),
    "cout40": (dict(kind="k3", batch=2, h=76, w=76, cin=64, cout=40), (7, 112), (7, 112)),
    "l0_first_b16": (dict(kind="first", batch=16, h=608, w=608, cin=3, cout=32), (22, 16916), (66, 5640)),
    "l1_s2d_b16": (dict(kind="s2d", batch=16, h=608, w=608, cin=32, cout=64), (5, 18728), (8, 11708)),
    "l3_k3_b16": (dict(kind="k3", batch=16, h=304, w=304, cin=32, cout=64), (7, 13380), (7, 13380)),
    "k3_128_256_b16": (dict(kind="k3", batch=16, h=76, w=76, cin=128, cout=256), (3, 2028), (1, 6084)),
}


def check_wplan(plan, want):
    if gemm_sms() != H100_SXM_SMS:
        return
    ks, upd = want
    if ks is not None:
        assert plan["ksplit"] == ks, (plan, want)
    if upd is not None:
        assert plan["updates"] == upd, (plan, want)


@pytest.mark.parametrize("name", list(WGRAD_CASES))
def test_px_wgrad_vs_float64(name):
    kw, want_seg, want_old = WGRAD_CASES[name]
    c = WgradCase(**kw, seed=len(name))
    ps, po = c.plan(True), c.plan(False)
    check_wplan(ps, want_seg)
    check_wplan(po, want_old)
    want = c.ref()
    got = c.unpack(c.run())
    old = c.unpack(c.run("ryolo_conv_wgrad"))
    torch.cuda.synchronize()
    m, mo = measure(got, want), measure(old, want)
    print("[px_wgrad] %-15s px_wgrad  (bn %3d tg %d ksplit %3d, %5d updates per chain, restarted every 32): %s"
          % (name, ps["bn"], ps["tg"], ps["ksplit"], ps["updates"], fmt(m)))
    print("[px_wgrad] %-15s conv_wgrad(bn %3d tg %d ksplit %3d, %5d updates per chain):                    %s"
          % (name, po["bn"], po["tg"], po["ksplit"], po["updates"], fmt(mo)))
    assert not torch.isnan(got).any()
    assert within(m), (name, m)
    if po["updates"] >= 700:
        # the 608 x 608 layers: one unrestarted accumulator over >= 700 updates is biased towards zero (measured on an
        # H100 SXM: bias/rms -9.0e-6 .. -2.1e-5 at batch 2, -7.5e-5 .. -1.7e-4 at batch 16)
        assert mo["bias"] < -PX_BIAS_TOL, (name, mo)


# ---------------------------------------------------------------------------------------------------------------
# 2. input gradient
def run_dgrad(dz, wt, h, w, stride, gbuf, ch_off, accumulate):
    """d x of the conv wt [cout, cin, k, k] (stride 1 / 2) for output gradient dz, into gbuf[..., ch_off:] as
    ParityPlan.backward runs it"""
    PP = _PP()
    b, cout = dz.shape[:2]
    cin, k = wt.shape[1], wt.shape[2]
    po = rup(cout, 64)
    dzb = split_buf(dz, po)
    dev = dz.device
    if stride == 1:
        pwd = torch.empty(ryolo_lib().lib.ryolo_px_packed_weight_bytes(cin, cout, k, PP.NTERMS), dtype=torch.uint8, device=dev)
        px_call("ryolo_px_pack_weights", vp(wt), cin, cout, k, PP.NTERMS, PP.W_CODE, 1, vp(pwd), stream())
        px_call("ryolo_px_conv", vp(dzb), NP * po, 0, po, cout, vp(pwd), PP.NTERMS, PP.A_CODE, b, h, w, k, cin,
              vp(gbuf, 4 * ch_off), gbuf.shape[-1], rup(cin, 4), accumulate, stream())
    else:
        p4 = rup(4 * cin, 64)
        pwd = torch.empty(ryolo_lib().lib.ryolo_px_packed_weight_bytes(4 * cin, cout, 2, PP.NTERMS), dtype=torch.uint8, device=dev)
        px_call("ryolo_px_pack_weights", vp(wt), 4 * cin, cout, -2, PP.NTERMS, PP.W_CODE, 3, vp(pwd), stream())
        dxs = f32_buf(b, h // 2, w // 2, p4, dev)
        px_call("ryolo_px_conv", vp(dzb), NP * po, 0, po, cout, vp(pwd), PP.NTERMS, PP.A_CODE, b, h // 2, w // 2, -2,
              4 * cin, vp(dxs), p4, p4, 0, stream())
        px_call("ryolo_px_depth_to_space", vp(dxs), p4, b, h, w, cin, vp(gbuf, 4 * ch_off), gbuf.shape[-1], accumulate,
              stream())


def ref_dgrad(dz, wt, h, w, stride):
    k = wt.shape[2]
    return torch.nn.grad.conv2d_input((dz.shape[0], wt.shape[1], h, w), wt.double(), dz.double(), stride=stride,
                                      padding=(k - 1) // 2)


DGRAD_CASES = {
    "k3_128_64_152": dict(batch=2, cin=128, cout=64, h=152, w=152, k=3, stride=1),
    "s2_64_128_304": dict(batch=2, cin=64, cout=128, h=304, w=304, k=3, stride=2),
    "k1_1024_512_19": dict(batch=2, cin=1024, cout=512, h=19, w=19, k=1, stride=1),
    "k3_cin40": dict(batch=2, cin=40, cout=64, h=38, w=38, k=3, stride=1),
    "k1_slice": dict(batch=2, cin=64, cout=128, h=38, w=38, k=1, stride=1, ch_off=64, gcs=192),
    "s2_slice": dict(batch=2, cin=32, cout=64, h=76, w=76, k=3, stride=2, ch_off=32, gcs=128),
}


def dgrad_inputs(batch, cin, cout, h, w, k, stride, seed):
    g = torch.Generator().manual_seed(seed)
    dz = torch.randn(batch, cout, h // stride, w // stride, generator=g).cuda()
    wt = (torch.randn(cout, cin, k, k, generator=g) / (cout * k * k) ** 0.5).cuda()
    return dz, wt


@pytest.mark.parametrize("name", list(DGRAD_CASES))
def test_px_dgrad_vs_float64(name):
    kw = dict(DGRAD_CASES[name])
    ch_off, gcs = kw.pop("ch_off", 0), kw.pop("gcs", None)
    batch, cin, h, w, stride = kw["batch"], kw["cin"], kw["h"], kw["w"], kw["stride"]
    gcs = rup(cin, 64) if gcs is None else gcs
    dz, wt = dgrad_inputs(**kw, seed=len(name))
    g = torch.Generator().manual_seed(99)
    # the gradient buffer: zero halo, sentinels in every interior channel outside the written columns
    cols = rup(cin, 4) if stride == 1 else cin
    base = f32_buf(batch, h, w, gcs)
    base[:, 1:-1, 1:-1] = torch.randn(batch, h, w, gcs, generator=g).cuda() + 7.0
    prior = torch.randn(batch, h, w, cols, generator=g).cuda()
    g0 = base.clone()
    run_dgrad(dz, wt, h, w, stride, g0, ch_off, 0)
    g1 = base.clone()
    g1[:, 1:-1, 1:-1, ch_off:ch_off + cols] = prior
    run_dgrad(dz, wt, h, w, stride, g1, ch_off, 1)
    torch.cuda.synchronize()
    want = ref_dgrad(dz, wt, h, w, stride)
    m = measure(nchw(g0, cin, ch_off), want)
    print("[px_dgrad] %-15s %s" % (name, fmt(m)))
    assert within(m), (name, m)
    outside = torch.ones(gcs, dtype=torch.bool, device="cuda")
    outside[ch_off:ch_off + cols] = False
    for gb in (g0, g1):
        assert torch.equal(gb[:, 0], base[:, 0]) and torch.equal(gb[:, -1], base[:, -1])     # halo rows stay zero
        assert torch.equal(gb[:, :, 0], base[:, :, 0]) and torch.equal(gb[:, :, -1], base[:, :, -1])
        assert torch.equal(gb[..., outside], base[..., outside])                            # sentinels intact
    if cols > cin:      # columns [cin, out_cols) of a stride-1 dgrad are written: nothing but zeros was added to them
        assert float(g0[:, 1:-1, 1:-1, ch_off + cin:ch_off + cols].abs().max()) == 0.0
    # accumulate = 1 is one fp32 add of the accumulate = 0 result to what the buffer held
    sl = (slice(None), slice(1, -1), slice(1, -1), slice(ch_off, ch_off + cols))
    assert torch.equal(g1[sl], prior + g0[sl])


# ---------------------------------------------------------------------------------------------------------------
# 3. BN + PReLU backward
BN_CASES = {
    "c8_act": dict(c=8, batch=2, h=20, w=20),
    "c40_up": dict(c=40, batch=2, h=19, w=19, up=True),
    "c64_gres_acc": dict(c=64, batch=2, h=38, w=38, gres="acc"),
    "c192_linear_gres": dict(c=192, batch=2, h=19, w=19, act=False, gres="set"),
    "c1024_running": dict(c=1024, batch=2, h=19, w=19, batch_stats=0),
    "c2048_one_pixel_per_block": dict(c=2048, batch=2, h=5, w=5),
    "c64_608_b16": dict(c=64, batch=16, h=304, w=304),
}


@pytest.mark.parametrize("name", list(BN_CASES))
def test_px_bn_act_bwd_vs_float64(name):
    case = BnCase(**BN_CASES[name], seed=len(name))
    if case.act:
        assert int((case.u() == 0).sum()) >= 4          # u exactly 0 is on the slope side, as in the kernel
    sums, dzb, gres = case.run()
    r = case.ref()
    e = bn_errors(case, sums, dzb, r)
    print("[px_bn_act_bwd] %-26s worst error / bound: %s" % (name, "  ".join("%s %.3f" % kv for kv in e.items())))
    assert all(v <= 1.0 for v in e.values()), e
    c, po = case.c, case.po
    # dz: halo and the channels [c, po) of every plane keep what the buffer held
    ini = case.dz_init
    assert torch.equal(dzb[:, 0], ini[:, 0]) and torch.equal(dzb[:, -1], ini[:, -1])
    assert torch.equal(dzb[:, :, 0], ini[:, :, 0]) and torch.equal(dzb[:, :, -1], ini[:, :, -1])
    for k in range(NP):
        assert torch.equal(dzb[..., k * po + c:(k + 1) * po], ini[..., k * po + c:(k + 1) * po])
    if gres is not None:
        got = nchw(gres, c)
        want = case.dy if case.old is None else case.old + case.dy
        assert torch.equal(got, want)
        assert torch.equal(gres[..., c:], case.gres_init[..., c:])
        assert float(gres[:, 0].abs().max()) == 0 and float(gres[:, :, 0].abs().max()) == 0


# ---------------------------------------------------------------------------------------------------------------
# 4. statistics
def test_px_bn_stats_and_finalize_vs_float64():
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(11)
    b, c, h, w = 2, 64, 38, 38
    mu = torch.randn(c, generator=g)
    sd = torch.rand(c, generator=g) + 0.5
    mu[:8] = 1e3 * sd[:8] * torch.sign(torch.randn(8, generator=g))       # mean / std = 1e3: one-pass variance
    z = (torch.randn(b, c, h, w, generator=g) * sd[None, :, None, None] + mu[None, :, None, None]).to(dev)
    z[:, 8] = 0.1                                                          # constant channel: variance 0
    z[:, 9] = -3.0e4
    po = 64
    zb = f32_buf(b, h, w, po + 64)
    zb[:, 1:-1, 1:-1, :c] = z.permute(0, 2, 3, 1)
    zb[..., c:] = 1e9                                                      # neighbouring channels are not read
    sums = torch.full((2 * c,), float("nan"), dtype=torch.float64, device=dev)
    px_call("ryolo_px_bn_stats", vp(zb), po + 64, b, h, w, c, vp(sums), stream())
    gamma = (torch.rand(c, generator=g) + 0.5).to(dev)
    beta = torch.randn(c, generator=g).to(dev)
    rm0 = torch.randn(c, generator=g).to(dev)
    rv0 = (torch.rand(c, generator=g) + 0.5).to(dev)
    rm, rv = rm0.clone(), rv0.clone()
    outs = [torch.full((c,), float("nan"), device=dev) for _ in range(4)]
    n = b * h * w
    eps, mom = 1e-5, 0.1
    px_call("ryolo_px_bn_finalize", vp(sums), c, float(n), eps, mom, vp(gamma), vp(beta), 0, *[vp(t) for t in outs],
          vp(rm), vp(rv), stream())
    torch.cuda.synchronize()
    mean, invstd, scale, shift = outs
    z64 = z.double()
    m64 = z64.mean((0, 2, 3))
    v64 = (z64 - m64[None, :, None, None]).pow(2).mean((0, 2, 3))           # two-pass
    want_inv = 1.0 / (v64 + eps).sqrt()
    e_mean = float(((mean.double() - m64).abs() / ulps_f32(m64)).max())
    e_inv = float(((invstd.double() - want_inv).abs() / ulps_f32(want_inv)).max())
    print("[px_bn_stats] worst |error| in fp32 ulps: mean %.2f, invstd %.2f" % (e_mean, e_inv))
    assert e_mean <= 2.0 and e_inv <= 2.0, (e_mean, e_inv)
    # constant channels: variance exactly 0 (clamped if the one-pass formula went negative), invstd = 1 / sqrt(eps)
    inv_eps = 1.0 / torch.sqrt(torch.tensor(0.0, device=dev) + eps)
    assert float(invstd[8]) == float(inv_eps) and float(invstd[9]) == float(inv_eps)
    assert torch.equal(scale, gamma * invstd)                               # one fp32 multiply
    sh_want = beta.double() - mean.double() * scale.double()
    assert bool(((shift.double() - sh_want).abs() <= 2 * U * (beta.double().abs() + (mean.double() * scale.double()).abs())
                 + 1e-38).all())
    # running statistics: momentum 0.1, unbiased variance
    rm_want = (1 - mom) * rm0.double() + mom * m64
    rv_want = (1 - mom) * rv0.double() + mom * v64 * n / (n - 1)
    tol_m = 4 * U * ((1 - mom) * rm0.double().abs() + mom * m64.abs())
    tol_v = 4 * U * ((1 - mom) * rv0.double().abs() + mom * v64 * n / (n - 1)) + 1e-12
    assert bool(((rm.double() - rm_want).abs() <= tol_m).all())
    assert bool(((rv.double() - rv_want).abs() <= tol_v).all())
    # eval mode: the running statistics, nothing written back (sums are not read)
    rm_e, rv_e = rm.clone(), rv.clone()
    outs_e = [torch.full((c,), float("nan"), device=dev) for _ in range(4)]
    px_call("ryolo_px_bn_finalize", None, c, 0.0, eps, mom, vp(gamma), vp(beta), 1, *[vp(t) for t in outs_e], vp(rm_e),
          vp(rv_e), stream())
    torch.cuda.synchronize()
    assert torch.equal(rm_e, rm) and torch.equal(rv_e, rv)
    assert torch.equal(outs_e[0], rm)
    want_inv_e = 1.0 / (rv.double() + eps).sqrt()
    assert float(((outs_e[1].double() - want_inv_e).abs() / ulps_f32(want_inv_e)).max()) <= 2.0
    assert torch.equal(outs_e[2], gamma * outs_e[1])


# ---------------------------------------------------------------------------------------------------------------
# 5. elementwise and layout kernels, bit for bit
def assert_planes(buf, plane, v, ch_off=0, up=False):
    """buf's planes at channels [ch_off, ch_off + c) == the split of fp32 v (NCHW), bitwise"""
    want = split3(v)
    got = planes_of(buf, plane, v.shape[1], ch_off)
    for k in range(NP):
        wk = want[k]
        if up:
            wk = wk.repeat_interleave(2, 2).repeat_interleave(2, 3)
        assert torch.equal(got[k].view(torch.int16), wk.view(torch.int16)), k


@pytest.mark.parametrize("form", ["plain", "residual", "upsample", "linear"])
def test_px_bn_act_fwd_bitwise(form):
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(21)
    b, c, h, w = 2, 72, 13, 11
    po = rup(c, 64)
    z = (torch.randn(b, c, h, w, generator=g) * 3).to(dev)
    scale = (torch.randn(c, generator=g) * 2).to(dev)
    shift = torch.randn(c, generator=g).to(dev)
    shift[0] = -(z[0, 0, 0, 0] * scale[0])                                   # u exactly 0
    slope = torch.tensor([0.13], device=dev)
    act = form != "linear"
    zb = f32_buf(b, h, w, po)
    zb[:, 1:-1, 1:-1, :c] = z.permute(0, 2, 3, 1)
    res = resb = None
    if form == "residual":
        res = (torch.randn(b, c, h, w, generator=g) * 2).to(dev)
        resb = split_buf(res, po)
    up = form == "upsample"
    oh, ow = (2 * h, 2 * w) if up else (h, w)
    y_init = torch.randn(b, oh + 2, ow + 2, NP * po, generator=g).to(torch.bfloat16).to(dev)
    yb = y_init.clone()
    px_call("ryolo_px_bn_act_fwd", vp(zb), po, b, h, w, c, vp(scale), vp(shift), vp(slope) if act else None, vp(resb),
          NP * po if res is not None else 0, po if res is not None else 0, vp(yb), NP * po, po, int(up), NP, stream())
    torch.cuda.synchronize()
    u = (z * scale[None, :, None, None]) + shift[None, :, None, None]
    if act:
        u = torch.where(u > 0, u, slope * u)
    if res is not None:
        u = u + merge3(*split3(res))
    assert_planes(yb, po, u, up=up)
    for k in range(NP):                                                     # channels [c, po) and the halo untouched
        assert torch.equal(yb[..., k * po + c:(k + 1) * po], y_init[..., k * po + c:(k + 1) * po])
    assert torch.equal(yb[:, 0], y_init[:, 0]) and torch.equal(yb[:, :, -1], y_init[:, :, -1])


@pytest.mark.parametrize("na,no,dlo", [(3, 7, 64), (72, 7, 512)])
def test_px_head_grad_bitwise(na, no, dlo):
    dev = torch.device("cuda")
    b, ny, nx = 2, 19, 17
    gr = torch.randn(b, na, ny, nx, no, generator=torch.Generator().manual_seed(na)).to(dev)
    dst = torch.zeros((b, ny + 2, nx + 2, NP * dlo), dtype=torch.bfloat16, device=dev)
    px_call("ryolo_px_head_grad", vp(gr), b, na, no, ny, nx, vp(dst), NP * dlo, dlo, NP, stream())
    torch.cuda.synchronize()
    v = gr.permute(0, 1, 4, 2, 3).reshape(b, na * no, ny, nx)              # channel a * no + k
    assert_planes(dst, dlo, v)
    for k in range(NP):
        assert float(dst[..., k * dlo + na * no:(k + 1) * dlo].float().abs().max()) == 0.0
    assert float(dst[:, 0].float().abs().max()) == 0.0


@pytest.mark.parametrize("bias", [False, True])
def test_px_to_nchw_bitwise(bias):
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(31)
    b, c, h, w, zcs = 2, 21, 19, 23, 64
    zb = torch.randn(b, h + 2, w + 2, zcs, generator=g).to(dev)
    bv = torch.randn(c, generator=g).to(dev) if bias else None
    out = torch.full((b, c, h, w), float("nan"), device=dev)
    px_call("ryolo_px_to_nchw", vp(zb), zcs, b, c, h, w, vp(bv), vp(out), stream())
    torch.cuda.synchronize()
    want = nchw(zb, c)
    if bias:
        want = want + bv[None, :, None, None]
    assert torch.equal(out.view(torch.int32), want.contiguous().view(torch.int32))


def test_px_im2col_first_bitwise():
    dev = torch.device("cuda")
    b, h, w = 2, 37, 29
    img = torch.randn(b, 3, h, w, generator=torch.Generator().manual_seed(41)).to(dev)
    col = torch.zeros((b, h + 2, w + 2, NP * 64), dtype=torch.bfloat16, device=dev)
    px_call("ryolo_px_im2col_first", vp(img), b, h, w, vp(col), NP * 64, 64, NP, stream())
    torch.cuda.synchronize()
    # column c * 9 + kh * 3 + kw, zero outside the image: F.unfold's order
    want = F.unfold(img, 3, padding=1).view(b, 27, h, w)
    assert_planes(col, 64, want)
    for k in range(NP):
        assert float(col[..., k * 64 + 27:(k + 1) * 64].float().abs().max()) == 0.0
    assert float(col[:, 0].float().abs().max()) == 0.0 and float(col[:, :, -1].float().abs().max()) == 0.0


def test_px_split_is_exact():
    """the three planes carry every fp32 value whose 24 bits lie above bf16's smallest subnormal 2^-133, i.e.
    |v| >= 2^-110: their sum, smallest first, is v bit for bit.  Below that the bits under 2^-133 are lost (the sum is
    within 2^-134 of v); ±0 come back as zeros (-0 as +0: the sum starts from +0)."""
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(51)
    e = torch.randint(-149, 100, (4096,), generator=g).double()
    mant = 1.0 + torch.rand(4096, generator=g, dtype=torch.float64)
    v = (mant * torch.pow(2.0, e)).float() * torch.sign(torch.randn(4096, generator=g))
    v = torch.cat([v, torch.tensor([0.0, -0.0, 1e30, -1e30, 2.0 ** -149, -(2.0 ** -149), 2.0 ** -126, 2.0 ** -110,
                                    1.4e-40, 3.0, 1.0 + 2.0 ** -23])]).float()
    x = v.view(1, -1, 1, 1).to(dev)
    c = x.shape[1]
    buf = split_buf(x, rup(c, 64))
    torch.cuda.synchronize()
    p = planes_of(buf, rup(c, 64), c)
    want = split3(x)
    for k in range(NP):
        assert torch.equal(p[k].view(torch.int16), want[k].view(torch.int16)), k
    back = merge3(*p)
    big = x.abs() >= 2.0 ** -110
    assert int(big.sum()) > 3000
    assert torch.equal(back[big].view(torch.int32), x[big].view(torch.int32))
    assert float((back[~big].double() - x[~big].double()).abs().max()) <= 2.0 ** -134
    zero = x == 0
    assert int(zero.sum()) == 2 and bool((back[zero] == 0).all())


# ---------------------------------------------------------------------------------------------------------------
# 6. the bounds bite
def test_bounds_reject_plausible_kernel_bugs():
    """Each check above, applied to a reference with one plausible bug put in, fails on the kernels' output."""
    # wgrad: one of the nine (dz plane, x plane) blocks dropped from the sum -- (a, b) = (2, 0)
    c = WgradCase(**dict(WGRAD_CASES["cout40"][0]), seed=len("cout40"))
    want = c.ref()
    got = c.unpack(c.run())
    torch.cuda.synchronize()
    assert within(measure(got, want))
    dz2 = split3(c.dz)[2].double()
    x0 = split3(c.x)[0].double()
    m = measure(got, want - c.ref_fn()(x0, dz2))
    print("[bite] wgrad without plane block (2, 0): %s" % fmt(m))
    assert not within(m), m
    # wgrad: one 64-pixel k-step lost (the first k-step of the second split)
    plan = c.plan()
    hp, wp = c.gh + 2, c.gw + 2
    flat = torch.zeros(c.b * hp * wp, dtype=torch.float64, device="cuda")
    j = plan["per_split"]
    flat[64 * j:64 * (j + 1)] = 1.0
    mask = flat.view(c.b, 1, hp, wp)[:, :, 1:-1, 1:-1]
    assert float(mask.sum()) >= 32
    m = measure(got, want - c.ref_fn()(c.x.double(), c.dz.double() * mask))
    print("[bite] wgrad without k-step %d: %s" % (j, fmt(m)))
    assert not within(m), m
    # dgrad: taps mirrored the wrong way
    kw = DGRAD_CASES["k3_128_64_152"]
    dz, wt = dgrad_inputs(**kw, seed=len("k3_128_64_152"))
    gb = f32_buf(kw["batch"], kw["h"], kw["w"], kw["cin"])
    run_dgrad(dz, wt, kw["h"], kw["w"], 1, gb, 0, 0)
    torch.cuda.synchronize()
    got = nchw(gb, kw["cin"])
    assert within(measure(got, ref_dgrad(dz, wt, kw["h"], kw["w"], 1)))
    m = measure(got, ref_dgrad(dz, wt.flip(2, 3), kw["h"], kw["w"], 1))
    print("[bite] dgrad with mirrored taps: %s" % fmt(m))
    assert not within(m), m
    # bn_act_bwd: the PReLU mask flipped on one element
    case = BnCase(**BN_CASES["c64_gres_acc"], seed=len("c64_gres_acc"))
    sums, dzb, _ = case.run()
    assert all(v <= 1.0 for v in bn_errors(case, sums, dzb, case.ref()).values())
    mk = case.mask().clone()
    i = int(case.d()[1, 5].abs().argmax())                  # the pixel of channel 5 with the largest |dy|
    y, x = divmod(i, case.w)
    mk[1, 5, y, x] = ~mk[1, 5, y, x]
    e = bn_errors(case, sums, dzb, case.ref(mk))
    print("[bite] bn_act_bwd with one PReLU mask bit flipped: %s" % e)
    assert max(e.values()) > 1.0, e
