"""Every kernel launch of the parity-precision training step and eval forward against float64 of the inputs it received.

ParityPlan (parity_path.py) runs each conv block as px_conv on split operands (three bf16 planes per fp32 value, plane k
of a view at channel ch_off + k * cs / 3) with fp32 element-wise kernels between the GEMMs.  test_parity_bwd_gpu.py runs
those kernels on buffers the test builds; here the plan's own launches are looked at, on the plan's own buffers: its
plane strides, concat slices, accumulate flags, the shared dz / dw scratch re-viewed per block, the head dz padding and
px_unpack_wgrad's cin_off on a whole-buffer wgrad.  rotate_yolov3_b200._lib.lib is swapped for a proxy whose
ryolo_px_* / ryolo_space_to_depth entries record the call, snapshot what it (or a later launch) overwrites, forward it
unchanged, synchronise and check its outputs against float64 of its inputs.  Three shapes, seeded init_darknet_weights, a
dense random cotangent G per head (loss = sum p * G), one training step, then one eval forward:

  bench  yolov3_cfg(), batch 2 x 608^2: the graph of the goldens and of bench's train_parity; GEMM tiles straddle images
  nc22   yolov3_cfg(classes=22, width=416, height=320), batch 3: 2016-filter heads (po 2048, a 6144-channel split dz,
         px_head_grad with no = 28, px_to_nchw with 2016 channels), an odd batch, h != w, grids 10x13 / 20x26 / 40x52
  tiny   yolov3_cfg(160 x 128, 6 anchors), batch 1: a 4 x 5 head grid (6 x 7 = 42 padded pixels, less than one 128-pixel
         GEMM tile), BatchNorm statistics over 20 pixels per channel

Bounds.  U = 2^-24.  A = the same operation in float64 on |operands|, the operands being the fp32 values the launch
received (a split buffer's operand is the exact sum of its three planes; weights the fp32 parameters); every ratio
|err| / bound must be <= 1, so a NaN fails.
  px_conv (forward z, head z, dgrad, the ksize -2 space-to-depth dgrad), K = terms x taps x channels of the launch,
  S = ceil(K / 512) accumulator segments of 8 k-steps (32 wgmma updates):
      |got - want| <= (2^-23 + 32 * 2^-23 + S * U) * (1 + 2^-7) A  [+ U |got| when it accumulates into a gradient]
      the three dropped plane products (i + j >= 3, <= 2^-25 A), the truncating accumulator inside each segment (one
      fp32 ulp of the segment's magnitude per update), one round-to-nearest add per segment, the fp32 add of the prior
      gradient; (1 + 2^-7) bounds the sum of the six |a_i w_j| terms by |a| |w|.  Forward reference: tapsum / conv_taps
      of test_train_step_f64_gpu on the real input (concat slice, im2col columns; stride 2 on the source view), dgrad:
      the mirrored taps / s2d_dgrad_ref; the channels of the gradient buffer outside the view must not change.
  px_wgrad + px_unpack_wgrad, wgrad_plan(..., segmented=True): per_split k-steps per split, ksplit splits:
      |got - want| <= (32 * 2^-23 + (ceil(per_split / 8) + ksplit + 9) U) (1 + 2^-7) A
      segments within each split, the round-to-nearest segment adds, the ksplit partials, the 9 plane-block adds of the
      unpack; the reference is wgrad_ref on the fp32 dz and x (the first layer on its im2col columns, stride-2 layers as
      the 3x3 / stride-2 weight gradient of the source view, concat slices at the view's channels).
  every GEMM launch, tensor-wide (test_parity_bwd_gpu): max |err| <= 5e-6 max |want|, rms(err) <= 2e-6 rms(want),
      |mean(err sign(want))| <= 1e-6 rms(want) -- the bias bound is the one an unsegmented accumulator fails.
  px_bn_stats: the fp64 sums within 2 n 2^-53 sum |terms|.  px_bn_finalize: mean within 2 fp32 ulps + n 2^-53 mean |z|,
      invstd = 1 / sqrtf((float) var + eps) within 3 U invstd of the two-pass float64 value (+ the one-pass fp64
      variance's n 2^-53 E[z^2] / var), scale = gamma * invstd bit for bit, shift within 2 U of its terms, running mean
      / variance (momentum, unbiased variance) within 4 U of their terms; eval mode: mean = running mean bit for bit,
      invstd within 2.5 U (one rounding fewer), nothing written back.  test_parity_bwd_gpu holds invstd to 2 fp32 ulps;
      that is not implied by the four roundings (IEEE fp32 restated on the host reaches 2.26 ulps on 2e6 random
      variances, 6e-5 of them above 2), and the step's BN channels reach it: 2.2 ulps on the 20- to 320-pixel channels
      of `tiny`.
  px_bn_act_fwd, px_to_nchw, px_head_grad, px_im2col_first, ryolo_space_to_depth (each plane), px_depth_to_space (plain
      and accumulating), the shortcut gradient of px_bn_act_bwd: bit for bit against a torch fp32 emulation on the
      plan's own buffers, the split p0 = bf16(v), p1 = bf16(v - p0), p2 = bf16(v - p0 - p1) at ch_off + k cs / 3; halos
      and padding channels zero (head dz channels [na no, po) of every plane included).  Whether a gradient write
      accumulates is decided by the test from the writes it saw earlier in the backward, not by the plan's flag.
  px_bn_act_bwd: bn_errors / DZ_ULPS of test_parity_bwd_gpu (PReLU branch from the kernel's own fp32 u).
  head bias gradient (float64 sum in ParityPlan.backward): within U |want| + n 2^-53 sum |G|.
  weight .grad equals the px_unpack_wgrad output bit for bit (the test reruns the unpack on the same dw).

test_covers_every_launch compares, per shape and pass, the recorded launches by entry point and block with the checked
ones (ryolo_px_pack_weights is checked through the px_conv that consumes it: that check uses the fp32 parameter).
test_bounds_reject_plausible_bugs puts eight bugs into stored tensors or references and requires each check to fail.

Measured on an H100 80GB HBM3 (132 SMs, power limit 700 W, 1980 MHz max SM clock), seeds as below.  `pytest -s` prints
one line per block (each launch kind's worst ratio, the signed bias / rms of its GEMMs) and a per-kind summary.  Worst
ratio over the blocks, bench / nc22 / tiny, training step (eval forward where it differs):
  px_conv z      element 0.092 / 0.076 / 0.073; max 0.18 (eval 0.24) / 0.20 (0.23) / 0.16 (0.20); rms <= 0.32; bias <= 0.44
  head z         element <= 0.087; max <= 0.18; rms <= 0.31 (tiny eval 0.38); bias <= 0.42 (tiny eval 0.49)
  dgrad          element 0.095 / 0.087 / 0.078; max <= 0.19; rms <= 0.31; bias <= 0.42
  wgrad+unpack   element 0.082 / 0.119 / 0.091; max <= 0.19; rms <= 0.40; bias <= 0.40
  bn_act_bwd     dz 0.32 / 0.30 / 0.27; d beta <= 0.010; d gamma <= 0.067; d slope < 1e-9
  BN statistics  sums <= 0.13; mean 0.25; invstd 0.67 / 0.70 / 0.75 (1.85 / 1.93 / 2.20 fp32 ulps), eval 0.64;
                 running mean 0.55, running variance 0.38, shift 0.50
  head bias      0.96 / 0.98 / 0.93
  bit for bit    every layout kernel and split, every padding channel and halo, .grad = the unpack output
Every GEMM's bias is negative, -8e-9 .. -4.9e-7 of rms (test_parity_bwd_gpu measures -2.3e-7 .. -3.4e-7 on random
operands): what the 32-update segments leave of the accumulator's round-toward-zero.  A training step is 763 launches
over 605 (entry point, block) pairs and an eval forward 313 over 303, all checked.  Parity training runs at nc = 22, at
batch 3 and at batch 1 on a 4 x 5 grid; no kernel or plan needed a change.  Bugs put in, worst ratio: x from two planes
1.27 (rms; dropping plane 2 is noise of 2^-17 relative, under the element bound); one lost 512-deep segment 1.7e5;
ryolo_conv_wgrad on the same planes (block 3, 1676 updates per chain) bias 20; a dgrad that overwrites 4.6e5; cin_off +
64 7.6e5; plane 1 of a concat slice read at the slice's rounded width instead of cs / 3: 990; a nonzero head dz padding
channel fails its bitwise check; a biased running variance 2.9e3, failing on 71 of the 72 BN blocks.  Whole file: 15-17 s
(7-8 s for the three shapes' steps and checks)."""
import ctypes
import math
import time
import traceback
from collections import Counter

import pytest
import torch
import torch.nn.functional as F

from builders import pkg
from f64_refs import (BF16, NP, PX_BIAS_TOL, PX_MAX_TOL, PX_RMS_TOL, TINY, U, BnCase, _shift, bitwise, bn_errors, cdiv,
                      conv_taps, d2s, gemm_sms, halo_zero, interior, measure, merge3, rup, s2d, s2d_dgrad_ref, split3,
                      tapsum, ulps_f32, wgrad_ref)
from helpers import SMALL_ANCHORS, init_darknet_weights, wgrad_plan

pytestmark = pytest.mark.gpu

U64 = 2.0 ** -53
SEG_UPDATES = 32              # wgmma k16 updates between two accumulator restarts (8 k-steps of 64)
SEG_K = 512                   # GEMM K per accumulator segment
TERMS = 1.0 + 2.0 ** -7       # sum of |a_i w_j| over the plane products, relative to |a| |w|
INV_TRAIN = 3.0               # invstd = 1 / sqrtf((float) var + eps): four fp32 roundings, the sqrt halves two of them
INV_EVAL = 2.5                # the running variance is fp32 already: three roundings
SHAPES = {
    "bench": (dict(), 2, 608, 608),
    "nc22": (dict(classes=22, width=416, height=320), 3, 320, 416),
    "tiny": (dict(width=160, height=128, classes=1, anchors=SMALL_ANCHORS, n_anchors=6), 1, 128, 160),
}
ENTRY = "ryolo_px_"
EXTRA_ENTRIES = ("ryolo_space_to_depth",)
NOT_LAUNCHES = ("ryolo_px_packed_weight_bytes",)


def plane_views(buf, lo, off, c):
    """interior [B, H, W, c] of the three planes of channels [off, off + c), plane k at off + k * lo"""
    return [interior(buf, off + k * lo, c) for k in range(NP)]


def merged(buf, lo, off, c):
    return merge3(*plane_views(buf, lo, off, c))


def lo_of(view):
    return view.cs // NP


def view_val(view):
    """the fp32 activation a split view carries"""
    return merged(view.buf, lo_of(view), view.ch_off, view.c)


def split_equal(planes, v):
    want = split3(v.contiguous())
    return all(torch.equal(p.contiguous().view(torch.int16), w.view(torch.int16)) for p, w in zip(planes, want))


def f32_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def planes_pad_zero(buf, lo, c):
    return all(bool((buf[..., k * lo + c:(k + 1) * lo] == 0).all()) for k in range(NP))


def worse(a, b):
    if a != a:
        return a
    return b if (b != b or b > a) else a


def failures(r):
    """keys of r that fail: a float ratio above 1 (or NaN), a False flag; keys starting with '_' are information"""
    return [k for k, v in r.items() if not k.startswith("_")
            and ((isinstance(v, bool) and not v) or (isinstance(v, float) and not v <= 1.0))]


# ---------------------------------------------------------------------------------------------------------------
# bounds
def conv_e(mag, k):
    """px_conv, GEMM depth K = k: dropped plane products, truncation inside each segment, one RN add per segment"""
    return (2.0 ** -23 + SEG_UPDATES * 2.0 ** -23 + cdiv(k, SEG_K) * U) * TERMS * mag


def wgrad_e(mag, pw):
    return (SEG_UPDATES * 2.0 ** -23 + (cdiv(pw["per_split"], 8) + pw["ksplit"] + NP * NP) * U) * TERMS * mag


def gemm_check(got, want, e):
    """element bound |got - want| <= e and the tensor-wide bounds of test_parity_bwd_gpu, as ratios (<= 1 passes)"""
    err = (got.double() - want).abs()
    m = measure(got, want)
    return {"elem": float((err / (e + TINY)).max()), "max": m["max"] / PX_MAX_TOL, "rms": m["rms"] / PX_RMS_TOL,
            "bias": abs(m["bias"]) / PX_BIAS_TOL, "_bias": m["bias"]}


def ulps(x):
    return ulps_f32(x)


def wgrad_s2(x, dz):
    """float64 weight gradient of the 3x3 / stride-2 / pad-1 conv: x [B, h, w, cin] (source grid), dz [B, h/2, w/2, cout];
    value and magnitude as [cout, cin, 3, 3]"""
    b, oh, ow, cout = dz.shape
    cin = x.shape[3]
    xp = F.pad(x.double(), (0, 0, 1, 1, 1, 1))
    d = dz.double().reshape(-1, cout)
    outs, mags = [], []
    for kh in range(3):
        for kw in range(3):
            a = _shift(xp, kh - 1, kw - 1, oh, ow, 2).reshape(-1, cin)
            outs.append(d.t() @ a)
            mags.append(d.abs().t() @ a.abs())
    return (torch.stack(outs).view(3, 3, cout, cin).permute(2, 3, 0, 1),
            torch.stack(mags).view(3, 3, cout, cin).permute(2, 3, 0, 1))


def unpack_emul(dw, po, pi, cout, cin, ks, off):
    """px_unpack_wgrad mode 0 in torch fp32, the kernel's order (plane-index sum from large to small); channels past the
    end of a dw row read as 0"""
    taps = ks * ks
    d = dw.reshape(taps, NP * po, NP * pi)
    s = torch.zeros((cout, cin, taps), dtype=torch.float32, device=dw.device)
    for order in range(2 * (NP - 1), -1, -1):
        for a in range(NP - 1, -1, -1):
            b = order - a
            if not 0 <= b < NP:
                continue
            part = d[:, a * po:a * po + cout, b * pi + off:b * pi + off + cin]
            if part.shape[2] < cin:
                part = F.pad(part, (0, cin - part.shape[2]))
            s = s + part.permute(1, 2, 0)
    return s.view(cout, cin, ks, ks)


class PlanBn(BnCase):
    """f64_refs.BnCase (test_parity_bwd_gpu) on a plan block's own tensors (z and dy fp32 NHWC, as the kernel read them)"""

    def __init__(self, z, d, mean, invstd, scale, shift, slope, po):
        self.z, self._d = z.permute(0, 3, 1, 2), d.permute(0, 3, 1, 2)
        self.c, self.po = z.shape[-1], po
        self.b, self.h, self.w = z.shape[0], z.shape[1], z.shape[2]
        self.act, self.up, self.bs, self.gres_mode = slope is not None, False, 1, None
        self.mean, self.invstd, self.scale, self.shift, self.slope = mean, invstd, scale, shift, slope

    def d(self):
        return self._d


# ---------------------------------------------------------------------------------------------------------------
class Run:
    """one checked pass (the training step or the eval forward) of one model; launch() is what the proxy calls"""

    def __init__(self, shape, phase, model, x, real, stash=False):
        self.shape, self.phase, self.model, self.x, self.real, self.want_stash = shape, phase, model, x, real, stash
        self.calls, self.checked, self.pending = Counter(), Counter(), Counter()
        self.res, self.errors, self.stash = {}, [], {}
        self.plan, self.cur, self.G = None, None, None
        self.written, self.wg, self.gw, self.rv_biased = {}, {}, {}, {}

    # ---- bookkeeping
    def put(self, kind, i, r):
        d = self.res.setdefault((kind, i), {})
        for k, v in r.items():
            if isinstance(v, bool):
                d[k] = d.get(k, True) and v
            elif isinstance(v, float):
                d[k] = worse(d[k], v) if k in d else v
            else:
                d[k] = v

    def _maps(self):
        plan = self.model._pplan
        if plan is not self.plan:
            self.plan = plan
            ml = self.model.module_list
            self.by_z = {b.z.data_ptr(): b for b in plan.blocks}
            self.by_w = {ml[b.i].Conv2d.weight.data_ptr(): b for b in plan.blocks}
            self.by_mean = {b.mean.data_ptr(): b for b in plan.blocks if not b.is_head}
            self.by_hdz = {b.dz.data_ptr(): b for b in plan.heads} if plan.train else {}
            self.by_dxs = {b.dxs.data_ptr(): b for b in plan.blocks if b.s2d} if plan.train else {}
            self.xs = [(b.xs.data_ptr(), b) for b in plan.blocks if b.s2d]
        return plan

    def block(self, name, a):
        plan = self._maps()
        if name == "ryolo_px_im2col_first":
            return plan.blocks[0]
        if name == "ryolo_space_to_depth":
            return next(b for p, b in self.xs if p <= a[6] < p + 2 * NP * b.p4)
        if name == "ryolo_px_pack_weights":
            return self.by_w[a[0]]
        if name == "ryolo_px_conv":
            return self.by_z.get(a[13], self.cur)
        if name in ("ryolo_px_to_nchw", "ryolo_px_bn_stats", "ryolo_px_bn_act_fwd"):
            return self.by_z[a[0]]
        if name == "ryolo_px_bn_finalize":
            return self.by_mean[a[8]]
        if name == "ryolo_px_head_grad":
            return self.by_hdz[a[6]]
        if name == "ryolo_px_bn_act_bwd":
            self.cur = self.by_z[a[3]]
            return self.cur
        if name == "ryolo_px_wgrad":
            if a[0] in self.by_hdz:
                self.cur = self.by_hdz[a[0]]
            return self.cur
        if name == "ryolo_px_unpack_wgrad":
            return self.cur
        if name == "ryolo_px_depth_to_space":
            return self.by_dxs[a[0]]
        return None

    def launch(self, name, fn, args):
        a = [v.value if isinstance(v, ctypes.c_void_p) else v for v in args]
        try:
            blk = self.block(name, a)
        except Exception:
            blk = None
            self.errors.append(((name, None), traceback.format_exc()))
        key = (name, blk.i if blk is not None else None)
        self.calls[key] += 1
        h = HANDLERS.get(name)
        snap = {}
        if h is not None and blk is not None and h[0] is not None:
            try:
                snap = h[0](self, blk, a)
            except Exception:
                self.errors.append((key, traceback.format_exc()))
                h = None
        st = fn(*args)
        if st != 0 or h is None or blk is None:
            return st
        torch.cuda.synchronize()
        try:
            if h[1](self, blk, a, snap):
                self.checked[key] += 1
        except Exception:
            self.errors.append((key, traceback.format_exc()))
        return st

    # ---- gradient-write bookkeeping: a write accumulates when earlier writes of this backward cover its channels
    def expect_acc(self, view):
        lo, hi = view.ch_off, view.ch_off + view.c
        return any(a <= lo and hi <= b for a, b in self.written.get(id(view.buf), []))

    def wrote(self, view):
        self.written.setdefault(id(view.buf), []).append((view.ch_off, view.ch_off + view.c))

    def weight(self, blk):
        return self.model.module_list[blk.i].Conv2d.weight.detach()


class Proxy:
    """stands in for the ctypes library: the parity entry points go through Run.launch, everything else is the library's"""

    def __init__(self, real, run):
        self._real, self._run = real, run

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if (name.startswith(ENTRY) or name in EXTRA_ENTRIES) and name not in NOT_LAUNCHES:
            run = self._run
            return lambda *args: run.launch(name, fn, args)
        return fn


# ---------------------------------------------------------------------------------------------------------------
# handlers: (pre -> snapshot or None, post -> True when the launch is checked)
def _im2col(run, blk, a, snap):
    plan, x = run.plan, run.x
    assert a[0] == x.data_ptr()
    b, _, h, w = x.shape
    want = F.unfold(x, 3, padding=1).view(b, 27, h, w).permute(0, 2, 3, 1)
    run.put("im2col", 0, {"bits": split_equal(plane_views(plan.col, 64, 0, 27), want),
                          "pad_zero": planes_pad_zero(plan.col, 64, 27), "halo": halo_zero(plan.col)})
    return True


def _s2d(run, blk, a, snap):
    k = (a[6] - blk.xs.data_ptr()) // (2 * blk.p4)
    src, c4 = blk.src, 4 * blk.cin
    sp = interior(src.buf, src.ch_off + k * lo_of(src), src.c)
    got = interior(blk.xs, k * blk.p4, c4)
    run.put("s2d", blk.i, {"bits": bitwise(got, s2d(sp)),
                           "pad_zero": bool((blk.xs[..., k * blk.p4 + c4:(k + 1) * blk.p4] == 0).all()),
                           "halo": halo_zero(blk.xs)})
    return True


def _pack(run, blk, a, snap):
    run.pending[(blk.i, "dgrad" if a[6] in (1, 3) else "fwd")] += 1
    return False


def _conv_fwd(run, blk, a):
    plan = run.plan
    w64 = run.weight(blk).double()
    if blk.i == 0:
        x = merged(plan.col, 64, 0, 27)
        want, mag = tapsum(x, [(0, 0, w64.reshape(blk.cout, 27).t())], blk.oh, blk.ow)
    else:
        want, mag = tapsum(view_val(blk.src), conv_taps(w64), blk.oh, blk.ow, blk.stride)
    k = a[6] * a[11] * a[11] * rup(a[4], 64)
    got = interior(blk.z, 0, blk.cout)
    r = gemm_check(got, want, conv_e(mag, k))
    r["pad_zero"] = bool((blk.z[..., blk.cout:] == 0).all()) and halo_zero(blk.z)
    run.put("head_z" if blk.is_head else "z", blk.i, r)


def _conv_dgrad(run, blk, a, snap):
    w64 = run.weight(blk).double()
    dz = merged(blk.dz, blk.po, 0, blk.cout)
    k = a[6] * a[11] * a[11] * rup(a[4], 64)
    src, gs = blk.src, blk.gsrc
    if blk.s2d:
        want, mag = s2d_dgrad_ref(dz, w64, src.h, src.w)
        c4 = 4 * blk.cin
        r = gemm_check(interior(blk.dxs, 0, c4), want, conv_e(mag, k))
        r["pad_zero"] = bool((blk.dxs[..., c4:] == 0).all()) and halo_zero(blk.dxs)
        run.put("dgrad", blk.i, r)
        return
    want, mag = tapsum(dz, conv_taps(w64, mirror=True), src.h, src.w)
    e = conv_e(mag, k)
    got = interior(gs.buf, gs.ch_off, gs.c)
    prior = interior(snap["gbuf"], gs.ch_off, gs.c)
    acc = run.expect_acc(gs)
    if run.want_stash and acc and "overwrite" not in run.stash and src.h * src.w <= 40 * 40:
        run.stash["overwrite"] = dict(i=blk.i, got=got.clone(), want=want.clone(), e=e.clone())
    if acc:
        want = want + prior.double()
        e = e + U * got.double().abs()
    r = gemm_check(got, want, e)
    r["acc_flag"] = bool(a[16]) == acc
    r["_acc"] = float(acc)
    allowed = torch.zeros(gs.cs, dtype=torch.bool, device=got.device)
    allowed[gs.ch_off:gs.ch_off + gs.c] = True
    r["outside"] = torch.equal(gs.buf[..., ~allowed], snap["gbuf"][..., ~allowed]) and halo_zero(gs.buf)
    run.wrote(gs)
    run.put("dgrad", blk.i, r)


def _conv_pre(run, blk, a):
    if a[13] == blk.z.data_ptr() or blk.s2d:
        return {}
    return {"gbuf": blk.gsrc.buf.clone()}


def _conv(run, blk, a, snap):
    if a[13] == blk.z.data_ptr():
        _conv_fwd(run, blk, a)
        which = "fwd"
    else:
        assert a[0] == blk.dz.data_ptr()
        _conv_dgrad(run, blk, a, snap)
        which = "dgrad"
    run.checked[("ryolo_px_pack_weights", blk.i)] += run.pending.pop((blk.i, which), 0)
    return True


def _to_nchw(run, blk, a, snap):
    bias = run.model.module_list[blk.i].Conv2d.bias
    want = interior(blk.z, 0, blk.cout).permute(0, 3, 1, 2)
    if bias is not None:
        want = want + bias.detach()[None, :, None, None]
    run.put("to_nchw", blk.i, {"bits": f32_equal(blk.out, want)})
    return True


def _bn_stats(run, blk, a, snap):
    c = blk.cout
    z = interior(blk.z, 0, c).reshape(-1, c).double()
    n = z.shape[0]
    s1, s2 = blk.sums[:c], blk.sums[c:2 * c]
    r1 = ((s1 - z.sum(0)).abs() / (2 * n * U64 * z.abs().sum(0) + TINY)).max()
    r2 = ((s2 - z.pow(2).sum(0)).abs() / (2 * n * U64 * z.pow(2).sum(0) + TINY)).max()
    run.put("bn_stats", blk.i, {"sums": float(max(r1, r2))})
    return True


def _bn_fin_pre(run, blk, a):
    bn = run.model.module_list[blk.i].BatchNorm2d
    return {"rm": bn.running_mean.clone(), "rv": bn.running_var.clone()}


def _bn_fin(run, blk, a, snap):
    bn = run.model.module_list[blk.i].BatchNorm2d
    c = blk.cout
    gamma, beta = bn.weight.detach(), bn.bias.detach()
    eps = float(torch.tensor(bn.eps, dtype=torch.float32))
    mom = float(torch.tensor(bn.momentum, dtype=torch.float32))
    rm0, rv0 = snap["rm"].double(), snap["rv"].double()
    r = {"scale_bits": f32_equal(blk.scale, gamma * blk.invstd)}
    sh_want = beta.double() - blk.mean.double() * blk.scale.double()
    r["shift"] = float(((blk.shift.double() - sh_want).abs()
                        / (2 * U * (beta.double().abs() + (blk.mean.double() * blk.scale.double()).abs()) + TINY)).max())
    if a[7]:                                        # eval: the running statistics
        want_inv = 1.0 / (rv0 + eps).sqrt()
        r["mean_bits"] = f32_equal(blk.mean, snap["rm"])
        r["invstd"] = float(((blk.invstd.double() - want_inv).abs() / (INV_EVAL * U * want_inv)).max())
        r["running_kept"] = f32_equal(bn.running_mean, snap["rm"]) and f32_equal(bn.running_var, snap["rv"])
        run.put("bn_finalize_eval", blk.i, r)
        return True
    z = interior(blk.z, 0, c).reshape(-1, c).double()
    n = z.shape[0]
    m64 = z.mean(0)
    v64 = (z - m64).pow(2).mean(0)
    q = z.pow(2).mean(0)
    want_inv = 1.0 / (v64 + eps).sqrt()
    r["mean"] = float(((blk.mean.double() - m64).abs() / (2 * ulps(m64) + n * U64 * z.abs().mean(0) + TINY)).max())
    err_inv = (blk.invstd.double() - want_inv).abs()
    r["invstd"] = float((err_inv / (INV_TRAIN * U * want_inv + want_inv * n * U64 * q / (v64 + eps))).max())
    r["_invstd_ulps"] = float((err_inv / ulps(want_inv)).max())
    corr = n / (n - 1)
    rm_w = (1 - mom) * rm0 + mom * m64
    tol_m = 4 * U * ((1 - mom) * rm0.abs() + mom * m64.abs()) + mom * (2 * ulps(m64) + n * U64 * z.abs().mean(0)) + TINY
    r["running_mean"] = float(((bn.running_mean.double() - rm_w).abs() / tol_m).max())

    def rv_ratio(cf):
        rv_w = (1 - mom) * rv0 + mom * v64 * cf
        tol_v = 4 * U * ((1 - mom) * rv0.abs() + mom * v64 * cf) + mom * cf * n * U64 * q + 1e-12
        return float(((bn.running_var.double() - rv_w).abs() / tol_v).max())
    r["running_var"] = rv_ratio(corr)
    run.rv_biased[blk.i] = rv_ratio(1.0)
    run.put("bn_finalize", blk.i, r)
    return True


def _bn_act_fwd(run, blk, a, snap):
    seq = run.model.module_list[blk.i]
    z = interior(blk.z, 0, blk.cout)
    u = (z * blk.scale) + blk.shift
    if blk.has_act:
        slope = seq.activation.weight.detach()
        u = torch.where(u > 0, u, slope * u)
    if blk.res is not None:
        u = u + view_val(blk.res)
    y = blk.y
    pl = plane_views(y.buf, lo_of(y), y.ch_off, y.c)
    if blk.fuse_up:
        ok = all(split_equal([p[:, ry::2, rx::2] for p in pl], u) for ry in range(2) for rx in range(2))
    else:
        ok = split_equal(pl, u)
    run.put("bn_act_fwd", blk.i, {"bits": ok})
    return True


def _head_grad(run, blk, a, snap):
    g = run.G[blk.i]
    b, na, ny, nx, no = g.shape
    v = g.permute(0, 2, 3, 1, 4).reshape(b, ny, nx, na * no)
    run.put("head_grad", blk.i, {"bits": split_equal(plane_views(blk.dz, blk.po, 0, na * no), v),
                                 "pad_zero": planes_pad_zero(blk.dz, blk.po, na * no) and halo_zero(blk.dz)})
    return True


def _bn_bwd_pre(run, blk, a):
    return {"gres": blk.gres.buf.clone()} if blk.gres is not None else {}


def _bn_bwd(run, blk, a, snap):
    seq = run.model.module_list[blk.i]
    c = blk.cout
    z = interior(blk.z, 0, c)
    g = interior(blk.gy.buf, blk.gy.ch_off, c)
    if blk.fuse_up:
        d = torch.zeros_like(g[:, ::2, ::2])
        for ry in range(2):
            for rx in range(2):
                d = d + g[:, ry::2, rx::2]
    else:
        d = g
    slope = seq.activation.weight.detach() if blk.has_act else None
    case = PlanBn(z, d, blk.mean, blk.invstd, blk.scale, blk.shift, slope, blk.po)
    r = bn_errors(case, blk.bsums, blk.dz, case.ref())
    r["dz_pad_zero"] = planes_pad_zero(blk.dz, blk.po, c) and halo_zero(blk.dz)
    if blk.gres is not None:
        gr = blk.gres
        prior = interior(snap["gres"], gr.ch_off, c)
        acc = run.expect_acc(gr)
        r["gres_bits"] = f32_equal(interior(gr.buf, gr.ch_off, c), prior + d if acc else d)
        r["gres_flag"] = bool(a[21]) == acc
        allowed = torch.zeros(gr.cs, dtype=torch.bool, device=z.device)
        allowed[gr.ch_off:gr.ch_off + c] = True
        r["gres_outside"] = torch.equal(gr.buf[..., ~allowed], snap["gres"][..., ~allowed]) and halo_zero(gr.buf)
        run.wrote(gr)
    run.put("bn_act_bwd", blk.i, r)
    return True


def _wgrad(run, blk, a, snap):
    run.wg[blk.i] = list(a)
    return False                                    # checked with its unpack


def _unpack(run, blk, a, snap):
    plan = run.plan
    aw = run.wg.pop(blk.i)
    w = run.weight(blk)
    mine = torch.full(tuple(w.shape), float("nan"), dtype=torch.float32, device=w.device)
    args = list(a)
    args[9] = mine.data_ptr()                       # the same launch into a tensor of the test's own
    assert run.real.ryolo_px_unpack_wgrad(*args) == 0
    torch.cuda.synchronize()
    run.gw[blk.i] = mine
    dz = merged(blk.dz, blk.po, 0, blk.cout)
    if blk.i == 0:
        wr, wm = wgrad_ref(merged(plan.col, 64, 0, 27), dz, [(0, 0)])
        want, mag = wr[0].reshape(w.shape), wm[0].reshape(w.shape)
    elif blk.s2d:
        want, mag = wgrad_s2(view_val(blk.src), dz)
    else:
        p = (blk.k - 1) // 2
        offs = [(kh - p, kw - p) for kh in range(blk.k) for kw in range(blk.k)]
        wr, wm = wgrad_ref(view_val(blk.src), dz, offs)
        want = wr.reshape(blk.k, blk.k, blk.cout, blk.cin).permute(2, 3, 0, 1)
        mag = wm.reshape(blk.k, blk.k, blk.cout, blk.cin).permute(2, 3, 0, 1)
    pw = wgrad_plan(aw[9], aw[5], aw[2], aw[6], aw[7], aw[8], gemm_sms(), segmented=True)
    e = wgrad_e(mag, pw)
    r = gemm_check(mine, want, e)
    r["operands"] = aw[0] == blk.dz.data_ptr() and aw[3] == blk.xw_buf.data_ptr() and aw[10] == blk.dw.data_ptr()
    r["_ksplit"], r["_per_split"] = float(pw["ksplit"]), float(pw["per_split"])
    run.put("wgrad", blk.i, r)
    if run.want_stash:
        old = wgrad_plan(aw[9], aw[5], aw[2], aw[6], aw[7], aw[8], gemm_sms())
        best = run.stash.get("conv_wgrad")
        if blk.i > 0 and (best is None or old["updates"] > best["updates"]):
            run.stash["conv_wgrad"] = dict(i=blk.i, updates=old["updates"], dz=blk.dz.clone(), aw=aw, ua=list(a),
                                           want=want.clone(), shape=tuple(w.shape))
        if (blk.k == 1 and not blk.s2d and not blk.is_head and blk.i > 0
                and ("unpack" not in run.stash or blk.cin > run.stash["unpack"]["cin"])):
            run.stash["unpack"] = dict(i=blk.i, cin=blk.cin, dw=blk.dw.clone(), ua=list(a), want=want.clone(),
                                       e=e.clone(), mine=mine.clone())
    run.checked[("ryolo_px_wgrad", blk.i)] += 1
    return True


def _d2s_pre(run, blk, a):
    return {"gbuf": blk.gsrc.buf.clone()}


def _d2s(run, blk, a, snap):
    gs = blk.gsrc
    v = d2s(interior(blk.dxs, 0, 4 * blk.cin), blk.cin)
    acc = run.expect_acc(gs)
    prior = interior(snap["gbuf"], gs.ch_off, gs.c)
    r = {"bits": f32_equal(interior(gs.buf, gs.ch_off, gs.c), prior + v if acc else v), "acc_flag": bool(a[8]) == acc}
    allowed = torch.zeros(gs.cs, dtype=torch.bool, device=v.device)
    allowed[gs.ch_off:gs.ch_off + gs.c] = True
    r["outside"] = torch.equal(gs.buf[..., ~allowed], snap["gbuf"][..., ~allowed]) and halo_zero(gs.buf)
    run.wrote(gs)
    run.put("d2s", blk.i, r)
    return True


HANDLERS = {
    "ryolo_px_im2col_first": (None, _im2col),
    "ryolo_space_to_depth": (None, _s2d),
    "ryolo_px_pack_weights": (None, _pack),
    "ryolo_px_conv": (_conv_pre, _conv),
    "ryolo_px_to_nchw": (None, _to_nchw),
    "ryolo_px_bn_stats": (None, _bn_stats),
    "ryolo_px_bn_finalize": (_bn_fin_pre, _bn_fin),
    "ryolo_px_bn_act_fwd": (None, _bn_act_fwd),
    "ryolo_px_head_grad": (None, _head_grad),
    "ryolo_px_bn_act_bwd": (_bn_bwd_pre, _bn_bwd),
    "ryolo_px_wgrad": (None, _wgrad),
    "ryolo_px_unpack_wgrad": (None, _unpack),
    "ryolo_px_depth_to_space": (_d2s_pre, _d2s),
}


def buffer_checks(run):
    """after a forward: every activation buffer's halo and the padding channels of every plane zero"""
    plan = run.plan
    real = {}
    for b in plan.blocks:
        for v in (b.src, None if b.is_head else b.y, b.res):
            if v is not None and v.buf is not None and v.buf.dtype == BF16:
                real[id(v.buf)] = (v.buf, max(real.get(id(v.buf), (None, 0))[1], v.ch_off + v.c))
    ok = all(halo_zero(buf) and planes_pad_zero(buf, buf.shape[-1] // NP, c) for buf, c in real.values())
    run.put("buffers", None, {"halo_and_pad": ok})


# ---------------------------------------------------------------------------------------------------------------
def make_model(kw, seed):
    from rotate_yolov3_b200 import cfgs
    m = pkg().Darknet(cfgs.yolov3_cfg(**kw), {"context_factor": 1.0}, arc="default", precision="parity")
    return init_darknet_weights(m, seed=seed)


def run_shape(name):
    import rotate_yolov3_b200 as pkg
    kw, batch, h, w = SHAPES[name]
    dev = torch.device("cuda")
    t0 = time.time()
    model = make_model(kw, seed=11).to(dev).train()
    x = torch.rand(batch, 3, h, w, generator=torch.Generator().manual_seed(12)).to(dev)
    real = pkg._lib.lib
    tr = Run(name, "train", model, x, real, stash=name == "bench")
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(pkg._lib, "lib", Proxy(real, tr))
        ps = model(x)
        torch.cuda.synchronize()
        buffer_checks(tr)
        gen = torch.Generator().manual_seed(13)
        gs = [torch.randn(p.shape, generator=gen).to(dev) for p in ps]
        tr.G = {b.i: g for b, g in zip(tr.plan.heads, gs)}
        loss = sum((p * g).sum() for p, g in zip(ps, gs))
        loss.backward()
        torch.cuda.synchronize()
    # after the step: head bias sums, .grad == the unpack output
    for b in tr.plan.blocks:
        seq = model.module_list[b.i]
        r = {"grad_bits": f32_equal(seq.Conv2d.weight.grad, tr.gw[b.i]) if b.i in tr.gw else False}
        if b.is_head:
            g = tr.G[b.i].double()
            want = g.sum((0, 2, 3)).reshape(-1)
            mag = g.abs().sum((0, 2, 3)).reshape(-1)
            n = g.shape[0] * g.shape[2] * g.shape[3]
            r["head_bias"] = float(((seq.Conv2d.bias.grad.double() - want).abs()
                                    / (U * want.abs() + n * U64 * mag + TINY)).max())
        tr.put("param_grad", b.i, r)
    tr.seconds = time.time() - t0
    # eval forward on the updated running statistics
    t1 = time.time()
    model.eval()
    ev = Run(name, "eval", model, x, real)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(pkg._lib, "lib", Proxy(real, ev))
        with torch.no_grad():
            model(x)
        torch.cuda.synchronize()
        buffer_checks(ev)
    ev.seconds = time.time() - t1
    for run in (tr, ev):
        _print_table(run)
    return tr, ev


KINDS = ("im2col", "s2d", "z", "head_z", "to_nchw", "bn_stats", "bn_finalize", "bn_finalize_eval", "bn_act_fwd",
         "head_grad", "bn_act_bwd", "wgrad", "dgrad", "d2s", "param_grad")


def worst(r):
    """worst ratio of a result (flags: 0 when true, inf when false)"""
    v = 0.0
    for k, x in r.items():
        if k.startswith("_"):
            continue
        if isinstance(x, bool):
            v = worse(v, 0.0 if x else math.inf)
        elif isinstance(x, float):
            v = worse(v, x)
    return v


def _print_table(run):
    print("\n[parity %s %s] %.1f s; worst |err| / bound per launch kind (flags: 0 = holds)" % (run.shape, run.phase,
                                                                                           run.seconds))
    for b in run.plan.blocks:
        cols = ["%-8s" % ("head" if b.is_head else ("s2d" if b.s2d else "k%d" % b.k)), "%4d" % b.cout,
                "%3dx%-3d" % (b.oh, b.ow)]
        for kind in KINDS:
            r = run.res.get((kind, b.i))
            if r is not None:
                cols.append("%s %.3f" % (kind, worst(r)))
                if kind in ("z", "head_z", "wgrad", "dgrad") and "_bias" in r:
                    cols.append("(bias %+.1e)" % r["_bias"])
        print("[parity %s %s] %3d %s" % (run.shape, run.phase, b.i, "  ".join(cols)))
    summ = {}
    for (kind, i), r in run.res.items():
        for k, v in r.items():
            if isinstance(v, float) and not k.startswith("_"):
                cur = summ.get((kind, k))
                if cur is None or v != v or v > cur[0]:
                    summ[(kind, k)] = (v, i)
    for (kind, k), (v, i) in sorted(summ.items()):
        print("[parity %s %s] summary %-16s %-14s %.3g (block %s)" % (run.shape, run.phase, kind, k, v, i))


@pytest.fixture(scope="module")
def runs():
    t0 = time.time()
    out = {name: run_shape(name) for name in SHAPES}
    print("[parity] all shapes %.1f s" % (time.time() - t0))
    return out


# ---------------------------------------------------------------------------------------------------------------
def test_covers_every_launch(runs):
    for name, (tr, ev) in runs.items():
        for run in (tr, ev):
            assert not run.errors, (name, run.phase, run.errors[0])
            assert run.calls and None not in {i for _, i in run.calls}, (name, run.phase)
            missing = {k: (n, run.checked.get(k, 0)) for k, n in run.calls.items() if run.checked.get(k, 0) != n}
            print("[parity %s %s] %d launches over %d (entry point, block) pairs, all checked: %s"
                  % (name, run.phase, sum(run.calls.values()), len(run.calls), not missing))
            assert not missing, (name, run.phase, sorted(missing.items())[:8])
        nb = len(tr.plan.blocks)
        by = Counter(n for n, _ in tr.calls.elements())
        n_s2d = sum(b.s2d for b in tr.plan.blocks)
        assert by["ryolo_px_conv"] == 2 * nb - 1 and by["ryolo_px_wgrad"] == nb == by["ryolo_px_unpack_wgrad"]
        assert by["ryolo_space_to_depth"] == NP * n_s2d and by["ryolo_px_depth_to_space"] == n_s2d
        assert by["ryolo_px_bn_act_bwd"] == nb - len(tr.plan.heads) == by["ryolo_px_bn_stats"]
        assert Counter(n for n, _ in ev.calls.elements())["ryolo_px_bn_finalize"] == nb - len(tr.plan.heads)
    # the shapes the file is about
    heads = {n: sorted({b.cout for b in tr.plan.heads}) for n, (tr, _) in runs.items()}
    assert heads == {"bench": [504], "nc22": [2016], "tiny": [14]}, heads
    tiny = runs["tiny"][0].plan
    assert min((b.oh, b.ow) for b in tiny.heads) == (4, 5)
    assert any(b.gsrc is not None and b.gsrc.ch_off > 0 for b in runs["bench"][0].plan.blocks)


@pytest.mark.parametrize("phase", ["train", "eval"])
@pytest.mark.parametrize("name", list(SHAPES))
def test_every_launch_within_its_bound(runs, name, phase):
    run = runs[name][0 if phase == "train" else 1]
    assert not run.errors, run.errors[0]
    bad = [(kind, i, k, r[k]) for (kind, i), r in run.res.items() for k in failures(r)]
    assert not bad, bad[:12]
    kinds = {kind for kind, _ in run.res}
    want = {"im2col", "s2d", "z", "head_z", "to_nchw", "bn_act_fwd", "buffers"}
    want |= ({"bn_stats", "bn_finalize", "head_grad", "bn_act_bwd", "wgrad", "dgrad", "d2s", "param_grad"}
             if phase == "train" else {"bn_finalize_eval"})
    assert kinds == want, kinds ^ want
    if phase == "train":              # both kinds of gradient write were checked
        accs = {r["_acc"] for (kind, _), r in run.res.items() if kind == "dgrad" and "_acc" in r}
        assert accs == {0.0, 1.0}, accs


def test_bounds_reject_plausible_bugs(runs):
    """each check, applied to a stored tensor or a reference with one plausible parity bug put in, fails"""
    run = runs["bench"][0]
    plan, model, st = run.plan, run.model, run.stash
    found = {}
    # a 3x3 conv whose K ends on a whole tap: two-plane operand, one lost 512-deep segment
    blk = [b for b in plan.blocks if b.k == 3 and not b.s2d and b.i > 0 and rup(b.cin, 64) % 512 == 0][-1]
    w = run.weight(blk)
    w64 = w.double()
    src = blk.src
    pl = plane_views(src.buf, lo_of(src), src.ch_off, src.c)
    got = interior(blk.z, 0, blk.cout)
    n = rup(blk.cin, 64) // 64
    k = 6 * 9 * n * 64
    want, mag = tapsum(view_val(src), conv_taps(w64), blk.oh, blk.ow)
    assert not failures(gemm_check(got, want, conv_e(mag, k)))
    x2 = (torch.zeros_like(pl[0], dtype=torch.float32) + pl[1].float()) + pl[0].float()
    want2, mag2 = tapsum(x2, conv_taps(w64), blk.oh, blk.ow)
    found["two_planes"] = gemm_check(got, want2, conv_e(mag2, k))
    # the last segment: term a0 * w0 (last in the term table), the last 8 (tap, 64-channel chunk) k-steps
    w0 = w.to(BF16).double()
    lost = torch.zeros_like(want)
    for r_ in range(9 * n - 8, 9 * n):
        tap, ch = divmod(r_, n)
        kh, kw = divmod(tap, 3)
        sl = slice(64 * ch, min(64 * ch + 64, blk.cin))
        part, _ = tapsum(pl[0][..., sl].double(), [(kh - 1, kw - 1, w0[:, sl, kh, kw].t())], blk.oh, blk.ow)
        lost += part
    found["lost_segment"] = gemm_check(got, want - lost, conv_e(mag, k))
    # ryolo_conv_wgrad (one unrestarted accumulator per split) on the same planes: biased towards zero
    cw = st["conv_wgrad"]
    aw, ua = cw["aw"], cw["ua"]
    b_ = plan.blocks[[b.i for b in plan.blocks].index(cw["i"])]
    dw = torch.zeros_like(b_.dw)
    vp = ctypes.c_void_p
    s = pkg()._lib.stream_ptr()
    assert run.real.ryolo_conv_wgrad(vp(cw["dz"].data_ptr()), aw[1], aw[2], vp(aw[3]), aw[4], aw[5], aw[6], aw[7], aw[8],
                                     aw[9], vp(dw.data_ptr()), s) == 0
    gw_old = torch.full(cw["shape"], float("nan"), device=dw.device)
    assert run.real.ryolo_px_unpack_wgrad(vp(dw.data_ptr()), *ua[1:9], vp(gw_old.data_ptr()), s) == 0
    torch.cuda.synchronize()
    m_old = measure(gw_old, cw["want"])
    found["conv_wgrad"] = {"bias": abs(m_old["bias"]) / PX_BIAS_TOL, "_bias": m_old["bias"]}
    # a dgrad that overwrites where it must accumulate
    ow = st["overwrite"]
    found["overwrite"] = gemm_check(ow["got"], ow["want"], ow["e"])
    # px_unpack_wgrad at cin_off + 64 (torch restatement, bit for bit equal to the kernel at the real cin_off)
    up = st["unpack"]
    ua = up["ua"]
    po, pi, cout, cin, ks, off = ua[1], ua[2], ua[5], ua[6], ua[7], ua[8]
    assert f32_equal(unpack_emul(up["dw"], po, pi, cout, cin, ks, off), up["mine"])
    found["cin_off_64"] = gemm_check(unpack_emul(up["dw"], po, pi, cout, cin, ks, off + 64), up["want"], up["e"])
    # plane 1 of a concat slice read at the slice's own rounded width instead of cs / 3
    sb = [b for b in plan.blocks if b.s2d and b.src.ch_off > 0][0]
    s2 = sb.src
    wrong = rup(s2.c, 64)
    assert wrong != lo_of(s2) and s2.ch_off + wrong + s2.c <= s2.cs
    p0, p1, p2 = plane_views(s2.buf, lo_of(s2), s2.ch_off, s2.c)
    p1w = interior(s2.buf, s2.ch_off + wrong, s2.c)
    xb = ((torch.zeros_like(p0, dtype=torch.float32) + p2.float()) + p1w.float()) + p0.float()
    wb = run.weight(sb).double()
    k_s = 6 * 4 * rup(4 * sb.cin, 64)
    want_s, mag_s = tapsum(view_val(s2), conv_taps(wb), sb.oh, sb.ow, 2)
    assert not failures(gemm_check(interior(sb.z, 0, sb.cout), want_s, conv_e(mag_s, k_s)))
    want_b, mag_b = tapsum(xb, conv_taps(wb), sb.oh, sb.ow, 2)
    found["plane_stride"] = gemm_check(interior(sb.z, 0, sb.cout), want_b, conv_e(mag_b, k_s))
    # a nonzero padding channel in a head dz
    hb = plan.heads[0]
    dzc = hb.dz.clone()
    assert planes_pad_zero(dzc, hb.po, hb.cout)
    dzc[0, 1, 1, hb.cout] = 1.0
    found["head_dz_pad"] = {"pad_zero": planes_pad_zero(dzc, hb.po, hb.cout)}
    # running variance with n instead of n - 1
    found["biased_running_var"] = {"running_var": max(run.rv_biased.values())}
    n_rv = sum(v > 1.0 for v in run.rv_biased.values())
    for name_, r in found.items():
        print("[bite] %-20s worst %.3g  %s" % (name_, worst(r), "  ".join(
            "%s %s" % (k_, ("%.3g" % v) if isinstance(v, float) else v) for k_, v in r.items())))
    print("[bite] biased running variance fails on %d of %d BN blocks; the unsegmented wgrad was block %d (%d updates "
          "per chain)" % (n_rv, len(run.rv_biased), cw["i"], cw["updates"]))
    for name_, r in found.items():
        assert failures(r), (name_, r)
    assert found["conv_wgrad"]["_bias"] < -PX_BIAS_TOL
