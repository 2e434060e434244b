"""Every kernel launch of the parity-precision training step and eval forward against float64 of the inputs it received.

ParityPlan (parity_path.py) runs each conv block as px_conv on split operands (three bf16 planes per fp32 value, plane k
of a view at channel ch_off + k * cs / 3) with fp32 element-wise kernels between the GEMMs.  test_parity_bwd_gpu.py runs
those kernels on buffers the test builds; here the plan's own launches are looked at, on the plan's own buffers: its
plane strides, concat slices, accumulate flags, the shared dz / dw scratch re-viewed per block, the head dz padding and
px_unpack_wgrad's cin_off on a whole-buffer wgrad.  rotate_yolov3_b200._lib.lib is swapped for a proxy whose
ryolo_px_* / ryolo_space_to_depth entries record the call, snapshot what it (or a later launch) overwrites, forward it
unchanged, synchronise and check its outputs against float64 of its inputs.  Every reference runs over image chunks of
at most a stated float64 budget, what a launch overwrites is copied to host memory chunk by chunk before it, and every
full reduction (BN sums and two-pass statistics, wgrad + unpack, d gamma / d beta / d slope, the head bias, the
tensor-wide GEMM ratios) is summed in float64 across the chunks, so the same checks run at every batch.  Seeded
init_darknet_weights, a dense random cotangent G per head (loss = sum p * G), one training step, then one eval forward;
each shape's plans are released before the next shape starts:

  bench    yolov3_cfg(), batch 2 x 608^2: the graph of the goldens; GEMM tiles straddle images
  nc22     yolov3_cfg(classes=22, width=416, height=320), batch 3: 2016-filter heads (po 2048, a 6144-channel split dz,
           px_head_grad with no = 28, px_to_nchw with 2016 channels), an odd batch, h != w, grids 10x13 / 20x26 / 40x52
  tiny     yolov3_cfg(160 x 128, 6 anchors), batch 1: a 4 x 5 head grid (6 x 7 = 42 padded pixels, less than one 128-pixel
           GEMM tile), BatchNorm statistics over 20 pixels per channel
  ms448 .. ms768   the --multi-scale sizes at batch 2, one model that switches size (train, eval, next size): eleven
           plan replacements under the proxy
  bench16  yolov3_cfg(), batch 16 x 608^2: the step bench.py's train_parity times.  px_wgrad's split-K chains are 8x
           those of batch 2 (layer 0: 93 025 k-steps), BN reductions over 5.9 M pixels per channel, and the layer-0 split
           buffers and the shared dz scratch past 2^31 bytes (16 x 610^2 x 192 bf16)

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
test_bounds_reject_plausible_bugs puts eight bugs into stored tensors or references of bench, and five into the
references of bench16 (BN sums over 15 of 16 images, a wgrad without its last image, px_wgrad's last split lost, image 15
of a dgrad one row off, the head bias over 15 images), and requires each check to fail.  test_chunking_changes_no_ratio
reruns bench with one image per chunk and requires the whole-batch ratios up to float64 rounding.
test_batch16_schedules_and_memory prints bench16's wgrad schedules, requires longer wgrad chains than any batch-<= 3
launch here, and holds what the checks allocate above the plan to HEADROOM16.

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
The eleven ms sizes, worst over all of them: z element 0.105, max 0.25 (eval), rms 0.33, bias 0.46; dgrad element 0.101;
wgrad element 0.122, max 0.22, rms 0.46; dz 0.32; invstd 0.70; head bias 0.99.  bench16: z element 0.099, max 0.25
(eval), rms 0.32, bias 0.44; head z element 0.097; dgrad element 0.111, max 0.18, rms 0.31, bias 0.42; wgrad element
0.023, max 0.32, rms 0.57 (block 0, 22 splits of 4229 k-steps: the longest chain here, 600 roundings against 137 at batch
<= 3), bias 0.41; dz 0.31; d beta 6e-4, d gamma 0.004; BN sums 0.013; invstd 0.69 (eval 0.64); running mean 0.56,
running variance 0.39; head bias 0.96.  Every GEMM's bias is negative, -8e-9 .. -4.9e-7 of rms (test_parity_bwd_gpu
measures -2.3e-7 .. -3.4e-7 on random operands): what the 32-update segments leave of the accumulator's round-toward-zero.
A training step is 763 launches over 605 (entry point, block) pairs and an eval forward 313 over 303, all checked, at
every shape.  No kernel needed a change.  Bugs put in, worst ratio: x from two planes 1.27 (rms; dropping plane 2 is
noise of 2^-17 relative, under the element bound); one lost 512-deep segment 1.7e5; ryolo_conv_wgrad on the same planes
(block 3, 1676 updates per chain) bias 20; a dgrad that overwrites 4.6e5; cin_off + 64 7.6e5; plane 1 of a concat slice
read at the slice's rounded width instead of cs / 3: 990; a nonzero head dz padding channel fails its bitwise check; a
biased running variance 2.9e3, failing on 71 of the 72 BN blocks.  At batch 16: BN sums without image 15 5e10; a wgrad
without image 15 2.3e5; px_wgrad's last split lost (block 105, 5 splits) 2.5e5; image 15 of a dgrad one row off 1.4e6; the
head bias without image 15 1.1e9.  One image per chunk against one chunk at bench: the ratios move by at most 1.5e-9,
the BN sums' ratio (whose bound is float64 rounding itself) by 5e-3.  Memory: the checks' peak above the plan is 2.97 GB
in the bench16 step and 1.79 GB in its eval forward (BUDGET16 = 3e9 per chunk).  Whole file: 55 s (44.5 s for the
fixture's 15 shapes; bench16's step and checks 10 s)."""
import ctypes
import math
import time
import traceback
import types
from collections import Counter

import pytest
import torch
import torch.nn.functional as F

from builders import pkg
from checked_step import Acc, _host, _img_bytes, chunks, ref_bytes, stats_ref
from f64_refs import (BF16, NP, PX_BIAS_TOL, PX_MAX_TOL, PX_RMS_TOL, TINY, U, DZ_ULPS, _shift, bitwise, cdiv, conv_taps,
                      d2s, gemm_sms, halo_zero, interior, measure, merge3, rup, s2d, s2d_dgrad_ref, split3, tapsum, ulps_f32,
                      wgrad_ref)
from helpers import SMALL_ANCHORS, init_darknet_weights, wgrad_plan

pytestmark = pytest.mark.gpu

U64 = 2.0 ** -53
SEG_UPDATES = 32              # wgmma k16 updates between two accumulator restarts (8 k-steps of 64)
SEG_K = 512                   # GEMM K per accumulator segment
TERMS = 1.0 + 2.0 ** -7       # sum of |a_i w_j| over the plane products, relative to |a| |w|
INV_TRAIN = 3.0               # invstd = 1 / sqrtf((float) var + eps): four fp32 roundings, the sqrt halves two of them
INV_EVAL = 2.5                # the running variance is fp32 already: three roundings
WHOLE = 1e30                  # a chunk budget that puts the whole batch in one chunk
BUDGET16 = 3e9                # float64 bytes of one chunk of images at batch 16 (f64_bytes / ref_bytes estimates)
HEADROOM16 = 2 * BUDGET16     # what the checks (and the step's own gradients) may allocate above the plan at batch 16
MS_SIZES = tuple(range(448, 769, 32))
SHAPES = {
    "bench": (dict(), 2, 608, 608, WHOLE),
    "nc22": (dict(classes=22, width=416, height=320), 3, 320, 416, None),
    "tiny": (dict(width=160, height=128, classes=1, anchors=SMALL_ANCHORS, n_anchors=6), 1, 128, 160, None),
    **{"ms%d" % s: (dict(), 2, s, s, None) for s in MS_SIZES},
    "bench16": (dict(), 16, 608, 608, BUDGET16),
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


def view_val(view, b0=0, b1=None):
    """the fp32 activation a split view carries, images [b0, b1)"""
    return merged(view.buf[b0:b1], lo_of(view), view.ch_off, view.c)


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


def outside_equal(buf, prior, ch_off, c):
    """the channels of buf outside [ch_off, ch_off + c) equal prior's (same images)"""
    allowed = torch.zeros(buf.shape[-1], dtype=torch.bool, device=buf.device)
    allowed[ch_off:ch_off + c] = True
    return torch.equal(buf[..., ~allowed], prior[..., ~allowed])


# ---------------------------------------------------------------------------------------------------------------
# bounds
def conv_e(mag, k):
    """px_conv, GEMM depth K = k: dropped plane products, truncation inside each segment, one RN add per segment"""
    return (2.0 ** -23 + SEG_UPDATES * 2.0 ** -23 + cdiv(k, SEG_K) * U) * TERMS * mag


def wgrad_chain(pw):
    """roundings on one wgrad output: the segment adds of one split, the ksplit partials, the unpack's plane blocks"""
    return cdiv(pw["per_split"], 8) + pw["ksplit"] + NP * NP


def wgrad_e(mag, pw):
    return (SEG_UPDATES * 2.0 ** -23 + wgrad_chain(pw) * U) * TERMS * mag


class GemmAcc(Acc):
    """the element bound |got - want| <= e and test_parity_bwd_gpu's tensor-wide max / rms / bias bounds, accumulated
    over image chunks (checked_step.Acc's moments), as ratios (<= 1 passes)"""

    def __init__(self):
        super().__init__()
        self.elem, self.emax, self.wmax, self.e2 = 0.0, 0.0, 0.0, 0.0

    def add(self, got, want, e):
        err = got.double() - want
        self.elem = worse(self.elem, float((err.abs() / (e + TINY)).max()))
        self.emax = worse(self.emax, float(err.abs().max()))
        self.wmax = max(self.wmax, float(want.abs().max()))
        self.e2 += float(err.pow(2).sum())
        self.moments(err, want)
        return self

    def result(self):
        rms = (self.w2 / self.n) ** 0.5
        bias = self.es / self.n / rms
        return {"elem": self.elem, "max": self.emax / self.wmax / PX_MAX_TOL,
                "rms": (self.e2 / self.n) ** 0.5 / rms / PX_RMS_TOL, "bias": abs(bias) / PX_BIAS_TOL, "_bias": bias}


def gemm_check(got, want, e):
    return GemmAcc().add(got, want, e).result()


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


# ---------------------------------------------------------------------------------------------------------------
class Run:
    """one checked pass (the training step or the eval forward) of one model; launch() is what the proxy calls.  The
    results (res, calls, checked, blocks: a summary of the plan's blocks) outlive release(), which drops the plan and
    every device tensor the run kept."""

    def __init__(self, shape, phase, model, x, real, budget=None, stash=False, bites=False):
        self.shape, self.phase, self.model, self.x, self.real, self.want_stash = shape, phase, model, x, real, stash
        self.batch, self.budget = x.shape[0], budget
        self.calls, self.checked, self.pending = Counter(), Counter(), Counter()
        self.res, self.errors, self.stash, self.bite = {}, [], {}, {} if bites else None
        self.plan, self.cur, self.G, self.blocks, self.base, self.peak = None, None, None, None, None, None
        self.written, self.wg, self.gw, self.rv_biased, self.zstat = {}, {}, {}, {}, None

    def chunks(self, bytes_per_image):
        return chunks(self.batch, bytes_per_image, self.budget)

    def lay(self, buf):
        """image chunks for bit-level checks of buf: a few copies of one image of it"""
        return self.chunks(8 * _img_bytes(buf))

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

    def put_bite(self, name, r):
        if self.bite is not None:
            d = self.bite.setdefault(name, {})
            for k, v in r.items():
                d[k] = worse(d[k], v) if k in d and not k.startswith("_") else v

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
            self.blocks = [types.SimpleNamespace(i=b.i, is_head=b.is_head, s2d=b.s2d, k=b.k, cout=b.cout, oh=b.oh,
                                                 ow=b.ow, gsrc_off=b.gsrc.ch_off if b.gsrc is not None else None)
                           for b in plan.blocks]
        return plan

    def release(self):
        """keep the results, drop the plan and every device tensor this run holds"""
        self.plan = self.by_z = self.by_w = self.by_mean = self.by_hdz = self.by_dxs = self.xs = self.cur = None
        self.model = self.x = self.G = self.zstat = None
        self.stash, self.gw, self.wg = {}, {}, {}

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
        if self.base is None:                       # the plan is built: what the checks add is measured from here
            torch.cuda.synchronize()
            self.base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
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
# handlers: (pre -> snapshot or None, post -> True when the launch is checked).  Every reference runs over image chunks
# of at most run.budget float64 bytes; what a launch overwrites is copied to host memory before it.
def _snap(run, buf):
    return _host(buf, run.lay(buf))


def _prior(snap, b0, b1, dev):
    return snap[b0:b1].to(dev)


def _im2col(run, blk, a, snap):
    plan, x = run.plan, run.x
    assert a[0] == x.data_ptr()
    _, _, h, w = x.shape
    ok = pad = True
    for b0, b1 in run.lay(plan.col):
        want = F.unfold(x[b0:b1], 3, padding=1).view(b1 - b0, 27, h, w).permute(0, 2, 3, 1)
        ok = ok and split_equal(plane_views(plan.col[b0:b1], 64, 0, 27), want)
        pad = pad and planes_pad_zero(plan.col[b0:b1], 64, 27)
    run.put("im2col", 0, {"bits": ok, "pad_zero": pad, "halo": halo_zero(plan.col)})
    return True


def _s2d(run, blk, a, snap):
    k = (a[6] - blk.xs.data_ptr()) // (2 * blk.p4)
    src, c4 = blk.src, 4 * blk.cin
    ok = pad = True
    for b0, b1 in run.lay(src.buf):
        sp = interior(src.buf[b0:b1], src.ch_off + k * lo_of(src), src.c)
        ok = ok and bitwise(interior(blk.xs[b0:b1], k * blk.p4, c4), s2d(sp))
        pad = pad and bool((blk.xs[b0:b1, ..., k * blk.p4 + c4:(k + 1) * blk.p4] == 0).all())
    run.put("s2d", blk.i, {"bits": ok, "pad_zero": pad, "halo": halo_zero(blk.xs)})
    return True


def _pack(run, blk, a, snap):
    run.pending[(blk.i, "dgrad" if a[6] in (1, 3) else "fwd")] += 1
    return False


def _conv_fwd(run, blk, a):
    plan = run.plan
    w64 = run.weight(blk).double()
    k = a[6] * a[11] * a[11] * rup(a[4], 64)
    acc, pad = GemmAcc(), halo_zero(blk.z)
    for b0, b1 in run.chunks(ref_bytes(blk)["fwd"]):
        if blk.i == 0:
            x = merged(plan.col[b0:b1], 64, 0, 27)
            want, mag = tapsum(x, [(0, 0, w64.reshape(blk.cout, 27).t())], blk.oh, blk.ow)
        else:
            want, mag = tapsum(view_val(blk.src, b0, b1), conv_taps(w64), blk.oh, blk.ow, blk.stride)
        acc.add(interior(blk.z[b0:b1], 0, blk.cout), want, conv_e(mag, k))
        del want, mag
        pad = pad and bool((blk.z[b0:b1, ..., blk.cout:] == 0).all())
    r = acc.result()
    r["pad_zero"] = pad
    run.put("head_z" if blk.is_head else "z", blk.i, r)


def _conv_dgrad(run, blk, a, snap):
    w64 = run.weight(blk).double()
    k = a[6] * a[11] * a[11] * rup(a[4], 64)
    src, gs = blk.src, blk.gsrc
    acc = GemmAcc()
    if blk.s2d:
        c4, pad = 4 * blk.cin, halo_zero(blk.dxs)
        for b0, b1 in run.chunks(ref_bytes(blk)["dgrad"]):
            want, mag = s2d_dgrad_ref(merged(blk.dz[b0:b1], blk.po, 0, blk.cout), w64, src.h, src.w)
            acc.add(interior(blk.dxs[b0:b1], 0, c4), want, conv_e(mag, k))
            del want, mag
            pad = pad and bool((blk.dxs[b0:b1, ..., c4:] == 0).all())
        r = acc.result()
        r["pad_zero"] = pad
        run.put("dgrad", blk.i, r)
        return
    acc_w = run.expect_acc(gs)
    outside, dev = halo_zero(gs.buf), gs.buf.device
    for b0, b1 in run.chunks(ref_bytes(blk)["dgrad"]):
        want, mag = tapsum(merged(blk.dz[b0:b1], blk.po, 0, blk.cout), conv_taps(w64, mirror=True), src.h, src.w)
        e = conv_e(mag, k)
        del mag
        cur = gs.buf[b0:b1]
        prior = _prior(snap["gbuf"], b0, b1, dev)
        got = interior(cur, gs.ch_off, gs.c)
        if run.want_stash and acc_w and "overwrite" not in run.stash and src.h * src.w <= 40 * 40:
            run.stash["overwrite"] = dict(i=blk.i, got=got.clone(), want=want.clone(), e=e.clone())
        if acc_w:
            want = want + interior(prior, gs.ch_off, gs.c).double()
            e = e + U * got.double().abs()
        acc.add(got, want, e)
        if b1 == run.batch and run.bite is not None:    # the last image read one row off
            run.put_bite("dgrad_row_off", {"elem": float(((got[-1].double() - want[-1].roll(1, 0)).abs()
                                                           / (e[-1] + TINY)).max())})
        outside = outside and outside_equal(cur, prior, gs.ch_off, gs.c)
        del want, e, prior
    r = acc.result()
    r["acc_flag"] = bool(a[16]) == acc_w
    r["_acc"] = float(acc_w)
    r["outside"] = outside
    run.wrote(gs)
    run.put("dgrad", blk.i, r)


def _conv_pre(run, blk, a):
    if a[13] == blk.z.data_ptr() or blk.s2d:
        return {}
    return {"gbuf": _snap(run, blk.gsrc.buf)}


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
    ok = True
    for b0, b1 in run.lay(blk.z):
        want = interior(blk.z[b0:b1], 0, blk.cout).permute(0, 3, 1, 2)
        if bias is not None:
            want = want + bias.detach()[None, :, None, None]
        ok = ok and f32_equal(blk.out[b0:b1], want)
    run.put("to_nchw", blk.i, {"bits": ok})
    return True


def _zstat(run, blk):
    """two-pass float64 statistics of the block's z (checked_step.stats_ref), computed once per block"""
    if run.zstat is None or run.zstat[0] is not blk:
        c = blk.cout
        run.zstat = (blk, stats_ref(interior(blk.z, 0, c), c, run.chunks(64 * c * blk.oh * blk.ow)))
    return run.zstat[1]


def _bn_stats(run, blk, a, snap):
    c = blk.cout
    ref = _zstat(run, blk)
    n = ref["n"]
    s1, s2 = blk.sums[:c], blk.sums[c:2 * c]
    r1 = ((s1 - ref["s1"]).abs() / (2 * n * U64 * ref["a1"] + TINY)).max()
    r2 = ((s2 - ref["s2"]).abs() / (2 * n * U64 * ref["s2"] + TINY)).max()
    run.put("bn_stats", blk.i, {"sums": float(max(r1, r2))})
    if run.bite is not None:                        # the sums over all images but the last
        z = interior(blk.z[-1:], 0, c).reshape(-1, c).double()
        run.put_bite("bn_sums_without_last", {"sums": float(((s1 - ref["s1"] + z.sum(0)).abs()
                                                             / (2 * n * U64 * ref["a1"] + TINY)).max())})
    return True


def _bn_fin_pre(run, blk, a):
    bn = run.model.module_list[blk.i].BatchNorm2d
    return {"rm": bn.running_mean.clone(), "rv": bn.running_var.clone()}


def _bn_fin(run, blk, a, snap):
    bn = run.model.module_list[blk.i].BatchNorm2d
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
    ref = _zstat(run, blk)
    n, m64, v64 = ref["n"], ref["m64"], ref["v64"]
    q, za = ref["s2"] / n, ref["a1"] / n
    want_inv = 1.0 / (v64 + eps).sqrt()
    r["mean"] = float(((blk.mean.double() - m64).abs() / (2 * ulps(m64) + n * U64 * za + TINY)).max())
    err_inv = (blk.invstd.double() - want_inv).abs()
    r["invstd"] = float((err_inv / (INV_TRAIN * U * want_inv + want_inv * n * U64 * q / (v64 + eps))).max())
    r["_invstd_ulps"] = float((err_inv / ulps(want_inv)).max())
    corr = n / (n - 1)
    rm_w = (1 - mom) * rm0 + mom * m64
    tol_m = 4 * U * ((1 - mom) * rm0.abs() + mom * m64.abs()) + mom * (2 * ulps(m64) + n * U64 * za) + TINY
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
    y, ok = blk.y, True
    for b0, b1 in run.lay(blk.z):
        u = (interior(blk.z[b0:b1], 0, blk.cout) * blk.scale) + blk.shift
        if blk.has_act:
            slope = seq.activation.weight.detach()
            u = torch.where(u > 0, u, slope * u)
        if blk.res is not None:
            u = u + view_val(blk.res, b0, b1)
        pl = plane_views(y.buf[b0:b1], lo_of(y), y.ch_off, y.c)
        if blk.fuse_up:
            ok = ok and all(split_equal([p[:, ry::2, rx::2] for p in pl], u) for ry in range(2) for rx in range(2))
        else:
            ok = ok and split_equal(pl, u)
    run.put("bn_act_fwd", blk.i, {"bits": ok})
    return True


def _head_grad(run, blk, a, snap):
    g = run.G[blk.i]
    _, na, _, _, no = g.shape
    ok = pad = True
    for b0, b1 in run.lay(blk.dz):
        gb = g[b0:b1]
        v = gb.permute(0, 2, 3, 1, 4).reshape(b1 - b0, gb.shape[2], gb.shape[3], na * no)
        ok = ok and split_equal(plane_views(blk.dz[b0:b1], blk.po, 0, na * no), v)
        pad = pad and planes_pad_zero(blk.dz[b0:b1], blk.po, na * no)
    run.put("head_grad", blk.i, {"bits": ok, "pad_zero": pad and halo_zero(blk.dz)})
    return True


def _bn_bwd_pre(run, blk, a):
    return {"gres": _snap(run, blk.gres.buf)} if blk.gres is not None else {}


def _dy(blk, b0, b1):
    """dy as px_bn_act_bwd loads it, images [b0, b1): the gy view, or the 2x2 sum of the up-sampled gradient"""
    g = interior(blk.gy.buf[b0:b1], blk.gy.ch_off, blk.cout)
    if not blk.fuse_up:
        return g
    d = torch.zeros_like(g[:, ::2, ::2])
    for ry in range(2):
        for rx in range(2):
            d = d + g[:, ry::2, rx::2]
    return d


def _bn_bwd(run, blk, a, snap):
    """f64_refs.BnCase.ref / bn_errors (test_parity_bwd_gpu) over image chunks: the channel sums first, then dz"""
    seq = run.model.module_list[blk.i]
    c = blk.cout
    slope = float(seq.activation.weight) if blk.has_act else 1.0
    sc, mean, invstd = blk.scale.double(), blk.mean.double(), blk.invstd.double()
    parts = run.chunks(16 * 8 * c * blk.oh * blk.ow)

    def terms(b0, b1):
        z, d = interior(blk.z[b0:b1], 0, c), _dy(blk, b0, b1)
        u = (z * blk.scale) + blk.shift
        mask = u > 0 if blk.has_act else torch.ones_like(u, dtype=torch.bool)
        d64 = d.double()
        du = torch.where(mask, d64, d64 * slope)
        zh = (z.double() - mean) * invstd
        return d, d64, u, mask, du, zh
    dbeta = dgamma = a1 = a2 = 0.0
    dslope = a_s = torch.zeros((), dtype=torch.float64, device=blk.z.device)
    for b0, b1 in parts:
        _, d64, u, mask, du, zh = terms(b0, b1)
        dbeta, dgamma = dbeta + du.sum((0, 1, 2)), dgamma + (du * zh).sum((0, 1, 2))
        a1, a2 = a1 + du.abs().sum((0, 1, 2)), a2 + (du * zh).abs().sum((0, 1, 2))
        if blk.has_act:
            du_ = (d64 * u.double())[~mask]
            dslope, a_s = dslope + du_.sum(), a_s + du_.abs().sum()
        del d64, u, mask, du, zh
    n = run.batch * blk.oh * blk.ow
    m1, m2 = dbeta / n, dgamma / n
    r = {"dbeta": float(((blk.bsums[:c] - dbeta).abs() / (1e-6 * a1 + 1e-300)).max()),
         "dgamma": float(((blk.bsums[c:2 * c] - dgamma).abs() / (1e-6 * a2 + 1e-300)).max())}
    if blk.has_act:
        r["dslope"] = float((blk.bsums[2 * c] - dslope).abs() / (1e-6 * a_s + 1e-300))
    dz_r, pad = 0.0, halo_zero(blk.dz)
    gr = blk.gres
    acc_g = run.expect_acc(gr) if gr is not None else False
    gbits = gout = True
    for b0, b1 in parts:
        d, _, _, _, du, zh = terms(b0, b1)
        want = sc * (du - m1 - zh * m2)
        mag = sc.abs() * (du.abs() + m1.abs() + a1 / n + zh.abs() * (m2.abs() + a2 / n))
        got = merged(blk.dz[b0:b1], blk.po, 0, c).double()
        dz_r = worse(dz_r, float(((got - want).abs() / (DZ_ULPS * U * mag + 1e-38)).max()))
        pad = pad and planes_pad_zero(blk.dz[b0:b1], blk.po, c)
        del du, zh, want, mag, got
        if gr is not None:
            cur = gr.buf[b0:b1]
            prior = _prior(snap["gres"], b0, b1, d.device)
            gbits = gbits and f32_equal(interior(cur, gr.ch_off, c), interior(prior, gr.ch_off, c) + d if acc_g else d)
            gout = gout and outside_equal(cur, prior, gr.ch_off, c)
            del prior
    r["dz"], r["dz_pad_zero"] = dz_r, pad
    if gr is not None:
        r["gres_bits"], r["gres_flag"] = gbits, bool(a[21]) == acc_g
        r["gres_outside"] = gout and halo_zero(gr.buf)
        run.wrote(gr)
    run.put("bn_act_bwd", blk.i, r)
    return True


def _wgrad(run, blk, a, snap):
    run.wg[blk.i] = list(a)
    return False                                    # checked with its unpack


def _wgrad_part(run, blk, b0, b1, dzm=None):
    """float64 weight gradient (value, magnitude as [cout, cin, k, k]) of images [b0, b1); dzm: a mask on dz"""
    dz = merged(blk.dz[b0:b1], blk.po, 0, blk.cout)
    if dzm is not None:
        dz = dz * dzm
    if blk.i == 0:                                  # on the im2col columns: [cout, 27] is the weight's [cout, 3, 3, 3]
        shape = tuple(run.weight(blk).shape)
        wr, wm = wgrad_ref(merged(run.plan.col[b0:b1], 64, 0, 27), dz, [(0, 0)])
        return wr[0].reshape(shape), wm[0].reshape(shape)
    if blk.s2d:
        return wgrad_s2(view_val(blk.src, b0, b1), dz)
    p = (blk.k - 1) // 2
    wr, wm = wgrad_ref(view_val(blk.src, b0, b1), dz, [(kh - p, kw - p) for kh in range(blk.k) for kw in range(blk.k)])
    return (wr.reshape(blk.k, blk.k, blk.cout, blk.cin).permute(2, 3, 0, 1),
            wm.reshape(blk.k, blk.k, blk.cout, blk.cin).permute(2, 3, 0, 1))


def _lost_split(run, blk, pw):
    """the float64 weight gradient of the k-steps of px_wgrad's last split: the dz pixels (padded-grid index, 64 per
    k-step) from (ksplit - 1) * per_split * 64 on"""
    gh, gw = blk.gh, blk.gw_
    start = (pw["ksplit"] - 1) * pw["per_split"] * 64
    lost = 0.0
    for img in range(start // ((gh + 2) * (gw + 2)), run.batch):
        q = (img * (gh + 2) + 1 + torch.arange(gh, device=blk.z.device)[:, None]) * (gw + 2) + 1 + torch.arange(
            gw, device=blk.z.device)
        lost = lost + _wgrad_part(run, blk, img, img + 1, (q >= start)[None, :, :, None].double())[0]
    return lost


def _unpack(run, blk, a, snap):
    aw = run.wg.pop(blk.i)
    w = run.weight(blk)
    mine = torch.full(tuple(w.shape), float("nan"), dtype=torch.float32, device=w.device)
    args = list(a)
    args[9] = mine.data_ptr()                       # the same launch into a tensor of the test's own
    assert run.real.ryolo_px_unpack_wgrad(*args) == 0
    torch.cuda.synchronize()
    run.gw[blk.i] = mine
    want = mag = 0.0
    for b0, b1 in run.chunks(ref_bytes(blk)["wgrad"]):
        wr, wm = _wgrad_part(run, blk, b0, b1)
        want, mag = want + wr, mag + wm
        if b1 == run.batch and run.bite is not None:
            last = _wgrad_part(run, blk, b1 - 1, b1)[0] if b1 - b0 > 1 else wr
        del wr, wm
    pw = wgrad_plan(aw[9], aw[5], aw[2], aw[6], aw[7], aw[8], gemm_sms(), segmented=True)
    e = wgrad_e(mag, pw)
    r = gemm_check(mine, want, e)
    r["operands"] = aw[0] == blk.dz.data_ptr() and aw[3] == blk.xw_buf.data_ptr() and aw[10] == blk.dw.data_ptr()
    r["_ksplit"], r["_per_split"], r["_chain"] = float(pw["ksplit"]), float(pw["per_split"]), float(wgrad_chain(pw))
    run.put("wgrad", blk.i, r)
    if run.bite is not None:
        run.put_bite("wgrad_without_last_image", gemm_check(mine, want - last, e))
        if pw["ksplit"] > 1 and "wgrad_lost_split" not in run.bite:
            run.put_bite("wgrad_lost_split", dict(gemm_check(mine, want - _lost_split(run, blk, pw), e), _i=float(blk.i),
                                                  _ksplit=float(pw["ksplit"])))
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
    return {"gbuf": _snap(run, blk.gsrc.buf)}


def _d2s(run, blk, a, snap):
    gs = blk.gsrc
    acc = run.expect_acc(gs)
    ok = outside = True
    for b0, b1 in run.lay(gs.buf):
        v = d2s(interior(blk.dxs[b0:b1], 0, 4 * blk.cin), blk.cin)
        cur, prior = gs.buf[b0:b1], _prior(snap["gbuf"], b0, b1, v.device)
        ok = ok and f32_equal(interior(cur, gs.ch_off, gs.c), interior(prior, gs.ch_off, gs.c) + v if acc else v)
        outside = outside and outside_equal(cur, prior, gs.ch_off, gs.c)
    r = {"bits": ok, "acc_flag": bool(a[8]) == acc, "outside": outside and halo_zero(gs.buf)}
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
    ok = all(halo_zero(buf) and all(planes_pad_zero(buf[b0:b1], buf.shape[-1] // NP, c) for b0, b1 in run.lay(buf))
             for buf, c in real.values())
    run.put("buffers", None, {"halo_and_pad": ok})


# ---------------------------------------------------------------------------------------------------------------
def make_model(kw, seed=11):
    from rotate_yolov3_b200 import cfgs
    m = pkg().Darknet(cfgs.yolov3_cfg(**kw), {"context_factor": 1.0}, arc="default", precision="parity")
    return init_darknet_weights(m, seed=seed).to(torch.device("cuda"))


def param_checks(run):
    """after the step: the head bias sums, .grad == the unpack output"""
    for b in run.plan.blocks:
        seq = run.model.module_list[b.i]
        r = {"grad_bits": f32_equal(seq.Conv2d.weight.grad, run.gw[b.i]) if b.i in run.gw else False}
        if b.is_head:
            g = run.G[b.i].double()
            want = g.sum((0, 2, 3)).reshape(-1)
            mag = g.abs().sum((0, 2, 3)).reshape(-1)
            n = g.shape[0] * g.shape[2] * g.shape[3]
            bound = U * want.abs() + n * U64 * mag + TINY
            got = seq.Conv2d.bias.grad.double()
            r["head_bias"] = float(((got - want).abs() / bound).max())
            if run.bite is not None:                # the sum over all images but the last
                run.put_bite("head_bias_without_last", {"head_bias": float(
                    ((got - (want - g[-1].sum((1, 2)).reshape(-1))).abs() / bound).max())})
        run.put("param_grad", b.i, r)


def run_shape(name, model, budget=None):
    """one checked training step and one checked eval forward of model at SHAPES[name]; budget: the chunk budget (the
    shape's own when None).  Returns the two Runs, their plans released."""
    import rotate_yolov3_b200 as pkg_
    _, batch, h, w, own = SHAPES[name]
    budget = own if budget is None else budget
    dev = torch.device("cuda")
    t0 = time.time()
    model.train().zero_grad(set_to_none=True)
    x = torch.rand(batch, 3, h, w, generator=torch.Generator().manual_seed(12)).to(dev)
    real = pkg_._lib.lib
    tr = Run(name, "train", model, x, real, budget, stash=name == "bench" and budget == WHOLE, bites=name == "bench16")
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(pkg_._lib, "lib", Proxy(real, tr))
        ps = model(x)
        torch.cuda.synchronize()
        buffer_checks(tr)
        gen = torch.Generator().manual_seed(13)
        gs = [torch.randn(p.shape, generator=gen).to(dev) for p in ps]
        tr.G = {b.i: g for b, g in zip(tr.plan.heads, gs)}
        loss = sum((p * g).sum() for p, g in zip(ps, gs))
        loss.backward()
        torch.cuda.synchronize()
    param_checks(tr)
    tr.peak = torch.cuda.max_memory_allocated() - tr.base
    if tr.want_stash:
        tr.bite = bench_bites(tr)
    tr.seconds = time.time() - t0
    del ps, gs, loss
    tr.release()
    # eval forward on the updated running statistics; the training plan is gone before the eval plan is built
    t1 = time.time()
    model.eval()
    ev = Run(name, "eval", model, x, real, budget)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(pkg_._lib, "lib", Proxy(real, ev))
        with torch.no_grad():
            model(x)
        torch.cuda.synchronize()
        buffer_checks(ev)
    ev.peak = torch.cuda.max_memory_allocated() - ev.base
    ev.seconds = time.time() - t1
    ev.release()
    model._pplan = model._pplan_key = None
    for run in (tr, ev):
        _print_table(run)
    return tr, ev


def bench_bites(run):
    """each check, applied to a stored tensor or a reference with one plausible parity bug put in (batch 2 x 608^2)"""
    plan, st = run.plan, run.stash
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
    found["conv_wgrad"] = {"bias": abs(m_old["bias"]) / PX_BIAS_TOL, "_bias": m_old["bias"], "_i": float(cw["i"]),
                           "_updates": float(cw["updates"])}
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
    found["biased_running_var"] = {"running_var": max(run.rv_biased.values()),
                                   "_fails_on": float(sum(v > 1.0 for v in run.rv_biased.values())),
                                   "_of": float(len(run.rv_biased))}
    return found


KINDS = ("im2col", "s2d", "z", "head_z", "to_nchw", "bn_stats", "bn_finalize", "bn_finalize_eval", "bn_act_fwd",
         "head_grad", "bn_act_bwd", "wgrad", "dgrad", "d2s", "param_grad")
GEMM_KINDS = ("z", "head_z", "dgrad", "wgrad")


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
    print("\n[parity %s %s] %.1f s, peak %.2f GB above the plan; worst |err| / bound per launch kind (flags: 0 = holds)"
          % (run.shape, run.phase, run.seconds, run.peak / 1e9))
    for b in run.blocks:
        cols = ["%-8s" % ("head" if b.is_head else ("s2d" if b.s2d else "k%d" % b.k)), "%4d" % b.cout,
                "%3dx%-3d" % (b.oh, b.ow)]
        for kind in KINDS:
            r = run.res.get((kind, b.i))
            if r is not None:
                cols.append("%s %.3f" % (kind, worst(r)))
                if kind in GEMM_KINDS and "_bias" in r:
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
    """every shape's two Runs; a shape's plans are released before the next shape starts, so the batch-16 step runs with
    no other plan resident.  The ms sizes are one model that switches size: train, eval, next size."""
    t0 = time.time()
    out, ms = {}, None
    for name, (kw, *_rest) in SHAPES.items():
        if name.startswith("ms"):
            ms = ms or make_model(kw)
            out[name] = run_shape(name, ms)
        else:
            out[name] = run_shape(name, make_model(kw))
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
        nb = len(tr.blocks)
        by = Counter(n for n, _ in tr.calls.elements())
        n_s2d = sum(b.s2d for b in tr.blocks)
        n_heads = sum(b.is_head for b in tr.blocks)
        assert by["ryolo_px_conv"] == 2 * nb - 1 and by["ryolo_px_wgrad"] == nb == by["ryolo_px_unpack_wgrad"]
        assert by["ryolo_space_to_depth"] == NP * n_s2d and by["ryolo_px_depth_to_space"] == n_s2d
        assert by["ryolo_px_bn_act_bwd"] == nb - n_heads == by["ryolo_px_bn_stats"]
        assert Counter(n for n, _ in ev.calls.elements())["ryolo_px_bn_finalize"] == nb - n_heads
    # the shapes the file is about
    heads = {n: sorted({b.cout for b in tr.blocks if b.is_head}) for n, (tr, _) in runs.items()}
    assert heads == {n: [2016] if n == "nc22" else [14] if n == "tiny" else [504] for n in SHAPES}, heads
    assert min((b.oh, b.ow) for b in runs["tiny"][0].blocks if b.is_head) == (4, 5)
    assert any(b.gsrc_off is not None and b.gsrc_off > 0 for b in runs["bench"][0].blocks)
    assert {n: runs[n][0].batch for n in ("bench", "bench16")} == {"bench": 2, "bench16": 16}


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


def test_batch16_schedules_and_memory(runs):
    """the 16 x 608^2 step train_parity times: its wgrad schedules, BN reductions and the checks' memory"""
    tr, ev = runs["bench16"]
    print("\n[parity bench16] block  kind  cout  grid      ksplit  per_split  chain  BN pixels/channel")
    for b in tr.blocks:
        r = tr.res[("wgrad", b.i)]
        print("[parity bench16] %5d  %-4s  %4d  %3dx%-3d  %6d  %9d  %5d  %s" % (
            b.i, "head" if b.is_head else ("s2d" if b.s2d else "k%d" % b.k), b.cout, b.oh, b.ow, r["_ksplit"],
            r["_per_split"], r["_chain"], "-" if b.is_head else "%d" % (tr.batch * b.oh * b.ow)))
    chain16 = max(r["_chain"] for (kind, _), r in tr.res.items() if kind == "wgrad")
    small = max(r["_chain"] for n, (t, _) in runs.items() if t.batch <= 3
                for (kind, _), r in t.res.items() if kind == "wgrad")
    print("[parity bench16] longest wgrad chain %d (batch <= 3: %d); peak above the plan: train %.2f GB, eval %.2f GB "
          "(allowed %.1f GB); step + checks %.1f s, eval %.1f s" % (chain16, small, tr.peak / 1e9, ev.peak / 1e9,
                                                                     HEADROOM16 / 1e9, tr.seconds, ev.seconds))
    assert chain16 > small
    assert max(b.oh * b.ow for b in tr.blocks if not b.is_head) * tr.batch == 16 * 608 * 608
    assert tr.peak <= HEADROOM16 and ev.peak <= HEADROOM16, (tr.peak, ev.peak)


BITES16 = ("bn_sums_without_last", "wgrad_without_last_image", "wgrad_lost_split", "dgrad_row_off",
           "head_bias_without_last")


def _print_bites(tag, found):
    for name_, r in found.items():
        print("[bite %s] %-26s worst %.3g  %s" % (tag, name_, worst(r), "  ".join(
            "%s %s" % (k_, ("%.3g" % v) if isinstance(v, float) else v) for k_, v in r.items())))


def test_bounds_reject_plausible_bugs(runs):
    """each check, applied to a stored tensor or a reference with one plausible parity bug put in, fails: eight at
    batch 2, five that only a batch of 16 images shows"""
    found = runs["bench"][0].bite
    _print_bites("bench", found)
    for name_, r in found.items():
        assert failures(r), (name_, r)
    assert found["conv_wgrad"]["_bias"] < -PX_BIAS_TOL
    f16 = runs["bench16"][0].bite
    _print_bites("bench16", f16)
    assert sorted(f16) == sorted(BITES16), sorted(f16)
    for name_, r in f16.items():
        assert failures(r), (name_, r)


# ratios whose bound is itself a float64 rounding bound move with the reference's own summation order: the BN sums
# (bound 2 n 2^-53 sum |terms|, the reference's recursive sum is within half of it) and the BN backward sums (bound
# 1e-6 sum |terms|, the reference within n 2^-53 sum |terms|: under 1e-4 of the bound at 739 200 pixels per channel)
F64_SLACK = {("bn_stats", "sums"): 0.5, ("bn_act_bwd", "dbeta"): 1e-4, ("bn_act_bwd", "dgamma"): 1e-4,
             ("bn_act_bwd", "dslope"): 1e-4}


def test_chunking_changes_no_ratio(runs):
    """2 x 608^2 with one image per chunk gives the whole-batch chunk's ratios, up to float64 rounding"""
    one = run_shape("bench", make_model(SHAPES["bench"][0]), budget=1)
    for whole, part in zip(runs["bench"], one):
        assert not part.errors, part.errors[0]
        assert set(whole.res) == set(part.res)
        bad, worst_d = [], {}
        for key, r in whole.res.items():
            q = part.res[key]
            assert set(r) == set(q), key
            for k, v in r.items():
                if isinstance(v, bool):
                    if v != q[k]:
                        bad.append((key, k, v, q[k]))
                    continue
                slack = F64_SLACK.get((key[0], k), 1e-9)
                d = abs(v - q[k])
                worst_d[(key[0], k)] = max(worst_d.get((key[0], k), 0.0), d)
                if not d <= 1e-6 * max(abs(v), abs(q[k])) + slack:
                    bad.append((key, k, v, q[k]))
        for (kind, k), d in sorted(worst_d.items()):
            print("[parity chunks %s] %-16s %-14s largest change %.2e" % (whole.phase, kind, k, d))
        assert not bad, bad[:12]
