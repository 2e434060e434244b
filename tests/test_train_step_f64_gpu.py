"""Every kernel launch of one bf16 training step at 608 x 608 against float64 of the inputs it actually received.

The step is the one bench.py measures: Darknet-53 / YOLOv3 (cfgs.yolov3_cfg(): 75 convs, 504-filter heads, 768- and
384-channel concat buffers) run by train_path.TrainPlan, here at batch 2 so that GEMM tiles straddle the image boundary of
the flat pixel index.  A dense random cotangent G per head (loss = sum (p * G)) reaches all 504 head channels.

Forward: after model(x) every buffer a forward kernel wrote is still there, so each launch is checked post hoc on the
plan's own input buffers (the im2col columns, a view, a concat slice, the space-to-depth copy): im2col bit for bit, the
multi-tensor weight pack bit for bit against ryolo_conv_pack_weights_ex, the raw conv z, the fp32 heads, the batch
statistics (two-pass float64) with the running-statistics update, and bn_act_fwd / bn_act_fwd_s2d.  Backward:
plan._backward_block is wrapped (instance attribute) so that each block's inputs are snapshotted, the production code runs
unchanged, and its outputs are checked right after: bn_act_bwd (dz, d beta, d gamma, d slope, the shortcut gradient), the
split-K weight gradient and its gather, the dgrad (mode-1 operands; mode-3 operands with ksize -2 and the depth_to_space
pass) including the accumulate flag and the channels outside the gradient view.  No graph sits between a kernel and its
reference, so no PReLU kink crossing blurs a check and the bounds are the single-kernel ones:

  A = the same operation in float64 on |operands|,  n = sequential accumulator updates (taps * cin_pad / 16 for the conv
  kernel; for the split-K wgrad the longest chain, wgrad_plan's updates of one split + the ksplit partials added in split
  order),  E = n * 2^-23 * A  (one fp32 ulp per update: the tensor pipe's accumulator does not round to nearest, DESIGN.md
  section 6)
  bf16 outputs   |got - want| <= 2^-8 (|want| + E + T) + E + T     (T: the fp32 epilogue terms of the kernel)
                 |mean((got - want) sign(want))| <= 2^-12 rms(want)     (no round-toward-zero bias)
  fp32 outputs   |got - want| <= E + 2^-24 |want|     (heads, weight gradients)
  every ratio must be <= 1, so a NaN anywhere in an output fails its check
  reductions     L * 2^-24 * sum |terms|, L = the longest fp32 addition chain of the kernel's reduction:
                 bn_stats / bn_act_bwd reduce (bnpipe.cuh): a thread owns one 8-channel group for the whole kernel and adds
                 its items of every piece its CTA takes: per_cta * ceil(items per row / 256) * rows per piece; then
                 block_partials adds the 256 / cgs threads of a channel; bn_sums_reduce_kernel adds ceil(grid / 8) rows per
                 part and the 8 parts (bn_chain below mirrors mk_pieces).  d slope: a thread adds all 8 channels, then a
                 5-level butterfly and the 8 warps.  Head bias (head_grad_nchw_kernel): 5-level warp sum, rows_per_block *
                 ceil(nx / 32) chunk sums per block, ordered_rows_add_kernel: ceil(blocks / 8) + 8, one add into the zeroed
                 gradient.
  BN statistics  invstd within 2^-12 relative and mean within 2^-12 std on every channel (below that the error is
                 invisible under the bf16 rounding of y).

The one-pass fp32 variance (E[z^2] - mean^2) is also run alone at the benchmark's count (c = 32, 304^2, batch 64: 5.9 M
pixels per channel) at |mean| / std in {0, 2, 8, 32}; the bound is required up to ratio 8 or twice the largest ratio the
608 step produced, whichever is larger.  A last test applies ten plausible bugs to the stored tensors or references and
requires each check to fail.

Measured on an H100 80GB HBM3 (132 SMs, power limit 400 W, 1980 MHz max SM clock), seeds as below, two runs bitwise
identical.  `pytest -s` prints the per-block table (one line per block: each kernel's worst |err| / bound and the block's
|mean| / std); its summary, the worst ratio per kernel over the 75 blocks and the block where it occurs:
  conv z (bf16)   0.996 (layer 0), bias 0.037 (64)       fp32 heads        0.142 (105)
  bn statistics   mean 0.001, invstd 0.007 (0); sums, finalisation and running statistics pass; |mean| / std <= 5.22 (87)
  bn_act_fwd      0.996 (0), bias 0.072 (57)             bn_act_bwd dz     0.996 (0), bias 0.051 (84)
  d beta          0.016 (76)   d gamma 0.030 (66)   d slope < 0.001   head bias 0.011 (81)
  dgrad           0.996 (2), bias 0.047 (78)             wgrad             0.106 (67)
The bf16 ratios just under 1 are half an ulp at the bottom of a binade: every bf16 output is the correctly rounded float64
result up to E.  test_wgrad's random-walk bound (KAPPA sqrt(n_add) 2^-24 A) alone is exceeded on the 19^2 layers (up to
1.61 at layer 67, 57 updates per chain): the post-PReLU operands are not sign-random and the accumulator's truncations
add up; the wgrad check therefore uses E.  BN statistics at 5.9 M pixels per channel: invstd relative error 2.7e-7 /
2.4e-6 / 3.7e-5 / 7.2e-5 / 6.1e-4 at |mean| / std = 0 / 2 / 8 / 10.4 / 32 (mean error <= 4.7e-6 std): the one-pass
variance meets the target up to twice the step's largest ratio and misses it at 32.  Bugs put in: every check fails by
a factor >= 1.8 (round-toward-zero z: bias 9.1; a lost split-K partial: 2377; one NaN in z fails), and the biased
running variance fails on 71 of the 72 BN blocks.  Whole file: 10 s (3.1 s for the step and its checks)."""
import time
import traceback

import pytest
import torch
import torch.nn.functional as F

import test_wgrad_gpu as wgrad_test
from helpers import init_darknet_weights, wgrad_plan

pytestmark = pytest.mark.gpu

BATCH = 2
SIZE = 608
U = 2.0 ** -24
HALF_BF16 = 2.0 ** -8
BIAS_TOL = 2.0 ** -12
STAT_TOL = 2.0 ** -12
TINY = 1e-30
F64 = torch.float64
BF16 = torch.bfloat16
MOMENTUM_DEFAULT = 0.1


def _pkg():
    import rotate_yolov3_b200 as pkg
    return pkg


def _layout():
    from rotate_yolov3_b200 import layout
    return layout


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def rup(x, m):
    return (x + m - 1) // m * m


def cdiv(a, b):
    return -(-a // b)


def interior(buf, off, c):
    """[B, H, W, c] view of channels [off, off + c) of a padded-NHWC buffer"""
    return buf[:, 1:-1, 1:-1, off:off + c]


def vint(view):
    return interior(view.buf, view.ch_off, view.c)


def halo_zero(buf):
    return bool((buf[:, 0] == 0).all() and (buf[:, -1] == 0).all() and (buf[:, :, 0] == 0).all()
                and (buf[:, :, -1] == 0).all())


def d2s(dxs, c):
    """depth_to_space of the interior of an s2d buffer: [B, h, w, 4c] -> [B, 2h, 2w, c]"""
    b, h, w, _ = dxs.shape
    t = dxs[..., :4 * c].reshape(b, h, w, 2, 2, c)
    return t.permute(0, 1, 3, 2, 4, 5).reshape(b, 2 * h, 2 * w, c)


def s2d(x):
    """space_to_depth: [B, 2h, 2w, c] -> [B, h, w, 4c], channel (py * 2 + px) * c + ci"""
    b, hh, ww, c = x.shape
    return x.reshape(b, hh // 2, 2, ww // 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(b, hh // 2, ww // 2, 4 * c)


def rtz_bf16(v32):
    """round-toward-zero fp32 -> bf16 (drop the low 16 bits)"""
    return (v32.contiguous().view(torch.int32) & -65536).view(torch.float32).to(BF16)


# ---------------------------------------------------------------------------------------------------------------
# float64 references: sums over taps of shifted NHWC operands, chunk-free (the largest operand is ~0.4 GB in float64)
def _shift(xp, dy, dx, oh, ow, s=1):
    return xp[:, 1 + dy:2 + dy + s * (oh - 1):s, 1 + dx:2 + dx + s * (ow - 1):s, :]


def tapsum(x, taps, oh, ow, s=1):
    """out[b, y, x] = sum over taps (dy, dx, M [C, N]) of x[b, s y + dy, s x + dx] @ M (zero outside x), float64; returns
    the value and the same sum on |x|, |M|"""
    xp = F.pad(x.double(), (0, 0, 1, 1, 1, 1))
    xa = xp.abs()
    b, c = x.shape[0], x.shape[3]
    n = taps[0][2].shape[1]
    out = torch.zeros(b * oh * ow, n, dtype=F64, device=x.device)
    mag = torch.zeros_like(out)
    for dy, dx, m in taps:
        out.addmm_(_shift(xp, dy, dx, oh, ow, s).reshape(-1, c), m)
        mag.addmm_(_shift(xa, dy, dx, oh, ow, s).reshape(-1, c), m.abs())
    return out.view(b, oh, ow, n), mag.view(b, oh, ow, n)


def conv_taps(w64, mirror=False, drop=None, flip=True):
    """taps of a k x k / pad (k-1)/2 conv with weight [cout, cin, k, k] (forward: M = W^T) or of its input gradient
    (mirror: dx[p] = sum dz[p - off] @ W_tap); drop = a tap (kh, kw) left out; flip=False: the input gradient with the
    taps NOT mirrored (a plausible packing bug)"""
    k = w64.shape[2]
    p = (k - 1) // 2
    taps = []
    for kh in range(k):
        for kw in range(k):
            if drop == (kh, kw):
                continue
            if mirror:
                taps.append((p - kh, p - kw, w64[:, :, kh, kw]) if flip else (kh - p, kw - p, w64[:, :, kh, kw]))
            else:
                taps.append((kh - p, kw - p, w64[:, :, kh, kw].t()))
    return taps


def s2d_dgrad_ref(dz, w64, h, w):
    """input gradient of the 3x3 / stride-2 / pad-1 conv on the [h, w] input grid (dz placed on the even pixels, then the
    mirrored taps), returned in the space-to-depth layout of the kernel's dxs output: value and magnitude"""
    b, oh, ow, cout = dz.shape
    up = torch.zeros((b, h, w, cout), dtype=F64, device=dz.device)
    up[:, ::2, ::2] = dz.double()
    want, mag = tapsum(up, conv_taps(w64, mirror=True), h, w)
    return s2d(want), s2d(mag)


def wgrad_ref(x, dz, offs):
    """dw[t, co, ci] = sum_p dz[p, co] x[p + offs[t], ci] (x, dz on the same grid): value and magnitude"""
    b, h, w, cin = x.shape
    cout = dz.shape[3]
    xp = F.pad(x.double(), (0, 0, 1, 1, 1, 1))
    d = dz.double().reshape(-1, cout)
    da = d.abs()
    outs, mags = [], []
    for dy, dx in offs:
        a = _shift(xp, dy, dx, h, w).reshape(-1, cin)
        outs.append(d.t() @ a)
        mags.append(da.t() @ a.abs())
    return torch.stack(outs), torch.stack(mags)


# ---------------------------------------------------------------------------------------------------------------
# bounds: each returns worst |err| / bound (and the bias over its bound); <= 1 passes
def bf16_check(got, want, e, t=0.0):
    err = got.double() - want
    bound = HALF_BF16 * (want.abs() + e + t) + e + t + TINY
    rms = float(want.pow(2).mean().sqrt())
    bias = abs(float((err * want.sign()).mean())) / (BIAS_TOL * rms + TINY)
    return {"max": float((err.abs() / bound).max()), "bias": bias}


def f32_check(got, want, e):
    err = (got.double() - want).abs()
    return {"max": float((err / (e + U * want.abs() + TINY)).max())}


def sum_check(got, want, l, mag):
    return float(((got.double() - want).abs() / (l * U * mag + TINY)).max())


def bitwise(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def passed(r):
    """every ratio <= 1 (a NaN ratio fails) and every flag true"""
    return all((v <= 1.0) if isinstance(v, float) else v for v in r.values() if isinstance(v, (float, bool)))


def wgrad_ratio(got, want, mag, plan):
    """split-K weight gradient: one fp32 ulp of the magnitude per update of the longest chain -- the updates of one split
    plus the ksplit partials added in split order -- and half an ulp of the fp32 result"""
    n = plan["updates"] + plan["ksplit"]
    return wgrad_test.worst_ratio(got, want, mag, 0, extra=n * 2.0 ** -23 * mag + U * want.abs())


# ---------------------------------------------------------------------------------------------------------------
# reduction chain lengths (mirror of mk_pieces in bnpipe.cuh)
def bn_chain(batch, h, w, c, rows_per_piece=1):
    cgs = c // 8
    max_px = 1280 // rows_per_piece // cgs
    if rows_per_piece == 2:
        max_px &= ~1
    ppr = cdiv(w, max_px)
    px = cdiv(w, ppr)
    if rows_per_piece == 2 and px % 2:
        px += 1
    total = batch * (h // rows_per_piece) * ppr
    per_cta = cdiv(total, 2 * sms())
    grid = cdiv(total, per_cta)
    per_thread = per_cta * cdiv(px * cgs, 256) * rows_per_piece
    rows = cdiv(grid, 8) + 8
    return dict(sums=per_thread + 256 // cgs + rows, slope=8 * per_thread + 5 + 8 + rows)


def head_bias_chain(batch, ny, nx):
    rpb = max(1, cdiv(ny * batch, 2048))
    blocks = cdiv(ny, rpb) * batch
    return 5 + rpb * cdiv(nx, 32) + cdiv(blocks, 8) + 8 + 1


# ---------------------------------------------------------------------------------------------------------------
# per-kernel checks
def fwd_ref(plan, blk, w):
    """float64 raw conv of the block on its actual input buffer, and its magnitude"""
    w64 = w.detach().to(BF16).double()
    if blk.i == 0:
        x = interior(plan.col, 0, 27)
        return tapsum(x, [(0, 0, w64.reshape(blk.cout, 27).t())], blk.oh, blk.ow)
    return tapsum(vint(blk.src), conv_taps(w64), blk.oh, blk.ow, blk.stride)


def conv_updates(blk):
    return blk.k_eff * blk.k_eff * blk.cin_pad // 16


def check_z(got, want, mag, n):
    return bf16_check(got, want, n * 2.0 ** -23 * mag)


def bn_act_fwd_ref(z, sc, sh, slope, res=None):
    """y = prelu(fma(z, scale, shift)) [+ res] in float64 on the kernel's fp32 scale / shift / slope; branch from the fp32
    u; returns (want, T)"""
    z64 = z.double()
    zs = z64 * sc.double()
    u64 = zs + sh.double()
    pos = u64.float() > 0
    a = torch.where(pos, u64, u64 * float(slope))
    r = res.double() if res is not None else 0.0
    want = a + r
    t = 3 * U * (zs.abs() + sh.double().abs() + (r.abs() if res is not None else 0.0))
    return want, t


def stats_check(z, c, sums, mean, invstd, scale, shift, rm0, rv0, rm, rv, gamma, beta, eps, mom, l, unbiased=True):
    """batch statistics: the kernel's sums against float64 (reduction bound), mean / invstd against the two-pass float64
    statistics (target 2^-12), the finalisation and the running statistics against both the float64 statistics and the
    fp32 arithmetic of bn_finalize_channel applied to the kernel's own sums"""
    z64 = z.double().reshape(-1, c)
    n = z64.shape[0]
    m64 = z64.mean(0)
    v64 = (z64 - m64).pow(2).mean(0)
    std = (v64 + eps).sqrt()
    s1, s2 = sums[:c].double(), sums[c:2 * c].double()
    r = {}
    r["sums"] = max(sum_check(s1, z64.sum(0), l, z64.abs().sum(0)), sum_check(s2, z64.pow(2).sum(0), l, z64.pow(2).sum(0)))
    r["mean"] = float(((mean.double() - m64).abs() / (STAT_TOL * std)).max())
    r["invstd"] = float(((invstd.double() - 1.0 / std).abs() / (STAT_TOL / std)).max())
    # bn_finalize_channel on the kernel's sums: mean = s1 / n (IEEE), var = s2 / n - mean^2 (contracted or not)
    cnt = torch.tensor(float(n), dtype=torch.float32, device=z.device)
    mean_e = sums[:c] / cnt
    q = (sums[c:2 * c] / cnt).double()
    me = mean_e.double()
    var_e = (q - me * me).clamp_min(0.0)
    dv = 2 * U * (q + me * me) + 2 * U * (var_e + eps)
    inv_e = 1.0 / (var_e + eps).sqrt()
    fin = [0.0 if torch.equal(mean, mean_e) else 2.0,
           float(((invstd.double() - inv_e).abs() / (inv_e * (dv / (2 * (var_e + eps)) + 4 * U))).max())]
    sc_want = gamma * invstd                                        # one fp32 multiply
    fin.append(0.0 if torch.equal(scale, sc_want) else 2.0)
    sh_want = beta.double() - mean.double() * scale.double()
    fin.append(float(((shift.double() - sh_want).abs() / (2 * U * (beta.double().abs() + (mean.double() * scale.double()).abs())
                                                          + TINY)).max()))
    corr = n / (n - 1) if unbiased else 1.0
    rm_e = (1 - mom) * rm0.double() + mom * me
    rv_e = (1 - mom) * rv0.double() + mom * var_e * corr
    fin.append(float(((rm.double() - rm_e).abs() / (4 * U * ((1 - mom) * rm0.double().abs() + mom * me.abs()) + TINY)).max()))
    fin.append(float(((rv.double() - rv_e).abs() / (4 * U * ((1 - mom) * rv0.double().abs() + mom * var_e * corr)
                                                    + mom * corr * dv + TINY)).max()))
    r["finalize"] = max(fin)
    # running statistics against the float64 statistics: the target error of mean / variance carried through momentum
    rm_w = (1 - mom) * rm0.double() + mom * m64
    rv_w = (1 - mom) * rv0.double() + mom * v64 * corr
    r["running"] = max(
        float(((rm.double() - rm_w).abs() / (4 * U * rm_w.abs() + mom * STAT_TOL * std + TINY)).max()),
        float(((rv.double() - rv_w).abs() / (4 * U * rv_w.abs() + mom * corr * 2 * STAT_TOL * std * std + TINY)).max()))
    ratio = float((m64.abs() / v64.sqrt().clamp_min(1e-30)).max())
    return r, ratio


def bn_bwd_check(z, d, dz_got, sums_got, mean, invstd, sc, sh, slope, chain, drop_m2=False):
    """float64 BatchNorm backward (batch statistics) through PReLU on the kernel's fp32 statistics, with d = the dy the
    kernel read (fp32).  The PReLU branch is decided by the fp32 u = fma(z, scale, shift) as in the kernel; elements within
    four fp32 ulps of u = 0 are left out of the element-wise dz bound (counted)."""
    c = z.shape[-1]
    z64 = z.double().reshape(-1, c)
    d64 = d.double().reshape(-1, c)
    n = z64.shape[0]
    zs = z64 * sc.double()
    u64 = zs + sh.double()
    u32 = u64.float().double()
    pos = u32 > 0
    near = u64.abs() <= 4 * U * (zs.abs() + sh.double().abs())
    du = torch.where(pos, d64, d64 * float(slope))
    zh = (z64 - mean.double()) * invstd.double()
    duzh = du * zh
    dbeta, dgamma = du.sum(0), duzh.sum(0)
    neg = ~pos
    dslope = (d64 * u32)[neg].sum()
    a1, a2 = du.abs().sum(0), duzh.abs().sum(0)
    a_s = (d64 * u32)[neg].abs().sum()
    m1 = dbeta / n
    m2 = torch.zeros_like(dgamma) if drop_m2 else dgamma / n
    want = sc.double() * (du - m1 - zh * m2)
    t = sc.double().abs() * (8 * U * (du.abs() + m1.abs() + (zh * m2).abs()) + chain["sums"] * U * (a1 + zh.abs() * a2) / n)
    keep = ~near
    r = bf16_check(dz_got.reshape(-1, c)[keep], want[keep], 0.0, t[keep])
    r["finite"] = bool(torch.isfinite(dz_got).all())
    r["dbeta"] = sum_check(sums_got[:c], dbeta, chain["sums"] + 1, a1)
    r["dgamma"] = sum_check(sums_got[c:2 * c], dgamma, chain["sums"] + 3, a2)
    r["dslope"] = float((sums_got[2 * c].double() - dslope).abs() / (chain["slope"] * U * a_s + TINY))
    return r, int(near.sum())


def dy_of(plan, blk, shift=0):
    """(dy as bn_act_bwd reads it, fp32 [B, oh, ow, c]; mode): the gy view, the 2x2 sum of the up-sampled gradient in the
    kernel's order, or the consumer's dxs in place (mode 2).  shift: read the gradient buffer that many channels off."""
    cons = getattr(blk, "dy_s2d", None)
    if cons is not None:
        return d2s(interior(cons.dxs, 0, cons.xs_cs), blk.cout).float(), 2
    g = interior(blk.gy.buf, blk.gy.ch_off + shift, blk.cout).float()
    if not blk.fuse_up:
        return g, 0
    s = torch.zeros_like(g[:, ::2, ::2])
    for ry in range(2):
        for rx in range(2):
            s = s + g[:, ry::2, rx::2]
    return s, 1


# ---------------------------------------------------------------------------------------------------------------
class Step:
    """one checked training step; batch, h, w default to the module's 608 step"""
    batch, h, w = BATCH, SIZE, SIZE


def _bn_of(model, blk):
    return model.module_list[blk.i].BatchNorm2d


def _slope_of(model, blk):
    return model.module_list[blk.i].activation.weight.detach().float()


def _weight(model, blk):
    return model.module_list[blk.i].Conv2d.weight.detach()


def forward_checks(st):
    plan, model = st.plan, st.model
    L = _layout()
    out = {}
    # im2col of the image: bit for bit, columns 27..63 and the halo zero
    want_col = F.unfold(st.x, 3, padding=1).view(st.batch, 27, st.h, st.w).permute(0, 2, 3, 1).to(BF16)
    st.im2col = dict(bits=bitwise(interior(plan.col, 0, 27), want_col),
                     pad_zero=bool((interior(plan.col, 27, 37) == 0).all()), halo=halo_zero(plan.col))
    # the multi-tensor pack against the single-operand pack into fresh buffers
    packs = []
    for blk in plan.blocks:
        if blk.owner is not None:          # a weight_from block runs its owner's packed operands
            continue
        w = _weight(model, blk)
        wf = w.reshape(blk.cout, 27, 1, 1).contiguous() if blk.i == 0 else w
        packs.append((blk.i, "fwd", torch.equal(blk.pw, L.pack_weights(blk.fdesc, wf, mode=2 if blk.s2d else 0))))
        if blk.i > 0:
            packs.append((blk.i, "dgrad", torch.equal(blk.pwd, L.pack_weights(blk.ddesc, w, mode=3 if blk.s2d else 1))))
    st.packs = packs
    ratios = []
    st.rv_biased = {}
    for blk in plan.blocks:
        if blk.owner is not None:          # weight_from blocks: their own launches (test_dilated_train_f64_gpu.py)
            continue
        r = {}
        w = _weight(model, blk)
        want, mag = fwd_ref(plan, blk, w)
        n = conv_updates(blk)
        if blk.is_head:
            bias = model.module_list[blk.i].Conv2d.bias.detach().double()
            got = blk.out.detach().permute(0, 2, 3, 1)
            r["z"] = f32_check(got, want + bias, n * 2.0 ** -23 * mag)["max"]
            out[blk.i] = r
            continue
        z = interior(blk.z, 0, blk.cout)
        rz = check_z(z, want, mag, n)
        r["z"], r["z_bias"] = rz["max"], rz["bias"]
        if blk.i in st.keep_fwd:
            st.stash[("z", blk.i)] = dict(want=want.clone(), mag=mag.clone(), n=n, got=z.clone())
        del want, mag
        if blk.has_bn:
            bn = _bn_of(model, blk)
            rs, ratio = stats_check(z, blk.cout, blk.sums, blk.mean, blk.invstd, blk.scale, blk.shift, st.rm0[blk.i],
                                    st.rv0[blk.i], bn.running_mean, bn.running_var, bn.weight.detach(), bn.bias.detach(),
                                    bn.eps, bn.momentum, bn_chain(st.batch, blk.oh, blk.ow, blk.cout)["sums"])
            r.update(rs)
            r["mean_over_std"] = ratio
            # the same check with the running variance taken as biased (n instead of n - 1): kept for the bound self-test
            rb_, _ = stats_check(z, blk.cout, blk.sums, blk.mean, blk.invstd, blk.scale, blk.shift, st.rm0[blk.i],
                                 st.rv0[blk.i], bn.running_mean, bn.running_var, bn.weight.detach(), bn.bias.detach(),
                                 bn.eps, bn.momentum, bn_chain(st.batch, blk.oh, blk.ow, blk.cout)["sums"], unbiased=False)
            st.rv_biased[blk.i] = max(rb_["running"], rb_["finalize"])
            ratios.append(ratio)
        else:
            # a bias (+ PReLU) conv without BatchNorm: fixed statistics, scale 1 and shift = the conv bias, bit for bit
            bias = model.module_list[blk.i].Conv2d.bias.detach()
            r["fixed_stats"] = bool((blk.scale == 1).all()) and torch.equal(blk.shift, bias)
        # bn_act_fwd
        res = vint(blk.res) if blk.res is not None else None
        want_y, t = bn_act_fwd_ref(z, blk.scale, blk.shift, _slope_of(model, blk), res)
        y = interior(blk.y.buf, blk.y.ch_off, blk.cout)
        if blk.fuse_up:
            base = y[:, ::2, ::2]
            r["up_copies"] = all(bitwise(y[:, ry::2, rx::2], base) for ry in range(2) for rx in range(2))
            y = base
        ry_ = bf16_check(y, want_y, 0.0, t)
        r["y"], r["y_bias"] = ry_["max"], ry_["bias"]
        if blk.i in st.keep_fwd and res is not None:
            st.stash[("y", blk.i)] = dict(z=z.clone(), res=res.clone(), got=y.clone(), sc=blk.scale.clone(),
                                          sh=blk.shift.clone(), slope=_slope_of(model, blk))
        out[blk.i] = r
    # space-to-depth copies (bn_act_fwd_s2d or ryolo_space_to_depth) bit for bit; every halo zero
    for blk in plan.blocks:
        if blk.s2d:
            out[blk.i]["xs"] = bitwise(interior(blk.xs, 0, 4 * blk.src.c), s2d(vint(blk.src)))
    bufs = {}
    for blk in plan.blocks:
        for v in (blk.src, blk.y if not blk.is_head else None):
            if v is not None and v.buf is not None:
                bufs[id(v.buf)] = v.buf
        if not blk.is_head:
            bufs[id(blk.z)] = blk.z
        if blk.s2d:
            bufs[id(blk.xs)] = blk.xs
    st.fwd_halo = all(halo_zero(b) for b in bufs.values())
    st.fwd = out
    st.max_ratio = max(ratios)


def check_block_bwd(st, blk, orig):
    """snapshot -> the production _backward_block -> checks; returns the results (never raises into autograd)"""
    plan, model = st.plan, st.model
    r = {}
    snap = {}
    try:
        if not blk.is_head:
            snap["z"] = interior(blk.z, 0, blk.cout).clone()
            snap["dy"], r["dy_mode"] = dy_of(plan, blk)
            if blk.i in st.keep_bwd and blk.fuse_up:
                snap["dy_shift"], _ = dy_of(plan, blk, shift=32)
            if blk.gres is not None:
                snap["gres_prior"] = vint(blk.gres).clone()
        if blk.gsrc is not None:
            snap["gbuf"] = blk.gsrc.buf.clone()
    except Exception:
        r["error"] = traceback.format_exc()
    orig(blk)
    if "error" in r:
        return r
    try:
        _bwd_checks(st, blk, snap, r)
    except Exception:
        r["error"] = traceback.format_exc()
    return r


def dz_checks(st, blk, snap, r):
    """the head cotangent's dz bit for bit, or bn_act_bwd of a BatchNorm block (dz, d beta, d gamma, d slope, the shortcut
    gradient); returns dz"""
    model = st.model
    if blk.is_head:
        dz = interior(blk.dz, 0, blk.cout)
        r["dz_bits"] = bitwise(dz, st.g_nhwc[blk.i].to(BF16))
        r["dz_pad_zero"] = bool((blk.dz[..., blk.cout:] == 0).all()) and halo_zero(blk.dz)
    else:
        dz = interior(blk.z, 0, blk.cout)
        chain = bn_chain(st.batch, blk.oh, blk.ow, blk.cout, 2 if r["dy_mode"] == 2 and blk.cout // 8 * 2 <= 640 else 1)
        rb, near = bn_bwd_check(snap["z"], snap["dy"], dz, blk.bsums, blk.mean, blk.invstd, blk.scale, blk.shift,
                                _slope_of(model, blk), chain)
        r["dz"], r["dz_bias"] = rb["max"], rb["bias"]
        for k in ("dbeta", "dgamma", "dslope"):
            r[k] = rb[k]
        r["near_zero_u"] = near
        r["n_elems"] = snap["z"].numel()
        if blk.i in st.keep_bwd:
            st.stash[("bn", blk.i)] = dict(z=snap["z"], dy=snap["dy"], dy_shift=snap.get("dy_shift"), dz=dz.clone(),
                                           sums=blk.bsums.clone(), mean=blk.mean.clone(), invstd=blk.invstd.clone(),
                                           sc=blk.scale.clone(), sh=blk.shift.clone(), slope=_slope_of(model, blk),
                                           chain=chain)
        if blk.gres is not None:
            d = snap["dy"]
            want = (snap["gres_prior"].float() + d).to(BF16) if blk.gres_acc else d.to(BF16)
            r["gres_bits"] = bitwise(vint(blk.gres), want)
        r["dz_halo"] = halo_zero(blk.z)
    return dz


def _bwd_checks(st, blk, snap, r):
    plan, model = st.plan, st.model
    w = _weight(model, blk)
    w64 = w.to(BF16).double()
    dz = dz_checks(st, blk, snap, r)
    # weight gradient (split-K layout) and its gather
    if blk.i == 0:
        x, offs, cin = interior(plan.col, 0, 27), [(0, 0)], 27
    elif blk.s2d:
        x, cin = interior(blk.xs, 0, blk.cin_eff), blk.cin_eff
        offs = [(qy - 1, qx - 1) for qy in range(2) for qx in range(2)]
    else:
        x, cin = vint(blk.src), blk.cin
        p = (blk.k - 1) // 2
        offs = [(kh - p, kw - p) for kh in range(blk.k) for kw in range(blk.k)]
    gh, gw_ = x.shape[1], x.shape[2]
    wr, wm = wgrad_ref(x, dz, offs)
    plan_w = wgrad_plan(blk.k_eff, blk.cin_pad, blk.cout_pad, st.batch, gh, gw_, wgrad_test.gemm_sms())
    got = blk.dw[:, :blk.cout, :cin]
    # test_wgrad's random-walk bound (KAPPA sqrt(n_add) 2^-24 A) is reported, not required: on the step's operands the
    # accumulator's truncations do not cancel
    r["wgrad"] = wgrad_ratio(got, wr, wm, plan_w)
    r["wgrad_rw"] = wgrad_test.worst_ratio(got, wr, wm, plan_w["n_add"])
    if blk.i in st.keep_bwd and blk.k == 3 and not blk.s2d:
        st.stash[("wgrad", blk.i)] = dict(x=x.clone(), dz=dz.clone(), offs=offs, got=got.clone(), plan=plan_w)
    del wr, wm
    if blk.i == 0:
        return
    # input gradient
    gbuf = blk.gsrc.buf
    allowed = torch.zeros(gbuf.shape[-1], dtype=torch.bool, device=gbuf.device)
    allowed[blk.gsrc.ch_off:blk.gsrc.ch_off + blk.gsrc.c] = True
    if blk.gres is not None and blk.gres.buf is gbuf:
        allowed[blk.gres.ch_off:blk.gres.ch_off + blk.gres.c] = True
    prior = interior(snap["gbuf"], blk.gsrc.ch_off, blk.gsrc.c)
    if blk.s2d:
        want, mag = s2d_dgrad_ref(dz, w64, blk.src.h, blk.src.w)
        n = 4 * rup(blk.cout, 64) // 16
        rd = check_z(interior(blk.dxs, 0, blk.cin_eff), want, mag, n)
        r["dgrad"], r["dgrad_bias"] = rd["max"], rd["bias"]
        del want, mag
        if blk.dxs_direct:
            allowed[:] = False
            if blk.gres is not None and blk.gres.buf is gbuf:
                allowed[blk.gres.ch_off:blk.gres.ch_off + blk.gres.c] = True
        else:
            v = d2s(interior(blk.dxs, 0, blk.cin_eff), blk.src.c)
            want_bits = (prior.float() + v.float()).to(BF16) if blk.gsrc_acc else v
            r["d2s_bits"] = bitwise(vint(blk.gsrc), want_bits)
    else:
        want, mag = tapsum(dz, conv_taps(w64, mirror=True), blk.src.h, blk.src.w)
        n = blk.k * blk.k * rup(blk.cout, 64) // 16
        e = n * 2.0 ** -23 * mag
        t = 0.0
        if blk.gsrc_acc:
            want = want + prior.double()
            t = U * (mag + prior.double().abs())
        got = vint(blk.gsrc)
        rd = bf16_check(got, want, e, t)
        r["dgrad"], r["dgrad_bias"] = rd["max"], rd["bias"]
        if blk.i in st.keep_bwd:
            st.stash[("dgrad", blk.i)] = dict(dz=dz.clone(), w64=w64, got=got.clone(), prior=prior.clone(),
                                              acc=blk.gsrc_acc, h=blk.src.h, w=blk.src.w, n=n,
                                              shifted=(interior(gbuf, blk.gsrc.ch_off - 32, blk.gsrc.c).clone()
                                                       if blk.gsrc.ch_off >= 32 else None))
        del want, mag
    outside = ~allowed
    r["outside_untouched"] = torch.equal(gbuf[..., outside], snap["gbuf"][..., outside]) and halo_zero(gbuf)


def _keep_sets(plan):
    """blocks whose tensors the bound self-test reuses: small grids only"""
    bl = plan.blocks
    k3 = [b for b in bl if b.k == 3 and not b.s2d and b.i > 0]
    acc1 = [b for b in bl if b.k == 1 and not b.s2d and not b.is_head and b.gsrc_acc]
    res = [b for b in bl if b.fuse_res]
    up = [b for b in bl if b.fuse_up and b.gy.ch_off + 32 + b.cout <= b.gy.cs]
    st_fwd = {res[-1].i}
    st_bwd = {k3[-1].i, acc1[-1].i, up[0].i}
    return st_fwd, st_bwd, dict(k3=k3[-1].i, acc1=acc1[-1].i, res=res[-1].i, up=up[0].i)


@pytest.fixture(scope="module")
def step():
    pkg = _pkg()
    from rotate_yolov3_b200 import cfgs
    t0 = time.time()
    dev = torch.device("cuda")
    model = pkg.Darknet(cfgs.yolov3_cfg(), {"context_factor": 1.0}, arc="default")
    init_darknet_weights(model, seed=1)
    model = model.to(dev).train()
    st = Step()
    st.model = model
    st.x = torch.rand(BATCH, 3, SIZE, SIZE, generator=torch.Generator().manual_seed(2)).to(dev)
    st.rm0, st.rv0, nbt0 = {}, {}, {}
    for i, m in enumerate(model.module_list):
        if hasattr(m, "BatchNorm2d"):
            st.rm0[i] = m.BatchNorm2d.running_mean.clone()
            st.rv0[i] = m.BatchNorm2d.running_var.clone()
            nbt0[i] = int(m.BatchNorm2d.num_batches_tracked)
    ps = model(st.x)
    torch.cuda.synchronize()
    plan = model._tplan
    st.plan = plan
    st.keep_fwd, st.keep_bwd, st.picks = _keep_sets(plan)
    st.stash = {}
    st.nbt_ok = all(int(model.module_list[i].BatchNorm2d.num_batches_tracked) == nbt0[i] + 1 for i in nbt0)
    forward_checks(st)
    torch.cuda.synchronize()
    st.t_fwd = time.time() - t0
    # dense head cotangents
    gen = torch.Generator().manual_seed(3)
    gs = [torch.randn(p.shape, generator=gen).to(dev) for p in ps]
    st.g_nhwc = {}
    for blk, g in zip(plan.heads, gs):
        b, na, ny, nx, no = g.shape
        st.g_nhwc[blk.i] = g.permute(0, 2, 3, 1, 4).reshape(b, ny, nx, na * no)     # channel a * no + k
    loss = sum((p * g).sum() for p, g in zip(ps, gs))
    st.bwd = {}
    orig = plan._backward_block

    def wrapped(blk):
        st.bwd[blk.i] = check_block_bwd(st, blk, orig)
    plan._backward_block = wrapped
    try:
        loss.backward()
    finally:
        del plan._backward_block
    torch.cuda.synchronize()
    # head bias gradients and the weight-gradient gathers (the unpack runs at the end of the backward segment)
    L = _layout()
    for blk in plan.blocks:
        r = st.bwd.setdefault(blk.i, {})
        if blk.is_head:
            g = st.g_nhwc[blk.i].double()
            gb = plan.garena[blk.gb_off:blk.gb_off + blk.cout]
            r["dbias"] = sum_check(gb, g.sum((0, 1, 2)), head_bias_chain(BATCH, blk.oh, blk.ow), g.abs().sum((0, 1, 2)))
        if blk.i == 0:
            want = blk.dw[0, :blk.cout, :27].reshape(blk.cout, 3, 3, 3)
        elif blk.s2d:
            c = blk.src.c
            d2 = blk.dw[:, :blk.cout, :4 * c].permute(1, 2, 0).reshape(blk.cout, 4 * c, 2, 2)
            want = L.s2d_weight_grad(d2, c)
        else:
            want = blk.dw[:, :blk.cout, :blk.cin].reshape(blk.k, blk.k, blk.cout, blk.cin).permute(2, 3, 0, 1)
        r["gw_bits"] = torch.equal(blk.gw, want)
    st.t_total = time.time() - t0
    _print_table(st)
    return st


def _print_table(st):
    print("\n[train608] forward %.1f s, whole step with checks %.1f s; largest |mean| / std of z: %.2f"
          % (st.t_fwd, st.t_total, st.max_ratio))
    print("[train608] worst |err| / bound per kernel (z: conv, y: bn_act_fwd, dz: bn_act_bwd, dgrad, wgrad)")
    for blk in st.plan.blocks:
        f, b = st.fwd[blk.i], st.bwd.get(blk.i, {})
        kind = "head" if blk.is_head else ("s2d" if blk.s2d else "k%d" % blk.k)
        cols = ["%-4s" % kind, "%4d" % blk.cout, "%3d^2" % blk.oh]
        for key, src in (("z", f), ("z_bias", f), ("mean", f), ("invstd", f), ("y", f), ("y_bias", f), ("dz", b),
                         ("dz_bias", b), ("dbeta", b), ("dgamma", b), ("dslope", b), ("wgrad", b), ("dgrad", b),
                         ("dgrad_bias", b), ("dbias", b), ("wgrad_rw", b)):
            if key in src:
                cols.append("%s %.3f" % (key, src[key]))
        if "mean_over_std" in f:
            cols.append("|m|/s %.2f" % f["mean_over_std"])
        print("[train608] %3d " % blk.i + "  ".join(cols))


# ---------------------------------------------------------------------------------------------------------------
def test_covers_the_whole_step(step):
    plan = step.plan
    assert len(plan.blocks) == 75
    assert sum(b.is_head for b in plan.blocks) == 3 and all(b.cout == 504 for b in plan.blocks if b.is_head)
    assert sorted({b.gsrc.cs for b in plan.blocks if b.gsrc is not None and b.gsrc.cs > b.gsrc.c}) == [384, 768]
    assert all(b.s2d for b in plan.blocks if b.stride == 2)       # the zero-insert fallback never runs at 608
    assert len(step.fwd) == 75 and len([i for i, r in step.bwd.items() if "wgrad" in r]) == 75
    assert all("error" not in r for r in step.bwd.values()), [r["error"] for r in step.bwd.values() if "error" in r][:1]


def test_im2col_and_weight_pack_bitwise(step):
    assert step.im2col == dict(bits=True, pad_zero=True, halo=True), step.im2col
    assert len(step.packs) == 149
    bad = [p[:2] for p in step.packs if not p[2]]
    assert not bad, bad


def test_forward_kernels_vs_float64(step):
    assert step.nbt_ok and step.fwd_halo
    bad = []
    for i, r in step.fwd.items():
        for k, v in r.items():
            if k == "mean_over_std":
                continue
            if (isinstance(v, bool) and not v) or (isinstance(v, float) and not v <= 1.0):     # NaN fails
                bad.append((i, k, v))
    assert not bad, bad


def test_backward_kernels_vs_float64(step):
    bad = []
    for i, r in step.bwd.items():
        assert "error" not in r, r["error"]
        for k, v in r.items():
            if k in ("dy_mode", "near_zero_u", "n_elems", "wgrad_rw"):
                continue
            if (isinstance(v, bool) and not v) or (isinstance(v, float) and not v <= 1.0):     # NaN fails
                bad.append((i, k, v))
        if "near_zero_u" in r:                # the PReLU branch is ambiguous on a tiny set only
            assert r["near_zero_u"] <= max(64, r["n_elems"] // 100000), (i, r["near_zero_u"])
    assert not bad, bad
    modes = {r["dy_mode"] for r in step.bwd.values() if "dy_mode" in r}
    assert modes == {0, 1, 2}, modes
    acc = [b for b in step.plan.blocks if b.gsrc is not None and b.gsrc_acc]
    assert acc and any(b.s2d and not b.dxs_direct for b in step.plan.blocks)


def bn_stats_errors(ratios, seed):
    """ryolo_bn_stats_finalize alone on bf16 z [64, 304, 304, 32] (5.9 M pixels per channel), 8 channels per |mean| / std
    in `ratios` (std 0.5 .. 3, both signs): per group the worst invstd relative error and mean error / std against the
    two-pass float64 statistics"""
    lib = _pkg()._lib
    dev = torch.device("cuda")
    b, h, w, c = 64, 304, 304, 32
    g = torch.Generator(device=dev).manual_seed(seed)
    std = torch.tensor([0.5, 1.0, 1.5, 3.0] * 2, dtype=F64, device=dev).repeat(4)
    sign = torch.tensor([1.0, -1.0] * 4, dtype=F64, device=dev).repeat(4)
    mu = torch.tensor(ratios, dtype=F64, device=dev).repeat_interleave(8) * std * sign
    z = torch.zeros((b, h + 2, w + 2, c), dtype=BF16, device=dev)
    for i in range(b):
        z[i, 1:-1, 1:-1] = (torch.randn(h, w, c, generator=g, device=dev, dtype=torch.float32) * std.float()
                            + mu.float()).to(BF16)
    s1 = torch.zeros(c, dtype=F64, device=dev)
    for i in range(b):
        s1 += z[i, 1:-1, 1:-1].double().sum((0, 1))
    m64 = s1 / (b * h * w)
    s2 = torch.zeros(c, dtype=F64, device=dev)
    for i in range(b):
        s2 += (z[i, 1:-1, 1:-1].double() - m64).pow(2).sum((0, 1))
    v64 = s2 / (b * h * w)
    eps = 1e-5
    sums = torch.zeros(2 * c, device=dev)
    gamma, beta = torch.ones(c, device=dev), torch.zeros(c, device=dev)
    outs = [torch.zeros(c, device=dev) for _ in range(4)]
    rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
    st_ = lib.lib.ryolo_bn_stats_finalize(lib.ptr(z), c, b, h, w, c, lib.ptr(sums), eps, MOMENTUM_DEFAULT, lib.ptr(gamma),
                                          lib.ptr(beta), *[lib.ptr(t) for t in outs], lib.ptr(rm), lib.ptr(rv), lib.stream_ptr())
    assert st_ == 0, lib.last_error()
    torch.cuda.synchronize()
    sd = (v64 + eps).sqrt()
    e_inv = (outs[1].double() * sd - 1.0).abs()
    e_mean = (outs[0].double() - m64).abs() / sd
    return [(float(e_inv[8 * k:8 * k + 8].max()), float(e_mean[8 * k:8 * k + 8].max())) for k in range(len(ratios))]


def test_bn_statistics_at_the_benchmark_count(step):
    """the one-pass fp32 variance at the benchmark's 5.9 M pixels per channel, |mean| / std in {0, 2, 8, 32}; the target
    is required up to ratio 8 or twice the largest ratio of the 608 step (that ratio itself is run as well)"""
    ratios = [0.0, 2.0, 8.0, 32.0]
    need = max(8.0, 2.0 * step.max_ratio)
    errs = bn_stats_errors(ratios, 7)
    if need > 8.0:
        ratios.append(need)
        errs.append(bn_stats_errors([need] * 4, 8)[0])
    for r, (ei, em) in zip(ratios, errs):
        print("[bn_stats 5.9M] |mean|/std %5.2f: invstd rel. error %.2e, mean error / std %.2e  (target %.2e)"
              % (r, ei, em, STAT_TOL))
    print("[bn_stats 5.9M] largest |mean|/std of the 608 step: %.2f -> required up to %.2f" % (step.max_ratio, need))
    for r, (ei, em) in zip(ratios, errs):
        if r <= need:
            assert ei <= STAT_TOL and em <= STAT_TOL, (r, ei, em)


def test_bounds_reject_plausible_bugs(step):
    """each check, applied to a reference (or stored tensor) with one plausible bug put in, fails"""
    st = step
    pk = st.picks
    # dgrad: one tap dropped / taps not mirrored (a 3x3 block), accumulate flag inverted (a 1x1 block that accumulates)
    d = st.stash[("dgrad", pk["k3"])]

    def dgrad_ratio(dd, taps, with_prior, got=None):
        want, mag = tapsum(dd["dz"], taps, dd["h"], dd["w"])
        e, t = dd["n"] * 2.0 ** -23 * mag, 0.0
        if with_prior:
            want = want + dd["prior"].double()
            t = U * (mag + dd["prior"].double().abs())
        return bf16_check(dd["got"] if got is None else got, want, e, t)
    assert passed(dgrad_ratio(d, conv_taps(d["w64"], mirror=True), d["acc"]))
    r1 = dgrad_ratio(d, conv_taps(d["w64"], mirror=True, drop=(0, 0)), d["acc"])
    r2 = dgrad_ratio(d, conv_taps(d["w64"], mirror=True, flip=False), d["acc"])
    a = st.stash[("dgrad", pk["acc1"])]
    assert a["acc"] and passed(dgrad_ratio(a, conv_taps(a["w64"], mirror=True), True))
    r3 = dgrad_ratio(a, conv_taps(a["w64"], mirror=True), False)
    # the up-sampling block reads its gradient from a slice of a concat buffer: 32 channels off
    u = st.stash[("bn", pk["up"])]
    args = (u["dz"], u["sums"], u["mean"], u["invstd"], u["sc"], u["sh"], u["slope"], u["chain"])
    assert passed(bn_bwd_check(u["z"], u["dy"], *args)[0])
    r4 = bn_bwd_check(u["z"], u["dy_shift"], *args)[0]
    # residual added twice
    y = st.stash[("y", pk["res"])]
    want, t = bn_act_fwd_ref(y["z"], y["sc"], y["sh"], y["slope"], y["res"])
    assert passed(bf16_check(y["got"], want, 0.0, t))
    r5 = bf16_check(y["got"], want + y["res"].double(), 0.0, t)
    # round-toward-zero bf16 conversion of z: the bias bound catches it
    zc = st.stash[("z", pk["res"])]
    v32 = zc["want"].float()
    assert passed(check_z(v32.to(BF16), zc["want"], zc["mag"], zc["n"]))
    r6 = check_z(rtz_bf16(v32), zc["want"], zc["mag"], zc["n"])
    # running variance with n instead of n - 1, applied on every BN block of the step (forward_checks): the worst block
    r7 = max(st.rv_biased.values())
    n7 = sum(v > 1.0 for v in st.rv_biased.values())
    # BN dz without the m2 term
    k = st.stash[("bn", pk["k3"])]
    r8 = bn_bwd_check(k["z"], k["dy"], k["dz"], k["sums"], k["mean"], k["invstd"], k["sc"], k["sh"], k["slope"], k["chain"],
                      drop_m2=True)[0]
    # weight gradient: one whole split-K partial lost (the middle split of a 76^2 3x3 layer)
    wg = st.stash[("wgrad", pk["k3"])]
    pw = wg["plan"]
    assert pw["ksplit"] > 1, pw
    want, mag = wgrad_ref(wg["x"], wg["dz"], wg["offs"])
    assert wgrad_ratio(wg["got"], want, mag, pw) <= 1.0
    b, h, w = wg["dz"].shape[:3]
    flat = torch.zeros(b * (h + 2) * (w + 2), dtype=F64, device=want.device)
    j = pw["ksplit"] // 2
    flat[64 * j * pw["per_split"]:64 * (j + 1) * pw["per_split"]] = 1.0
    mask = flat.view(b, h + 2, w + 2)[:, 1:-1, 1:-1, None]
    lost, _ = wgrad_ref(wg["x"], wg["dz"].double() * mask, wg["offs"])
    r9 = {"max": wgrad_ratio(wg["got"], want - lost, mag, pw)}
    # one NaN in an otherwise correct output (a stale or unwritten element) fails the check
    zn = zc["got"].clone()
    zn.view(-1)[zn.numel() // 3] = float("nan")
    r10 = check_z(zn, zc["want"], zc["mag"], zc["n"])
    found = dict(dropped_tap=r1, unmirrored=r2, lost_accumulate=r3, concat_off_by_32=r4, residual_twice=r5, rtz_z=r6,
                 running_var_biased=r7, dz_without_m2=r8, lost_split=r9, nan_in_z=r10)
    for name, r in found.items():
        print("[bite] %-18s %s" % (name, r if isinstance(r, float) else {k_: round(v, 3) for k_, v in r.items()
                                                                            if isinstance(v, float)}))
    assert r6["bias"] > 1.0, r6
    print("[bite] biased running variance fails on %d of %d BN blocks" % (n7, len(st.rv_biased)))
    assert r7 > 1.0, r7
    for name in ("dropped_tap", "unmirrored", "lost_accumulate", "concat_off_by_32", "residual_twice", "dz_without_m2",
                 "lost_split", "nan_in_z"):
        assert not passed(found[name]), (name, found[name])
