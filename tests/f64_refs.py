"""TEST INFRASTRUCTURE: the float64 references, rounding bounds and layout helpers that the kernel-against-float64 tests
share (test_train_step_f64_gpu.py, test_dilated_train_f64_gpu.py, test_multiclass_f64_gpu.py,
test_detect_forward_f64_gpu.py, test_parity_step_f64_gpu.py, test_se_f64_gpu.py, test_parity_bwd_gpu.py,
test_wgrad_gpu.py and their neighbours).  Each bound is stated in the docstring of the test file that introduced it.

Every check returns worst |err| / bound (and the bias over its bound); <= 1 passes, and a NaN ratio fails."""
import ctypes
import math

import torch
import torch.nn.functional as F

from builders import ryolo_lib
from helpers import wgrad_plan

U = 2.0 ** -24
HALF_BF16 = 2.0 ** -8
BIAS_TOL = 2.0 ** -12
STAT_TOL = 2.0 ** -12
TINY = 1e-30
KAPPA = 1.0
F64 = torch.float64
BF16 = torch.bfloat16


def gemm_sms(reserved=0):
    """the SM count the GEMM launches plan for (the library's rule for ryolo_set_reserved_sms)"""
    n = torch.cuda.get_device_properties(0).multi_processor_count
    return n - reserved if n - reserved > 8 else n


# ---------------------------------------------------------------------------------------------------------------
# layouts
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


def bitwise(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def d2s(dxs, c):
    """depth_to_space of the interior of an s2d buffer: [B, h, w, 4c] -> [B, 2h, 2w, c]"""
    b, h, w, _ = dxs.shape
    t = dxs[..., :4 * c].reshape(b, h, w, 2, 2, c)
    return t.permute(0, 1, 3, 2, 4, 5).reshape(b, 2 * h, 2 * w, c)


def s2d(x):
    """space_to_depth: [B, 2h, 2w, c] -> [B, h, w, 4c], channel (py * 2 + px) * c + ci"""
    b, hh, ww, c = x.shape
    return x.reshape(b, hh // 2, 2, ww // 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(b, hh // 2, ww // 2, 4 * c)


def nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def rtz_bf16(v32):
    """round-toward-zero fp32 -> bf16 (drop the low 16 bits)"""
    return (v32.contiguous().view(torch.int32) & -65536).view(torch.float32).to(BF16)


def bf(t):
    """t rounded to bf16, as fp32"""
    return t.to(torch.bfloat16).float()


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


# the dilated and stride-2 convs of yolov3-m: tap sums of shifted NHWC operands (value, magnitude)
def dil_conv(x, w64, dh, dw, adjoint=False):
    """the 3x3 conv with dilation and padding (dh, dw) of NHWC x with weight [cout, cin, 3, 3]; adjoint: its input
    gradient from dz (taps mirrored, W not transposed)"""
    b, h, wd, c = x.shape
    xp = F.pad(x.double(), (0, 0, dw, dw, dh, dh))
    xa = xp.abs()
    n = w64.shape[1] if adjoint else w64.shape[0]
    out = torch.zeros(b * h * wd, n, dtype=F64, device=x.device)
    mag = torch.zeros_like(out)
    for kh in range(3):
        for kw in range(3):
            oy, ox = (kh - 1) * dh, (kw - 1) * dw
            m = w64[:, :, kh, kw] if adjoint else w64[:, :, kh, kw].t()
            if adjoint:
                oy, ox = -oy, -ox
            sl = (slice(None), slice(dh + oy, dh + oy + h), slice(dw + ox, dw + ox + wd))
            out.addmm_(xp[sl].reshape(-1, c), m)
            mag.addmm_(xa[sl].reshape(-1, c), m.abs())
    return out.view(b, h, wd, n), mag.view(b, h, wd, n)


def dil_wgrad_ref(x, dz, dh, dw):
    """dW[kh * 3 + kw, co, ci] = sum_p dz(p, co) x(p + (dh (kh - 1), dw (kw - 1)), ci): value and magnitude"""
    b, h, wd, cin = x.shape
    xp = F.pad(x.double(), (0, 0, dw, dw, dh, dh))
    d = dz.double().reshape(-1, dz.shape[3])
    da = d.abs()
    outs, mags = [], []
    for kh in range(3):
        for kw in range(3):
            a = xp[:, kh * dh:kh * dh + h, kw * dw:kw * dw + wd].reshape(-1, cin)
            outs.append(d.t() @ a)
            mags.append(da.t() @ a.abs())
    return torch.stack(outs), torch.stack(mags)


def s2_refs(x, dz, w64):
    """3x3 / stride 2 / pad 1 conv on the odd grid of x: torch's float64 weight gradient in the kernel's [t, co, ci]
    layout and the input gradient (conv_transpose2d, output padding up to x's size), each with its magnitude"""
    x64, d64 = nchw(x.double()), nchw(dz.double())
    h, w = x.shape[1], x.shape[2]
    op = (h - (2 * dz.shape[1] - 1), w - (2 * dz.shape[2] - 1))
    shape = tuple(w64.shape)

    def gw(a, d):
        return torch.nn.grad.conv2d_weight(a, shape, d, stride=2, padding=1).permute(2, 3, 0, 1).reshape(9, shape[0],
                                                                                                         shape[1])

    def dx(d, ww):
        return nhwc(F.conv_transpose2d(d, ww, stride=2, padding=1, output_padding=op))
    return gw(x64, d64), gw(x64.abs(), d64.abs()), dx(d64, w64), dx(d64.abs(), w64.abs())


def yolov3_heads(nc):
    """(anchors [na, 3] in pixels, grid, stride) of the three heads of the 608x608 yolov3 cfg, in output row order"""
    from rotate_yolov3_b200 import cfgs
    from rotate_yolov3_b200.parse_config import parse_model_cfg
    heads = []
    for mdef, ng in zip([m for m in parse_model_cfg(cfgs.yolov3_cfg(classes=nc)) if m["type"] == "yolo"], (19, 38, 76)):
        lo, hi = [int(v) for v in mdef["mask"].split("-")]
        heads.append((torch.tensor(mdef["anchors"][lo:hi + 1], dtype=torch.float32), ng, 608 / ng))
    return heads


def decode_ref(p, anchors, stride, ctx, nc):
    """float64 model/models.py:198-227 ('default' arc): returns (io [B, na*ny*nx, 6+nc], per-component magnitude M)"""
    bs, _, ny, nx = p.shape
    na = anchors.shape[0]
    t = p.double().view(bs, na, nc + 6, ny, nx).permute(0, 1, 3, 4, 2)
    a = anchors.double().to(p.device)
    aw = (a[:, 0] / stride).view(1, na, 1, 1)
    ah = (a[:, 1] / stride).view(1, na, 1, 1)
    at = a[:, 2].view(1, na, 1, 1)
    gx = torch.arange(nx, device=p.device, dtype=torch.float64).view(1, 1, 1, nx)
    gy = torch.arange(ny, device=p.device, dtype=torch.float64).view(1, 1, ny, 1)
    sx, sy = torch.sigmoid(t[..., 0]), torch.sigmoid(t[..., 1])
    w0 = torch.exp(t[..., 2]) * aw * stride
    h = torch.exp(t[..., 3]) * ah * stride / ctx
    th = torch.atan(t[..., 4])
    want = [(sx + gx) * stride, (sy + gy) * stride, w0 - h * (ctx - 1), h, th + at]
    mag = [(sx.abs() + gx) * stride, (sy.abs() + gy) * stride, w0.abs() + (h * (ctx - 1)).abs(), h.abs(),
           th.abs() + at.abs()]
    for k in range(5, nc + 6):
        s = torch.ones_like(sx) if (nc == 1 and k == 6) else torch.sigmoid(t[..., k])
        want.append(s)
        mag.append(s.abs())
    flat = lambda xs: torch.stack(xs, -1).reshape(bs, na * ny * nx, nc + 6)
    return flat(want), flat(mag)


# ---------------------------------------------------------------------------------------------------------------
# bounds
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


def check_z(got, want, mag, n):
    return bf16_check(got, want, n * 2.0 ** -23 * mag)


def passed(r):
    """every ratio <= 1 (a NaN ratio fails) and every flag true"""
    return all((v <= 1.0) if isinstance(v, float) else v for v in r.values() if isinstance(v, (float, bool)))


def worst_ratio(got, want, mag, n_add, extra=None):
    """max over entries of |got - want| / bound; <= 1 everywhere means the kernel is within the float64 bound"""
    bound = KAPPA * math.sqrt(n_add) * U * mag + TINY
    if extra is not None:
        bound = bound + extra
    return float(((got.double() - want).abs() / bound).max())


def wgrad_ratio(got, want, mag, plan):
    """split-K weight gradient: one fp32 ulp of the magnitude per update of the longest chain -- the updates of one split
    plus the ksplit partials added in split order -- and half an ulp of the fp32 result"""
    n = plan["updates"] + plan["ksplit"]
    return worst_ratio(got, want, mag, 0, extra=n * 2.0 ** -23 * mag + U * want.abs())


def bad_entries(d, skip=("dy_mode", "near_zero_u", "n_elems", "wgrad_rw", "mean_over_std")):
    """(block, key, value) of every failing entry of per-block results: an error, a ratio above 1 (or NaN), a False flag"""
    out = []
    for i, r in d.items():
        for k, v in r.items():
            if k == "error":
                out.append((i, k, v[-600:]))
            elif k in skip:
                continue
            elif (isinstance(v, bool) and not v) or (isinstance(v, float) and not v <= 1.0):
                out.append((i, k, v))
    return out


# ---------------------------------------------------------------------------------------------------------------
# reduction chain lengths
def bn_pieces(batch, h, w, c, rows_per_piece=1, sms=None):
    """the piece schedule of bn_stats / bn_act_bwd (mirror of mk_pieces in bnpipe.cuh): pieces of `px` pixels of
    `rows_per_piece` rows, `per_cta` of them per CTA of a `grid`-CTA launch"""
    cgs = c // 8
    max_px = 1280 // rows_per_piece // cgs
    if rows_per_piece == 2:
        max_px &= ~1
    ppr = cdiv(w, max_px)
    px = cdiv(w, ppr)
    if rows_per_piece == 2 and px % 2:
        px += 1
    total = batch * (h // rows_per_piece) * ppr
    per_cta = cdiv(total, 2 * (sms or gemm_sms()))
    return dict(px=px, total=total, per_cta=per_cta, grid=cdiv(total, per_cta), rows=rows_per_piece)


def bn_chain(batch, h, w, c, rows_per_piece=1, sms=None):
    """bn_stats / bn_act_bwd: the longest fp32 addition chains of the channel sums and of d slope"""
    pg = bn_pieces(batch, h, w, c, rows_per_piece, sms)
    per_thread = pg["per_cta"] * cdiv(pg["px"] * (c // 8), 256) * rows_per_piece
    rows = cdiv(pg["grid"], 8) + 8
    return dict(sums=per_thread + 256 // (c // 8) + rows, slope=8 * per_thread + 5 + 8 + rows)


def head_bias_blocks(batch, ny):
    """head_grad_nchw_kernel: (rows per block, blocks)"""
    rpb = max(1, cdiv(ny * batch, 2048))
    return rpb, cdiv(ny, rpb) * batch


def head_bias_chain(batch, ny, nx):
    rpb, blocks = head_bias_blocks(batch, ny)
    return 5 + rpb * cdiv(nx, 32) + cdiv(blocks, 8) + 8 + 1


def conv_schedule(np_, cout, res, sms=None):
    """the persistent implicit-GEMM launch (conv.cu conv_geom / launch_conv / ConvSmem) over np_ padded pixels: its
    tiles, grid and tiles per CTA, the operand ring and the output staging tiles a CTA cycles through"""
    bn = 256 if cout > 128 else (128 if cout > 64 else 64)
    tiles = cdiv(np_, 128) * (rup(cout, bn) // bn)
    grid = min(tiles, sms or gemm_sms())
    return dict(bn=bn, tiles=tiles, grid=grid, per_cta=cdiv(tiles, grid),
                stages=3 if bn == 256 else ((5 if res else 6) if bn == 128 else 8),
                staging=2 if res and bn < 256 else 1, m_tail=np_ % 128)


def se_chain(h, w, c):
    """longest fp32 addition chain of se_partial_kernel + the span sum (csrc/se.cu se_nsplit)"""
    items = h * w * (c // 8)
    nsplit = max(1, min(128, -(-items // 4096)))
    span = -(-(h * w) // nsplit)
    lanes = 256 // (c // 8)
    return -(-span // lanes) + lanes + nsplit


def se_block_chain(h, w, c):
    """longest fp32 addition chain of the in-place eval SE's channel sums (csrc/se.cu se_pool_kernel): the pixels one
    thread adds over its rows, then one atomicAdd per thread and row block in any order"""
    rpb = -(-h // 64) if h > 64 else 1
    pstep = 256 // (c // 8)
    return rpb * -(-w // pstep) + pstep * -(-h // rpb)


# ---------------------------------------------------------------------------------------------------------------
# squeeze-excitation: float64 references of ryolo_se_fwd / ryolo_se_bwd on the kernels' own inputs.  se carries h, w, c,
# cr and the kernels' fp32 outputs m, p, s (ds, dm for the backward) as flat [B * c] / [B * cr] tensors.
def ratio(got, want, bound):
    return float(((got.double() - want).abs() / (bound + TINY)).max())


def se_fwd_refs(se, x, w1, w2):
    """float64 references of the forward outputs from the kernels' own inputs; returns {name: (ref, bound)}"""
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


def se_bwd_refs(se, gu, x, gx_old, w1, w2, gw1, gw2):
    """float64 references of ryolo_se_bwd's outputs from its own inputs (gx_old: the prior gx it accumulates onto, None
    when it writes first); returns {name: (ref, bound)}"""
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


def se_fwd_ratios(se, x, u, w1, w2):
    """ryolo_se_fwd's m, p, s and u against se_fwd_refs: {name: worst ratio}, u with its rounding-bias ratio"""
    B = x.shape[0]
    refs = se_fwd_refs(se, x, w1, w2)
    r = dict(m=ratio(se.m.view(B, se.c), *refs["m"]), p=ratio(se.p.view(B, se.cr), *refs["p"]),
             s=ratio(se.s.view(B, se.c), *refs["s"]))
    r.update({"u_" + k: v for k, v in bf16_check(u, *refs["u"]).items()})
    return r, refs


def se_block_s_ref(sums, w1, w2, hw):
    """ryolo_se_block's scale from its own fp32 channel sums [B, c]: mean = sums * fp32(1 / hw) (2 U), p = W1 mean
    ((c + 1) U |W1| |mean|, carried through W2 with the mean's 2 U), s = sigmoid(W2 relu(p)) as in the SE bounds;
    returns (s, bound)"""
    c, cr = w1.shape[1], w1.shape[0]
    m = sums.double() / hw
    p_err = (c + 3) * U * (m.abs() @ w1.abs().t())
    hid = (m @ w1.t()).clamp(min=0)
    s64 = torch.sigmoid(hid @ w2.t())
    s_b = s64 * (1 - s64) * ((cr + 1) * U * ((hid + p_err) @ w2.abs().t()) + p_err @ w2.abs().t()) + 4 * U * s64
    return s64, s_b


# ---------------------------------------------------------------------------------------------------------------
# the bf16 weight gradient (csrc/wgrad.cu) on one set of operands
def wgrad(dzb, zcs, cout_pad, xb, xcs, cin_pad, b, h, w, k, dw, stream=None):
    L = ryolo_lib()
    sp = ctypes.c_void_p(stream.cuda_stream) if stream is not None else L.stream_ptr(dw.device)
    st = L.lib.ryolo_conv_wgrad(L.ptr(dzb), zcs, cout_pad, L.ptr(xb), xcs, cin_pad, b, h, w, k, L.ptr(dw), sp)
    assert st == 0, L.last_error()


def ref_wgrad(x, dz, k, stride=1):
    """float64 weight gradient of the k x k conv (k = 2: taps at offsets -1..0, the space-to-depth form) and its magnitude"""
    x64, dz64 = x.double(), dz.double()
    if k == 2:
        shape = (dz.shape[1], x.shape[1], 2, 2)
        f = lambda a, d: torch.nn.grad.conv2d_weight(F.pad(a, (1, 0, 1, 0)), shape, d, stride=1, padding=0)
    else:
        shape = (dz.shape[1], x.shape[1], k, k)
        f = lambda a, d: torch.nn.grad.conv2d_weight(a, shape, d, stride=stride, padding=(k - 1) // 2)
    return f(x64, dz64), f(x64.abs(), dz64.abs())


def unpacked(dw, k, cout_pad, cin_pad, cout, cin):
    return dw.view(k, k, cout_pad, cin_pad)[:, :, :cout, :cin].permute(2, 3, 0, 1)


def s2d_nchw(x):
    """space-to-depth of an NCHW tensor: channel (py * 2 + px) * C + c holds pixel (2Y + py, 2X + px)"""
    return torch.cat([x[:, :, py::2, px::2] for py in range(2) for px in range(2)], 1)


class Case:
    """one wgrad launch: operands in padded NHWC, their float64 reference and the mirrored launch plan"""

    def __init__(self, batch, h, w, cout, ksize, cin=None, s2d_c=None, narrow=False, seed=0):
        from rotate_yolov3_b200 import layout as L
        dev = torch.device("cuda")
        g = torch.Generator().manual_seed(seed)
        self.b, self.k = batch, ksize
        if s2d_c is not None:        # 3x3/stride-2 layer on a [b, C, 2h, 2w] input, in its space-to-depth form
            self.x_full = bf(torch.randn(batch, s2d_c, 2 * h, 2 * w, generator=g)).to(dev)
            self.x = s2d_nchw(self.x_full)
            cin = 4 * s2d_c
        else:
            self.x = bf(torch.randn(batch, cin, h, w, generator=g)).to(dev)
        self.h, self.w, self.cin, self.cout = h, w, cin, cout
        self.dz = bf(torch.randn(batch, cout, h, w, generator=g)).to(dev)
        self.cin_pad = L.round_up(cin, 64)
        self.cout_pad = L.round_up(cout, 64 if cout <= 64 else (128 if cout <= 128 else 256))
        self.xcs = L.round_up(cin, 32) if narrow else self.cin_pad
        self.zcs = L.round_up(cout, 32) if narrow else self.cout_pad
        if s2d_c is not None:        # built by the library's own space-to-depth kernel, as the training step does
            xf = L.to_padded_nhwc(self.x_full, L.round_up(s2d_c, 64))
            self.xb = L.alloc_padded(batch, h, w, self.xcs, dev)
            L_ = ryolo_lib()
            st = L_.lib.ryolo_space_to_depth(L_.ptr(xf), xf.shape[-1], batch, 2 * h, 2 * w, s2d_c, L_.ptr(self.xb),
                                             self.xcs, L_.stream_ptr(dev))
            assert st == 0, L_.last_error()
        else:
            self.xb = L.to_padded_nhwc(self.x, self.xcs)
        self.dzb = L.to_padded_nhwc(self.dz, self.zcs)
        self._ref = None

    def plan(self, reserved=0):
        return wgrad_plan(self.k, self.cin_pad, self.cout_pad, self.b, self.h, self.w, gemm_sms(reserved))

    def ref(self):
        if self._ref is None:
            self._ref = ref_wgrad(self.x, self.dz, self.k)
        return self._ref

    def new_dw(self, fill=None):
        shape = (self.k * self.k, self.cout_pad, self.cin_pad)
        if fill is None:
            return torch.zeros(shape, dtype=torch.float32, device="cuda")
        return fill.clone()

    def run(self, dw, stream=None):
        wgrad(self.dzb, self.zcs, self.cout_pad, self.xb, self.xcs, self.cin_pad, self.b, self.h, self.w, self.k, dw, stream)
        return dw

    def got(self, dw):
        return unpacked(dw, self.k, self.cout_pad, self.cin_pad, self.cout, self.cin)


# (case kwargs, expected plan: bn, tg always; ksplit and a short last split on a 132-SM H100 SXM)
CASES = {
    "k3_c64_tg3": (dict(batch=4, h=76, w=76, cin=64, cout=64, ksize=3), dict(bn=64, tg=3, ksplit=24, short_last=True, last=13)),
    "k3_c128_tg1": (dict(batch=2, h=76, w=76, cin=128, cout=64, ksize=3), dict(bn=128, tg=1, ksplit=12, short_last=True)),
    "s2d_c32_tg2": (dict(batch=4, h=38, w=38, s2d_c=32, cout=64, ksize=2), dict(bn=128, tg=2, ksplit=7, short_last=True)),
    "s2d_c16_tg2": (dict(batch=4, h=38, w=38, s2d_c=16, cout=64, ksize=2), dict(bn=64, tg=2, ksplit=7)),
    "s2d_c64_bn256": (dict(batch=2, h=38, w=38, s2d_c=64, cout=128, ksize=2), dict(bn=256, tg=1, ksplit=4, short_last=True)),
    "k1_c768_3n2m": (dict(batch=2, h=38, w=38, cin=768, cout=256, ksize=1), dict(bn=256, tg=1, ksplit=4, tiles=6)),
    "k3_narrow32": (dict(batch=2, h=40, w=40, cin=32, cout=32, ksize=3, narrow=True), dict(bn=64, tg=3, ksplit=4)),
}


# ---------------------------------------------------------------------------------------------------------------
# parity precision: fp32 operands as three bf16 planes
NP = 3
PX_MAX_TOL, PX_RMS_TOL, PX_BIAS_TOL = 5e-6, 2e-6, 1e-6
DZ_ULPS = 8


def px_call(name, *args):
    L = ryolo_lib()
    st = getattr(L.lib, name)(*args)
    assert st == 0, (name, L.last_error())


def vp(t, byte_off=0):
    return None if t is None else ctypes.c_void_p(t.data_ptr() + byte_off)


def stream():
    return ryolo_lib().stream_ptr()


def split3(v):
    """the kernels' split of fp32 v into three bf16 planes (plane k = bf16 of what planes < k left over)"""
    p0 = v.to(torch.bfloat16)
    r = v - p0.float()
    p1 = r.to(torch.bfloat16)
    r = r - p1.float()
    return p0, p1, r.to(torch.bfloat16)


def merge3(p0, p1, p2):
    """the kernels' rebuild: fp32 sum starting from 0, smallest plane first"""
    return ((torch.zeros_like(p0, dtype=torch.float32) + p2.float()) + p1.float()) + p0.float()


def planes_of(buf, plane, c, ch_off=0):
    """the NP planes of channels [ch_off, ch_off + c) of a split buffer, interior pixels, NCHW"""
    return [buf[:, 1:-1, 1:-1, k * plane + ch_off:k * plane + ch_off + c].permute(0, 3, 1, 2) for k in range(NP)]


def from_buf(buf, plane, c, ch_off=0):
    return merge3(*planes_of(buf, plane, c, ch_off))


def f32_buf(b, h, w, cs, dev="cuda"):
    return torch.zeros((b, h + 2, w + 2, cs), dtype=torch.float32, device=dev)


def measure(got, want):
    err = got.double() - want
    rms = float(want.pow(2).mean().sqrt())
    return dict(max=float(err.abs().max()) / float(want.abs().max()), rms=float(err.pow(2).mean().sqrt()) / rms,
                bias=float((err * want.sign()).mean()) / rms)


def ulps_f32(x):
    """fp32 spacing at |x| (the distance to the next float away from zero)"""
    a = x.float().abs()
    return (torch.nextafter(a, torch.full_like(a, math.inf)) - a).double()


class BnCase:
    def __init__(self, c, batch, h, w, act=True, up=False, batch_stats=1, gres=None, seed=0, zero_u=True):
        dev = torch.device("cuda")
        g = torch.Generator().manual_seed(seed)
        self.c, self.b, self.h, self.w, self.act, self.up, self.bs, self.gres_mode = c, batch, h, w, act, up, batch_stats, gres
        self.po = rup(c, 64)
        mu = torch.randn(c, generator=g) * 2.0
        sd = torch.rand(c, generator=g) * 2.0 + 0.25
        z = (torch.randn(batch, c, h, w, generator=g) * sd[None, :, None, None] + mu[None, :, None, None]).to(dev)
        nz = min(4, c) if zero_u else 0
        for ch in range(nz):                 # four pixels of the first channels share one value z0 ...
            z[0, ch, 1, :3] = z[0, ch, 0, 0]
        self.mean = z.double().mean((0, 2, 3)).float()
        self.invstd = (1.0 / (z.double().var((0, 2, 3), unbiased=False) + 1e-5).sqrt()).float()
        gamma = (torch.rand(c, generator=g) * 0.8 + 0.6).to(dev)
        beta = (torch.randn(c, generator=g) * 0.2).to(dev)
        self.scale = gamma * self.invstd
        self.shift = beta - self.mean * self.scale
        for ch in range(nz):                 # ... where u = (z0 * scale) + shift is exactly 0: shift = -(z0 * scale)
            self.shift[ch] = -(z[0, ch, 0, 0] * self.scale[ch])
        self.z = z
        self.slope = torch.tensor([0.17], device=dev)
        dh, dw_ = (2 * h, 2 * w) if up else (h, w)
        self.dy = torch.randn(batch, c, dh, dw_, generator=g).to(dev)
        self.old = torch.randn(batch, c, h, w, generator=g).to(dev) if gres == "acc" else None

    def u(self):
        return (self.z * self.scale[None, :, None, None]) + self.shift[None, :, None, None]

    def d(self):
        """dy as the kernel loads it: the 2x2 upsample's four gradients added in fp32, in the kernel's order"""
        if not self.up:
            return self.dy
        s = torch.zeros_like(self.z)
        for ry in range(2):
            for rx in range(2):
                s = s + self.dy[:, :, ry::2, rx::2]
        return s

    def mask(self):
        return self.u() > 0 if self.act else torch.ones_like(self.z, dtype=torch.bool)

    def run(self):
        dev = self.z.device
        b, c, h, w, po = self.b, self.c, self.h, self.w, self.po
        zb = f32_buf(b, h, w, po)
        zb[:, 1:-1, 1:-1, :c] = self.z.permute(0, 2, 3, 1)
        dh, dw_ = self.dy.shape[2:]
        dyb = f32_buf(b, dh, dw_, po)
        dyb[:, 1:-1, 1:-1, :c] = self.dy.permute(0, 2, 3, 1)
        sums = torch.full((2 * c + 1,), float("nan"), dtype=torch.float64, device=dev)
        g = torch.Generator().manual_seed(5)
        self.dz_init = torch.randn(b, h + 2, w + 2, NP * po, generator=g).to(torch.bfloat16).to(dev)   # sentinels
        dzb = self.dz_init.clone()
        gres = None
        if self.gres_mode is not None:
            gres = f32_buf(b, h, w, po)
            gres[:, 1:-1, 1:-1, c:] = 5.0
            if self.old is not None:
                gres[:, 1:-1, 1:-1, :c] = self.old.permute(0, 2, 3, 1)
            self.gres_init = gres.clone()
        px_call("ryolo_px_bn_act_bwd", vp(dyb), po, int(self.up), vp(zb), po, b, h, w, c, vp(self.scale), vp(self.shift),
                vp(self.mean), vp(self.invstd), vp(self.slope) if self.act else None, self.bs, vp(sums), vp(dzb),
                NP * po, po, vp(gres), po if gres is not None else 0, int(self.old is not None), NP, stream())
        torch.cuda.synchronize()
        return sums, dzb, gres

    def ref(self, mask=None):
        """float64 BN backward through PReLU on the kernel's inputs; mask: which u count as > 0"""
        mask = self.mask() if mask is None else mask
        d = self.d().double()
        slope = float(self.slope) if self.act else 1.0
        u = self.u().double()
        du = torch.where(mask, d, d * slope)
        zh = (self.z.double() - self.mean.double()[None, :, None, None]) * self.invstd.double()[None, :, None, None]
        dbeta, dgamma = du.sum((0, 2, 3)), (du * zh).sum((0, 2, 3))
        neg = ~mask
        dslope = (d * u)[neg].sum() if self.act else torch.zeros((), dtype=torch.float64, device=d.device)
        mags = (du.abs().sum((0, 2, 3)), (du * zh).abs().sum((0, 2, 3)), (d * u)[neg].abs().sum() if self.act else None)
        n = du.shape[0] * du.shape[2] * du.shape[3]
        sc = self.scale.double()[None, :, None, None]
        if self.bs:
            m1, m2 = (dbeta / n)[None, :, None, None], (dgamma / n)[None, :, None, None]
            dz = sc * (du - m1 - zh * m2)
            # the kernel's channel means are sums of fp32 du and du * zhat: each is off by a few ulps of the mean of the
            # |terms|, which is far above |mean| when the terms cancel
            a1, a2 = (mags[0] / n)[None, :, None, None], (mags[1] / n)[None, :, None, None]
            dz_mag = sc.abs() * (du.abs() + m1.abs() + a1 + zh.abs() * (m2.abs() + a2))
        else:
            dz, dz_mag = sc * du, (sc * du).abs()
        return dict(dbeta=dbeta, dgamma=dgamma, dslope=dslope, mags=mags, dz=dz, dz_mag=dz_mag)


def bn_errors(case, sums, dzb, r):
    """worst error of each output over its bound (<= 1 passes)"""
    c = case.c
    out = dict(dbeta=float(((sums[:c] - r["dbeta"]).abs() / (1e-6 * r["mags"][0] + 1e-300)).max()),
               dgamma=float(((sums[c:2 * c] - r["dgamma"]).abs() / (1e-6 * r["mags"][1] + 1e-300)).max()))
    if case.act:
        out["dslope"] = float((sums[2 * c] - r["dslope"]).abs() / (1e-6 * r["mags"][2] + 1e-300))
    got = from_buf(dzb, case.po, c).double()
    out["dz"] = float(((got - r["dz"]).abs() / (DZ_ULPS * U * r["dz_mag"] + 1e-38)).max())
    return out
