"""TEST INFRASTRUCTURE: one checked bf16 training step and the per-launch checks of the eval forward, against float64 of
the inputs each kernel actually received.  The only module of the suite that wraps plan methods: the float64 tests
(test_train_step_f64_gpu.py, test_train_scale_f64_gpu.py, test_dilated_train_f64_gpu.py, test_multiclass_f64_gpu.py,
test_se_f64_gpu.py, test_detect_forward_f64_gpu.py) bring their model, shape and extra checks and read the results this
module records.

Training step (run_step): after model(x) every buffer a forward kernel wrote is still there, so forward_checks checks
each launch post hoc on the plan's own input buffers; plan._backward_block is wrapped (instance attribute) so that what
each block overwrites is snapshotted, the production code runs unchanged and its outputs are checked right after
(check_block_bwd).  The bounds are stated in test_train_step_f64_gpu.py.  Every check runs over image chunks of at most
`budget` float64 bytes, so that the same checks hold at a batch whose activations fill the card
(test_train_scale_f64_gpu.py): the snapshot copies only what a block overwrites to host memory, and every full
reduction is summed in float64 over the chunks.  schedule_rows mirrors what each launch's schedule derives from the
shape, from a plan built or only laid out (plan_layout).

Squeeze-excitation: forward_checks checks ryolo_se_fwd's m, p, s and u post hoc; plan._se_bwd is wrapped as well
(check_se_bwd), because the SE backward runs inside its producing block's _backward_block, right before that block's
bn_act_bwd reads gx: the wrapper checks the SE on its own inputs, and check_block_bwd reads dy after the block, which is
the gx the SE left.  The SE bounds are stated in test_se_f64_gpu.py.

Eval forward (map_plan, check_first, check_conv, check_s2d_step, check_se_step, check_buffers): the steps of the eval
plan mapped to the graph's layers and every conv launch checked on its own input buffers; the bounds are stated in
test_detect_forward_f64_gpu.py."""
import time
import traceback
import types

import torch
import torch.nn.functional as F

from builders import ryolo_lib
from f64_refs import (BF16, BIAS_TOL, F64, HALF_BF16, STAT_TOL, TINY, U, bf16_check, bitwise, bn_act_fwd_ref, bn_chain,
                      bn_pieces, conv_schedule, conv_taps, d2s, f32_check, gemm_sms, halo_zero, head_bias_blocks,
                      head_bias_chain, interior, ratio, rup, s2d, s2d_dgrad_ref, se_block_s_ref, se_bwd_refs, se_fwd_ratios,
                      sum_check, tapsum, vint, wgrad_ratio, wgrad_ref, worst_ratio)
from helpers import wgrad_plan


def _layout():
    from rotate_yolov3_b200 import layout
    return layout


# ---------------------------------------------------------------------------------------------------------------
# the training step: per-kernel checks
class Step:
    """one checked training step: the model, its input x and shape (batch, h, w), and what the checks record"""

    def __init__(self, model, x):
        self.model, self.x = model, x
        self.batch, _, self.h, self.w = x.shape
        self.stash, self.keep_fwd, self.keep_bwd, self.keep_se = {}, set(), set(), set()


def _bn_of(model, blk):
    return model.module_list[blk.i].BatchNorm2d


def slope_of(model, blk):
    return model.module_list[blk.i].activation.weight.detach().float()


def _weight(model, blk):
    return model.module_list[blk.i].Conv2d.weight.detach()


def conv_updates(blk):
    return blk.k_eff * blk.k_eff * blk.cin_pad // 16


def f64_bytes(c_in, c_out, hw_in, hw_out):
    """float64 working set per image of a tap-sum reference and its check: the padded operand, its |.|, one shifted
    copy; value, magnitude and about eight temporaries of the result"""
    return 8 * (3 * c_in * hw_in + 10 * c_out * hw_out)


def ref_bytes(blk):
    """float64 bytes per image of the block's conv, wgrad and dgrad references and their checks"""
    gh, gw = (blk.src.h // 2, blk.src.w // 2) if blk.s2d else (blk.src.h, blk.src.w)
    cin = 27 if blk.i == 0 else blk.cin_eff
    hw = blk.src.h * blk.src.w
    out = dict(fwd=f64_bytes(cin, blk.cout, (gh + 2) * (gw + 2), blk.oh * blk.ow),
               wgrad=f64_bytes(cin, blk.cout, (gh + 2) * (gw + 2), gh * gw))
    if blk.s2d:        # dz zero-inserted on the input grid, then the mirrored 3x3 taps
        out["dgrad"] = f64_bytes(blk.cout, blk.src.c, hw, hw) + 8 * hw * blk.cout
    elif blk.i > 0:
        out["dgrad"] = f64_bytes(blk.cout, blk.cin, hw, hw)
    return out


def _img_bytes(t):
    return t[0].numel() * t.element_size()


def _host(t, chunk_list):
    """t (an image-major device view) copied to host memory chunk by chunk"""
    return torch.cat([t[b0:b1].cpu() for b0, b1 in chunk_list])


def _channels_host(buf, ch, b0, b1):
    """channels ch of images [b0, b1) of buf, copied to host memory (no device copy when ch is every channel)"""
    v = buf[b0:b1]
    return (v if len(ch) == v.shape[-1] else v.index_select(3, ch)).cpu()


def _max_offset(v, buf):
    """largest element offset into the buffer buf that its view v addresses"""
    return v.storage_offset() - buf.storage_offset() + sum((s - 1) * d for s, d in zip(v.shape, v.stride()))


def _overlap(a, b):
    return a is not None and b is not None and a.buf is b.buf and a.ch_off < b.ch_off + b.c and b.ch_off < a.ch_off + a.c


def stats_ref(z, c, chunk_list):
    """the float64 reductions stats_ratios needs, over image chunks of z [B, h, w, c] (two passes)"""
    s1 = torch.zeros(c, dtype=F64, device=z.device)
    a1, s2, q = s1.clone(), s1.clone(), s1.clone()
    for b0, b1 in chunk_list:
        z64 = z[b0:b1].double().reshape(-1, c)
        s1 += z64.sum(0)
        a1 += z64.abs().sum(0)
        s2 += z64.pow(2).sum(0)
        del z64
    n = z.numel() // c
    m64 = s1 / n
    for b0, b1 in chunk_list:
        q += (z[b0:b1].double().reshape(-1, c) - m64).pow(2).sum(0)
    return dict(n=n, m64=m64, v64=q / n, s1=s1, a1=a1, s2=s2)


def stats_ratios(ref, device, c, sums, mean, invstd, scale, shift, rm0, rv0, rm, rv, gamma, beta, eps, mom, l,
                 unbiased=True):
    """batch statistics: the kernel's sums against float64 (reduction bound), mean / invstd against the two-pass float64
    statistics of ref (target 2^-12), the finalisation and the running statistics against both the float64 statistics and
    the fp32 arithmetic of bn_finalize_channel applied to the kernel's own sums"""
    n, m64, v64 = ref["n"], ref["m64"], ref["v64"]
    std = (v64 + eps).sqrt()
    s1, s2 = sums[:c].double(), sums[c:2 * c].double()
    r = {}
    r["sums"] = max(sum_check(s1, ref["s1"], l, ref["a1"]), sum_check(s2, ref["s2"], l, ref["s2"]))
    r["mean"] = float(((mean.double() - m64).abs() / (STAT_TOL * std)).max())
    r["invstd"] = float(((invstd.double() - 1.0 / std).abs() / (STAT_TOL / std)).max())
    # bn_finalize_channel on the kernel's sums: mean = s1 / n (IEEE), var = s2 / n - mean^2 (contracted or not)
    cnt = torch.tensor(float(n), dtype=torch.float32, device=device)
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
    r, near = bn_bwd_check_chunked(lambda: [(z, d, dz_got)], z.shape[-1], sums_got, mean, invstd, sc, sh, slope, chain,
                                   drop_m2)
    return r, near


def bn_bwd_check_chunked(parts, c, sums_got, mean, invstd, sc, sh, slope, chain, drop_m2=False):
    """bn_bwd_check over image chunks: parts() yields (z, d, dz_got) of each chunk; two passes, the channel sums first"""
    def terms(z, d):
        z64 = z.double().reshape(-1, c)
        d64 = d.double().reshape(-1, c)
        zs = z64 * sc.double()
        u64 = zs + sh.double()
        u32 = u64.float().double()
        pos = u32 > 0
        near = u64.abs() <= 4 * U * (zs.abs() + sh.double().abs())
        du = torch.where(pos, d64, d64 * float(slope))
        zh = (z64 - mean.double()) * invstd.double()
        return d64, u32, pos, near, du, zh
    dbeta = dgamma = a1 = a2 = dslope = a_s = 0.0
    n = near_n = 0
    finite = True
    for z, d, dz_got in parts():
        d64, u32, pos, near, du, zh = terms(z, d)
        duzh = du * zh
        dbeta, dgamma = dbeta + du.sum(0), dgamma + duzh.sum(0)
        a1, a2 = a1 + du.abs().sum(0), a2 + duzh.abs().sum(0)
        neg = ~pos
        dslope = dslope + (d64 * u32)[neg].sum()
        a_s = a_s + (d64 * u32)[neg].abs().sum()
        n += du.shape[0]
        near_n += int(near.sum())
        finite = finite and bool(torch.isfinite(dz_got).all())
        del d64, u32, pos, near, du, zh, duzh
    m1 = dbeta / n
    m2 = torch.zeros_like(dgamma) if drop_m2 else dgamma / n
    acc = Acc()
    for z, d, dz_got in parts():
        _, _, _, near, du, zh = terms(z, d)
        want = sc.double() * (du - m1 - zh * m2)
        t = sc.double().abs() * (8 * U * (du.abs() + m1.abs() + (zh * m2).abs())
                                 + chain["sums"] * U * (a1 + zh.abs() * a2) / n)
        keep = ~near
        acc.add(dz_got.reshape(-1, c)[keep], want[keep], 0.0, t[keep])
        del near, du, zh, want, t, keep
    r = acc.result()
    r["finite"] = finite
    r["dbeta"] = sum_check(sums_got[:c], dbeta, chain["sums"] + 1, a1)
    r["dgamma"] = sum_check(sums_got[c:2 * c], dgamma, chain["sums"] + 3, a2)
    r["dslope"] = float((sums_got[2 * c].double() - dslope).abs() / (chain["slope"] * U * a_s + TINY))
    return r, near_n


def dy_of(plan, blk, shift=0, imgs=slice(None)):
    """(dy as bn_act_bwd reads it, fp32 [B, oh, ow, c]; mode): the gy view, the 2x2 sum of the up-sampled gradient in the
    kernel's order, or the consumer's dxs in place (mode 2).  shift: read the gradient buffer that many channels off;
    imgs: the images to read."""
    cons = getattr(blk, "dy_s2d", None)
    if cons is not None:
        return d2s(interior(cons.dxs, 0, cons.xs_cs)[imgs], blk.cout).float(), 2
    g = interior(blk.gy.buf, blk.gy.ch_off + shift, blk.cout)[imgs].float()
    if not blk.fuse_up:
        return g, 0
    s = torch.zeros_like(g[:, ::2, ::2])
    for ry in range(2):
        for rx in range(2):
            s = s + g[:, ry::2, rx::2]
    return s, 1


def forward_checks(st):
    """every forward launch post hoc on the plan's buffers, over image chunks of at most st.budget float64 bytes"""
    plan, model = st.plan, st.model
    L = _layout()
    B = st.batch
    out = {}
    # im2col of the image: bit for bit, columns 27..63 and the halo zero; the largest element offset checked
    col = plan.col
    bits = pad = True
    for b0, b1 in chunks(B, 8 * 27 * st.h * st.w, st.budget):
        want = F.unfold(st.x[b0:b1], 3, padding=1).view(b1 - b0, 27, st.h, st.w).permute(0, 2, 3, 1).to(BF16)
        bits = bits and bitwise(interior(col, 0, 27)[b0:b1], want)
        pad = pad and bool((interior(col, 27, 37)[b0:b1] == 0).all())
        del want
    st.checked_offsets = {"col": (col.numel(), _max_offset(interior(col, 27, 37), col))}
    st.im2col = dict(bits=bits, pad_zero=pad, halo=halo_zero(col))
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
        w64 = _weight(model, blk).to(BF16).double()
        if blk.i == 0:
            x, taps, s = interior(plan.col, 0, 27), [(0, 0, w64.reshape(blk.cout, 27).t())], 1
        else:
            x, taps, s = vint(blk.src), conv_taps(w64), blk.stride
        n = conv_updates(blk)
        cl = chunks(B, ref_bytes(blk)["fwd"], st.budget)
        if blk.is_head:
            bias = model.module_list[blk.i].Conv2d.bias.detach().double()
            got = blk.out.detach().permute(0, 2, 3, 1)
            worst = []
            for b0, b1 in cl:
                want, mag = tapsum(x[b0:b1], taps, blk.oh, blk.ow, s)
                worst.append(f32_check(got[b0:b1], want + bias, n * 2.0 ** -23 * mag)["max"])
                del want, mag
            r["z"] = float(torch.tensor(worst, dtype=F64).max())
            out[blk.i] = r
            continue
        z = interior(blk.z, 0, blk.cout)
        acc, kept = Acc(), []
        for b0, b1 in cl:
            want, mag = tapsum(x[b0:b1], taps, blk.oh, blk.ow, s)
            acc.add(z[b0:b1], want, n * 2.0 ** -23 * mag)
            if blk.i in st.keep_fwd:
                kept.append((want, mag))
            del want, mag
        rz = acc.result()
        r["z"], r["z_bias"] = rz["max"], rz["bias"]
        if blk.i in st.keep_fwd:
            st.stash[("z", blk.i)] = dict(want=torch.cat([k[0] for k in kept]), mag=torch.cat([k[1] for k in kept]),
                                          n=n, got=z.clone())
        del kept
        cz = chunks(B, 8 * 6 * _img_bytes(z), st.budget)
        if blk.has_bn:
            bn = _bn_of(model, blk)
            args = (stats_ref(z, blk.cout, cz), z.device, blk.cout, blk.sums, blk.mean, blk.invstd, blk.scale,
                    blk.shift, st.rm0[blk.i], st.rv0[blk.i], bn.running_mean, bn.running_var, bn.weight.detach(),
                    bn.bias.detach(), bn.eps, bn.momentum, bn_chain(B, blk.oh, blk.ow, blk.cout)["sums"])
            rs, mos = stats_ratios(*args)
            r.update(rs)
            r["mean_over_std"] = mos
            ratios.append(mos)
            # the same check with the running variance taken as biased (n instead of n - 1): kept for the bound self-test
            rb, _ = stats_ratios(*args, unbiased=False)
            st.rv_biased[blk.i] = max(rb["running"], rb["finalize"])
        else:
            # a bias (+ PReLU) conv without BatchNorm: fixed statistics, scale 1 and shift = the conv bias, bit for bit
            bias = model.module_list[blk.i].Conv2d.bias.detach()
            r["fixed_stats"] = bool((blk.scale == 1).all()) and torch.equal(blk.shift, bias)
        # bn_act_fwd; an up-sampling block writes each pixel four times
        res = vint(blk.res) if blk.res is not None else None
        y = interior(blk.y.buf, blk.y.ch_off, blk.cout)
        yv = y[:, ::2, ::2] if blk.fuse_up else y
        acc, copies = Acc(), True
        for b0, b1 in cz:
            want_y, t = bn_act_fwd_ref(z[b0:b1], blk.scale, blk.shift, slope_of(model, blk),
                                       res[b0:b1] if res is not None else None)
            if blk.fuse_up:
                copies = copies and all(bitwise(y[b0:b1, ry::2, rx::2], yv[b0:b1]) for ry in range(2) for rx in range(2))
            acc.add(yv[b0:b1], want_y, 0.0, t)
            del want_y, t
        ry_ = acc.result()
        r["y"], r["y_bias"] = ry_["max"], ry_["bias"]
        if blk.fuse_up:
            r["up_copies"] = copies
        if blk.i in st.keep_fwd and res is not None:
            st.stash[("y", blk.i)] = dict(z=z.clone(), res=res.clone(), got=yv.clone(), sc=blk.scale.clone(),
                                          sh=blk.shift.clone(), slope=slope_of(model, blk))
        out[blk.i] = r
    # space-to-depth copies (bn_act_fwd_s2d or ryolo_space_to_depth) bit for bit; every halo zero
    for blk in plan.blocks:
        if blk.s2d:
            src = vint(blk.src)
            xs = interior(blk.xs, 0, 4 * blk.src.c)
            out[blk.i]["xs"] = all(bitwise(xs[b0:b1], s2d(src[b0:b1])) for b0, b1 in chunks(B, 4 * _img_bytes(xs), st.budget))
    # squeeze-excitation (ryolo_se_fwd after the producing block's bn_act_fwd): m, p, s and u on the block's output x,
    # recorded under the SE's layer index
    for se in ses_of(plan):
        fc = model.module_list[se.i].fc
        out[se.i], _ = se_fwd_ratios(se, vint(se.x), vint(se.u), fc[0].weight.detach().double(),
                                     fc[2].weight.detach().double())
        out[se.i]["halo_u"] = halo_zero(se.u.buf)
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


def ses_of(plan):
    """the SE blocks of a training plan, each attached to the block that produces its input x"""
    return [b.se for b in plan.blocks if getattr(b, "se", None) is not None]


def snapshot(st, blk):
    """before the block's backward, what it overwrites and its checks read, copied to host memory over image chunks: z
    (which becomes dz in place), the prior of an accumulated gradient view, the channels of the shared gradient buffer
    outside the views the block (and its SE) write; for the blocks in st.keep_bwd, dy read 32 channels off.  dy itself
    is read after the block, from buffers the block does not write."""
    B = st.batch
    snap = {}

    def host(t):
        return _host(t, chunks(B, _img_bytes(t), st.budget))
    if not blk.is_head:
        snap["z"] = host(interior(blk.z, 0, blk.cout))
        assert not _overlap(blk.gy, blk.gsrc) and not _overlap(blk.gy, blk.gres) and blk.gy.buf is not blk.z
        if blk.gres is not None and blk.gres_acc:
            snap["gres_prior"] = host(vint(blk.gres))
        if blk.i in st.keep_bwd and blk.fuse_up:
            snap["dy_shift"], _ = dy_of(st.plan, blk, shift=32)
    if blk.gsrc is not None:
        gbuf = blk.gsrc.buf
        if blk.gsrc_acc:
            snap["prior"] = host(vint(blk.gsrc))
        # a space-to-depth block whose producer reads its dgrad output in place writes no gradient view of its own
        se = getattr(blk, "se", None)
        views = [blk.gres, se.gx if se is not None else None, None if blk.s2d and blk.dxs_direct else blk.gsrc]
        allowed = torch.zeros(gbuf.shape[-1], dtype=torch.bool)
        for v in views:
            if v is not None and v.buf is gbuf:
                allowed[v.ch_off:v.ch_off + v.c] = True
        snap["outside"] = (~allowed).nonzero().flatten().to(gbuf.device)
        if len(snap["outside"]):
            snap["gbuf_outside"] = torch.cat([_channels_host(gbuf, snap["outside"], b0, b1)
                                              for b0, b1 in chunks(B, _img_bytes(gbuf), st.budget)])
    return snap


def outside_untouched(st, blk, snap):
    """the channels of the block's gradient buffer outside the views it writes are as snapshot() left them, and the halo
    is zero"""
    gbuf = blk.gsrc.buf
    same = not len(snap["outside"]) or all(
        torch.equal(_channels_host(gbuf, snap["outside"], b0, b1), snap["gbuf_outside"][b0:b1])
        for b0, b1 in chunks(st.batch, _img_bytes(gbuf), st.budget))
    return same and halo_zero(gbuf)


def check_block_bwd(st, blk, orig):
    """snapshot -> the production _backward_block -> checks; returns the results (never raises into autograd)"""
    r, snap = {}, {}
    try:
        snap = snapshot(st, blk)
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
    gradient) on the dy it read; returns dz"""
    plan, model = st.plan, st.model
    B = st.batch
    dev = st.x.device
    if blk.is_head:
        dz = interior(blk.dz, 0, blk.cout)
        g = st.g_nhwc[blk.i]
        r["dz_bits"] = all(bitwise(dz[b0:b1], g[b0:b1].to(BF16)) for b0, b1 in chunks(B, 4 * _img_bytes(dz), st.budget))
        r["dz_pad_zero"] = bool((blk.dz[..., blk.cout:] == 0).all()) and halo_zero(blk.dz)
        return dz
    dz = interior(blk.z, 0, blk.cout)
    _, r["dy_mode"] = dy_of(plan, blk, imgs=slice(0, 1))
    chain = bn_chain(B, blk.oh, blk.ow, blk.cout, 2 if r["dy_mode"] == 2 and blk.cout // 8 * 2 <= 640 else 1)
    cl = chunks(B, 8 * 12 * blk.oh * blk.ow * blk.cout, st.budget)

    def parts():
        for b0, b1 in cl:
            yield snap["z"][b0:b1].to(dev), dy_of(plan, blk, imgs=slice(b0, b1))[0], dz[b0:b1]
    rb, near = bn_bwd_check_chunked(parts, blk.cout, blk.bsums, blk.mean, blk.invstd, blk.scale, blk.shift,
                                    slope_of(model, blk), chain)
    r["dz"], r["dz_bias"] = rb["max"], rb["bias"]
    for k in ("dbeta", "dgamma", "dslope", "finite"):
        r[k] = rb[k]
    r["near_zero_u"] = near
    r["n_elems"] = dz.numel()
    if blk.i in st.keep_bwd:
        st.stash[("bn", blk.i)] = dict(z=snap["z"].to(dev), dy=dy_of(plan, blk)[0], dy_shift=snap.get("dy_shift"),
                                       dz=dz.clone(), sums=blk.bsums.clone(), mean=blk.mean.clone(),
                                       invstd=blk.invstd.clone(), sc=blk.scale.clone(), sh=blk.shift.clone(),
                                       slope=slope_of(model, blk), chain=chain)
    if blk.gres is not None:
        gres = vint(blk.gres)
        ok = True
        for b0, b1 in cl:
            d = dy_of(plan, blk, imgs=slice(b0, b1))[0]
            want = (snap["gres_prior"][b0:b1].to(dev).float() + d).to(BF16) if blk.gres_acc else d.to(BF16)
            ok = ok and bitwise(gres[b0:b1], want)
        r["gres_bits"] = ok
    r["dz_halo"] = halo_zero(blk.z)
    return dz


def _bwd_checks(st, blk, snap, r):
    plan, model = st.plan, st.model
    B = st.batch
    dev = st.x.device
    w64 = _weight(model, blk).to(BF16).double()
    dz = dz_checks(st, blk, snap, r)
    # weight gradient (split-K layout): the float64 reference summed over image chunks
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
    wr = wm = 0.0
    for b0, b1 in chunks(B, ref_bytes(blk)["wgrad"], st.budget):
        a, m = wgrad_ref(x[b0:b1], dz[b0:b1], offs)
        wr, wm = wr + a, wm + m
        del a, m
    plan_w = wgrad_plan(blk.k_eff, blk.cin_pad, blk.cout_pad, B, gh, gw_, gemm_sms())
    got = blk.dw[:, :blk.cout, :cin]
    # test_wgrad's random-walk bound (KAPPA sqrt(n_add) 2^-24 A) is reported, not required: on the step's operands the
    # accumulator's truncations do not cancel
    r["wgrad"] = wgrad_ratio(got, wr, wm, plan_w)
    r["wgrad_rw"] = worst_ratio(got, wr, wm, plan_w["n_add"])
    if blk.i in st.keep_bwd:
        st.stash[("wgrad", blk.i)] = dict(x=x.clone(), dz=dz.clone(), offs=offs, got=got.clone(), plan=plan_w)
    del wr, wm
    if blk.i == 0:
        return
    # input gradient
    gbuf = blk.gsrc.buf
    if blk.s2d:
        dxs = interior(blk.dxs, 0, blk.cin_eff)
        n = 4 * rup(blk.cout, 64) // 16
        acc, bits = Acc(), True
        for b0, b1 in chunks(B, ref_bytes(blk)["dgrad"], st.budget):
            want, mag = s2d_dgrad_ref(dz[b0:b1], w64, blk.src.h, blk.src.w)
            acc.add(dxs[b0:b1], want, n * 2.0 ** -23 * mag)
            del want, mag
            if not blk.dxs_direct:
                v = d2s(dxs[b0:b1], blk.src.c)
                want_bits = (snap["prior"][b0:b1].to(dev).float() + v.float()).to(BF16) if blk.gsrc_acc else v
                bits = bits and bitwise(vint(blk.gsrc)[b0:b1], want_bits)
        rd = acc.result()
        r["dgrad"], r["dgrad_bias"] = rd["max"], rd["bias"]
        if not blk.dxs_direct:
            r["d2s_bits"] = bits
    else:
        got = vint(blk.gsrc)
        n = blk.k * blk.k * rup(blk.cout, 64) // 16
        acc = Acc()
        for b0, b1 in chunks(B, ref_bytes(blk)["dgrad"], st.budget):
            want, mag = tapsum(dz[b0:b1], conv_taps(w64, mirror=True), blk.src.h, blk.src.w)
            e, t = n * 2.0 ** -23 * mag, 0.0
            if blk.gsrc_acc:
                prior = snap["prior"][b0:b1].to(dev).double()
                want = want + prior
                t = U * (mag + prior.abs())
                del prior
            acc.add(got[b0:b1], want, e, t)
            del want, mag, e, t
        rd = acc.result()
        r["dgrad"], r["dgrad_bias"] = rd["max"], rd["bias"]
        if blk.i in st.keep_bwd:
            st.stash[("dgrad", blk.i)] = dict(dz=dz.clone(), w64=w64, got=got.clone(),
                                              prior=snap["prior"].to(dev) if blk.gsrc_acc else None,
                                              acc=blk.gsrc_acc, h=blk.src.h, w=blk.src.w, n=n,
                                              shifted=(interior(gbuf, blk.gsrc.ch_off - 32, blk.gsrc.c).clone()
                                                       if blk.gsrc.ch_off >= 32 else None))
    r["outside_untouched"] = outside_untouched(st, blk, snap)


# ---------------------------------------------------------------------------------------------------------------
# the training step: the run
class _LeanDot(torch.autograd.Function):
    """sum(p * G) whose gradient is G itself: no cotangent-sized temporaries"""

    @staticmethod
    def forward(ctx, p, g):
        ctx.g = g
        return sum((p[b] * g[b]).sum() for b in range(p.shape[0]))

    @staticmethod
    def backward(ctx, go):
        assert float(go) == 1.0
        return ctx.g, None


def dense_loss(st, ps, seed):
    """loss = sum (p * G) with a dense random cotangent G per head (it reaches every head channel), drawn in the shape of
    p and permuted on the host into the layout of the fp32 head buffer, so that the cotangent the plan receives is G
    itself (one copy of G on the device, no product or transpose of it); st.g_nhwc views G in the layout of the head's
    dz"""
    gen = torch.Generator().manual_seed(seed)
    st.g_nhwc = {}
    loss = 0.0
    for blk, p in zip(st.plan.heads, ps):
        b, na, ny, nx, no = p.shape
        g = torch.randn(p.shape, generator=gen).permute(0, 1, 4, 2, 3).reshape(b, na * no, ny, nx).to(p.device)
        st.g_nhwc[blk.i] = g.permute(0, 2, 3, 1)                              # channel a * no + k
        loss = loss + _LeanDot.apply(p, g.view(b, na, no, ny, nx).permute(0, 1, 3, 4, 2))
    return loss


def check_se_bwd(st, se, prod, orig, stream):
    """gu, x and the prior gx snapshotted -> the production ryolo_se_bwd -> ds, dm, gW1, gW2 and gx checked (recorded
    under the SE's layer index).  The producing block's bn_act_bwd reads gx next, as the SE left it: check_block_bwd reads
    it after the block."""
    model = st.model
    r, snap = {"acc": int(se.gx_acc)}, None
    try:
        snap = dict(gu=vint(se.gu).clone(), x=vint(se.x).clone(), gx_old=vint(se.gx).clone() if se.gx_acc else None)
    except Exception:
        r["error"] = traceback.format_exc()
    orig(se, stream)
    st.bwd[se.i] = r
    if snap is None:
        return
    try:
        assert prod.gy is se.gx and getattr(prod, "dy_s2d", None) is None and not prod.fuse_up
        fc = model.module_list[se.i].fc
        refs = se_bwd_refs(se, snap["gu"], snap["x"], snap["gx_old"], fc[0].weight.detach().double(),
                           fc[2].weight.detach().double(), se.gw1, se.gw2)
        B = st.batch
        r["ds"] = ratio(se.ds.view(B, se.c), *refs["ds"])
        r["dm"] = ratio(se.dm.view(B, se.c), *refs["dm"])
        r["gw1"] = ratio(se.gw1.view(se.cr, se.c), *refs["gw1"])
        r["gw2"] = ratio(se.gw2.view(se.c, se.cr), *refs["gw2"])
        r.update({"gx_" + k: v for k, v in bf16_check(vint(se.gx), *refs["gx"]).items()})
        r["halo_gu"], r["halo_gx"] = halo_zero(se.gu.buf), halo_zero(se.gx.buf)
        if se.i in st.keep_se:
            st.stash[("se", se.i)] = dict(snap, refs=refs, gx=vint(se.gx).clone())
    except Exception:
        r["error"] = traceback.format_exc()


def backward(st, loss, block_check=check_block_bwd, head_grads=None):
    """loss.backward() with plan._backward_block wrapped: block_check(st, blk, orig) snapshots what the block overwrites,
    runs orig(blk) and returns the block's results for st.bwd (None: nothing recorded).  head_grads(st, grads) sees the
    head cotangents before the production _head_grads.  A plan with SE blocks also has plan._se_bwd wrapped
    (check_se_bwd): it runs inside the producing block's _backward_block, in production order."""
    plan = st.plan
    st.bwd = {}
    orig = plan._backward_block

    def wrapped(blk):
        r = block_check(st, blk, orig)
        if r is not None:
            st.bwd[blk.i] = r
    patched = {"_backward_block": wrapped}
    prod_of = {id(b.se): b for b in plan.blocks if getattr(b, "se", None) is not None}
    if prod_of:
        orig_se = plan._se_bwd

        def se_bwd(se, stream):
            check_se_bwd(st, se, prod_of[id(se)], orig_se, stream)
        patched["_se_bwd"] = se_bwd
    if head_grads is not None:
        orig_hg = plan._head_grads

        def hg(grads):
            head_grads(st, grads)
            orig_hg(grads)
        patched["_head_grads"] = hg
    for name, fn in patched.items():
        setattr(plan, name, fn)
    try:
        loss.backward()
    finally:
        for name in patched:
            delattr(plan, name)
    torch.cuda.synchronize()


def gather_checks(st, gw_bits=True):
    """the head bias sums (their own reduction chain) and, with gw_bits, each block's .grad gather of its split-K dW"""
    plan = st.plan
    L = _layout()
    for blk in plan.blocks:
        r = st.bwd.setdefault(blk.i, {})
        if blk.is_head and blk.owner is None:
            g = st.g_nhwc[blk.i]
            s = a = 0.0
            for b0, b1 in chunks(st.batch, 8 * 3 * g[0].numel(), st.budget):
                g64 = g[b0:b1].double()
                s, a = s + g64.sum((0, 1, 2)), a + g64.abs().sum((0, 1, 2))
            gb = plan.garena[blk.gb_off:blk.gb_off + blk.cout]
            r["dbias"] = sum_check(gb, s, head_bias_chain(st.batch, blk.oh, blk.ow), a)
        if not gw_bits:
            continue
        if blk.i == 0:
            want = blk.dw[0, :blk.cout, :27].reshape(blk.cout, 3, 3, 3)
        elif blk.s2d:
            c = blk.src.c
            d2 = blk.dw[:, :blk.cout, :4 * c].permute(1, 2, 0).reshape(blk.cout, 4 * c, 2, 2)
            want = L.s2d_weight_grad(d2, c)
        else:
            want = blk.dw[:, :blk.cout, :blk.cin].reshape(blk.k, blk.k, blk.cout, blk.cin).permute(2, 3, 0, 1)
        r["gw_bits"] = torch.equal(blk.gw, want)
    if gw_bits:
        for se in ses_of(plan):
            fc = st.model.module_list[se.i].fc
            st.bwd.setdefault(se.i, {})["gw_bits"] = (torch.equal(fc[0].weight.grad, se.gw1.view(se.cr, se.c))
                                                      and torch.equal(fc[2].weight.grad, se.gw2.view(se.c, se.cr)))


def run_step(st, cot_seed=None, *, budget=None, prepare=None, linear_fwd=None, loss=None, head_grads=None,
             block_check=check_block_bwd, gw_bits=True):
    """one checked training step of st.model on st.x.

    budget: the float64 bytes of one chunk of images in every check (default CHUNK_BYTES).  prepare(st) runs once the
    checked forward has built st.plan, before any check.  linear_fwd(st, blk) runs right after each plan._linear_fwd
    launch; the plan must exist to be wrapped, so with linear_fwd the checked step follows one warm-up step that builds
    it.  loss(st, ps) gives the loss (default: dense_loss with cot_seed); head_grads and block_check as in backward();
    gw_bits as in gather_checks()."""
    model = st.model
    st.budget = CHUNK_BYTES if budget is None else budget
    t0 = time.time()
    plan = None
    if linear_fwd is not None:
        model(st.x)
        plan = model._tplan
    st.rm0, st.rv0, nbt0 = {}, {}, {}
    for i, m in enumerate(model.module_list):
        if hasattr(m, "BatchNorm2d"):
            st.rm0[i] = m.BatchNorm2d.running_mean.clone()
            st.rv0[i] = m.BatchNorm2d.running_var.clone()
            nbt0[i] = int(m.BatchNorm2d.num_batches_tracked)
    if linear_fwd is not None:
        orig_f = plan._linear_fwd

        def lin_fwd(blk, s):
            orig_f(blk, s)
            linear_fwd(st, blk)
        plan._linear_fwd = lin_fwd
    try:
        ps = model(st.x)
    finally:
        if linear_fwd is not None:
            del plan._linear_fwd
    torch.cuda.synchronize()
    assert plan is None or model._tplan is plan
    st.plan = plan = model._tplan
    if prepare is not None:
        prepare(st)
    # every BatchNorm module belongs to a block; its running statistics move once when the block's BatchNorm runs, never
    # for a weight_from block
    by = {b.i: b for b in plan.blocks}
    st.nbt_ok = all(i in by and int(model.module_list[i].BatchNorm2d.num_batches_tracked)
                    == nbt0[i] + (by[i].owner is None and by[i].has_bn) for i in nbt0)
    forward_checks(st)
    torch.cuda.synchronize()
    st.t_fwd = time.time() - t0
    backward(st, loss(st, ps) if loss is not None else dense_loss(st, ps, cot_seed), block_check, head_grads)
    gather_checks(st, gw_bits)
    st.t_total = time.time() - t0
    return st


# ---------------------------------------------------------------------------------------------------------------
# the training step's launch schedules, from the plan's geometry
def plan_layout(model, batch, h, w, device="cpu", shared=None):
    """a TrainPlan laid out without storage (every activation a stride-0 stand-in of its shape) and the activation-pool
    bytes it needs: the geometry of every launch, on any machine"""
    from rotate_yolov3_b200.pool import ActivationPool
    from rotate_yolov3_b200.train_path import TrainPlan
    pool = ActivationPool(device)
    plan, need, _ = pool._layout(lambda: TrainPlan(model, batch, h, w, torch.device(device), pool,
                                                   {} if shared is None else shared))
    return plan, need


def schedule_rows(plan, sms):
    """per block of the training step, what its launches derive from the shape: the forward and dgrad conv (tiles, CTAs,
    tiles per CTA against the staging ring), the split-K wgrad plan, the BN pieces of bn_stats / bn_act_bwd, the head-bias
    blocks, and the largest element offset into any buffer the block's kernels address"""
    B = plan.batch
    rows = []
    for blk in plan.blocks:
        gh, gw = (blk.src.h // 2, blk.src.w // 2) if blk.s2d else (blk.src.h, blk.src.w)
        np_ = B * (gh + 2) * (gw + 2)
        r = dict(i=blk.i, kind="head" if blk.is_head else ("s2d" if blk.s2d else "k%d" % blk.k), grid=(blk.oh, blk.ow),
                 fwd=conv_schedule(np_, blk.cout, False, sms))
        if blk.i > 0:
            r["dgrad"] = conv_schedule(np_, blk.cin_eff, bool(blk.gsrc_acc) and not blk.s2d, sms)
        r["wgrad"] = wgrad_plan(blk.k_eff, blk.cin_pad, blk.cout_pad, B, gh, gw, sms)
        if blk.is_head:
            r["head_bias"] = head_bias_blocks(B, blk.oh)
            bufs = [blk.src.buf, blk.dz, blk.out]
        else:
            rpp = 2 if getattr(blk, "dy_s2d", None) is not None and blk.cout // 8 * 2 <= 640 else 1
            r["bn_fwd"] = bn_pieces(B, blk.oh, blk.ow, blk.cout, 1, sms)
            r["bn_bwd"] = bn_pieces(B, blk.oh, blk.ow, blk.cout, rpp, sms)
            bufs = [blk.src.buf, blk.z, blk.y.buf, blk.gy.buf]
        bufs += [plan.col if blk.i == 0 else blk.gsrc.buf]
        if blk.s2d:
            bufs += [blk.xs, blk.dxs]
        if getattr(blk, "dz_up", None) is not None:
            bufs.append(blk.dz_up)
        r["max_offset"] = max(b.numel() for b in bufs if b is not None) - 1
        rows.append(r)
    return rows


# ---------------------------------------------------------------------------------------------------------------
# the eval forward: float64 references and the plan's steps mapped to the graph
CHUNK_BYTES = 4e9          # float64 working set of one chunk of images


class Acc:
    """bf16_check over image chunks: the worst ratio (NaN propagates) and the rounding-bias ratio of the whole tensor"""

    def __init__(self):
        self.maxes, self.es, self.w2, self.n = [], 0.0, 0.0, 0

    def add(self, got, want, e, t=0.0):
        self.maxes.append(bf16_check(got, want, e, t)["max"])
        self.moments(got.double() - want, want)

    def moments(self, err, want):
        """the whole-tensor sums of the bias ratio: signed error along want, want^2, element count"""
        self.es += float((err * want.sign()).sum())
        self.w2 += float(want.pow(2).sum())
        self.n += want.numel()

    def result(self):
        rms = (self.w2 / self.n) ** 0.5
        return {"max": float(torch.tensor(self.maxes, dtype=F64).max()),
                "bias": abs(self.es / self.n) / (BIAS_TOL * rms + TINY)}


def chunks(batch, bytes_per_image, budget=None):
    """[b0, b1) image ranges covering the batch, each within `budget` bytes (default CHUNK_BYTES) at bytes_per_image, or
    one image when one image alone needs more"""
    per = max(1, min(batch, int((budget or CHUNK_BYTES) // bytes_per_image)))
    return [(b, min(batch, b + per)) for b in range(0, batch, per)]


def conv_want(s, bias, slope, res=None):
    """act(S + bias) + res in float64 and T, the fp32 epilogue roundings (bias add, PReLU multiply, residual add)"""
    u = s + bias
    act = torch.where(u > 0, u, u * slope) if slope is not None else u
    t = 2 * U * (s.abs() + bias.abs())
    if res is None:
        return act, t
    r = res.double()
    return act + r, t + U * (act.abs() + r.abs())


def first_check(got_xs, x_nchw, wf, bias, slope, acc=None):
    """the first layer on the fp32 image with bf16(wf), + bias, PReLU, in the space-to-depth layout of got_xs"""
    x = x_nchw.permute(0, 2, 3, 1)
    s, a = tapsum(x, conv_taps(wf.to(BF16).double()), x.shape[1], x.shape[2])
    want, t = conv_want(s, bias.double(), slope)
    e = 4 * 2.0 ** -23 * a + 2.0 ** -16 * a
    acc = acc or Acc()
    acc.add(got_xs, s2d(want), s2d(e), s2d(t))
    return acc


def fold_ratio(model, i, drop_eps=False):
    """_folded's fp32 (scale, bias) against float64 utils/torch_utils.py:45-69, in units of their rounding bounds"""
    _, scale, bias, _ = model._folded(i, torch.device("cuda"))
    seq = model.module_list[i]
    bn = seq.BatchNorm2d
    g, be, m, v = (t.detach().double() for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var))
    s64 = g / torch.sqrt(v + (0.0 if drop_eps else bn.eps))
    b64 = be - m * s64
    if seq.Conv2d.bias is not None:
        b64 = b64 + seq.Conv2d.bias.detach().double() * s64
    rs = (scale.double() - s64).abs() / (3 * U * s64.abs() + TINY)
    rb = (bias.double() - b64).abs() / (U * (4 * (m * s64).abs() + b64.abs()) + TINY)
    return max(float(rs.max()), float(rb.max()))


def packed_want(model, i, s2d_layer, taps, cout_pad, cin_pad):
    wt, scale, _, _ = model._folded(i, torch.device("cuda"))
    if s2d_layer:
        wt = _layout().s2d_weight(wt)
    wf = wt * scale.view(-1, 1, 1, 1) if scale is not None else wt
    want = torch.zeros((taps, cout_pad, cin_pad), dtype=BF16, device=wt.device)
    for t, (_, _, m) in enumerate(conv_taps(wf)):
        want[t, :wf.shape[0], :wf.shape[1]] = m.t().to(BF16)
    return want


class View:
    def __init__(self, buf, off, c):
        self.buf, self.off, self.c = buf, off, c

    @property
    def ptr(self):
        return self.buf.data_ptr() + 2 * self.off

    def interior(self):
        return interior(self.buf, self.off, self.c)


class Run:
    """one checked eval forward: the model, its plan and input, and what the checks record"""

    def __init__(self, name, model):
        self.name, self.model = name, model


def slope(model, i):
    seq = model.module_list[i]
    return float(seq.activation.weight.detach().float().item()) if hasattr(seq, "activation") else None


def map_plan(st):
    """walk module_defs beside the plan's steps: each layer's output as a View, the steps of each conv layer, the s2d
    copies; asserts the plan's pointers are the graph's wiring"""
    model, plan = st.model, st.plan
    defs = model.module_defs
    steps = plan["steps"]
    outs, conv_of, s2d_of, se_of, scaled = {}, {}, {}, {}, {}
    k = 0
    for i, d in enumerate(defs):
        t = d["type"]
        if t == "convolutional":
            if k < len(steps) and steps[k][0] == "s2d":
                s2d_of[i] = k
                k += 1
            kind, a = steps[k]
            conv_of[i] = k
            k += 1
            if kind == "first":
                assert a["xs"] is not None and a["out"].buf is None      # layer 0 lives in layer 1's s2d buffer only
                outs[0] = None
                continue
            assert kind == "conv", (i, kind)
            out = a["keep"][2]
            desc = a["desc"]
            nxt = defs[i + 1]["type"] if i + 1 < len(defs) else None
            if desc.out_dtype == ryolo_lib().DT_F32:
                outs[i] = out
                continue
            v = View(out.buf, out.ch_off, out.c)
            assert v.ptr == a["y"]
            if (nxt == "shortcut" and desc.has_residual) or (nxt == "upsample" and desc.upsample2x):
                outs[i], outs[i + 1] = None, v
            else:
                assert not desc.has_residual and not desc.upsample2x
                outs[i] = v
        elif t == "route":
            ls = [int(x) for x in d["layers"].split(",")]
            ls = [l if l > 0 else i + l for l in ls]
            if len(ls) == 1:
                outs[i] = outs[ls[0]]
            else:
                buf, off = outs[ls[0]].buf, 0
                for l in ls:                                       # producers at their route offsets, one buffer
                    assert outs[l].buf is buf and outs[l].off == off, (i, l)
                    off += outs[l].c
                outs[i] = View(buf, 0, off)
        elif t in ("shortcut", "upsample"):
            assert i in outs, (t, i)                                # materialised by the fused conv
        elif t == "yolo":
            outs[i] = None
        elif t == "se":
            kind, a = steps[k]
            se_of[i] = k
            k += 1
            src = outs[i - 1]
            assert a["x"] == src.ptr and a["xcs"] == src.buf.shape[-1] and a["c"] == src.c, i
            assert (a["h"], a["w"]) == tuple(src.interior().shape[1:3])
            if kind == "se_fwd":
                # out of place: u = x * s in a buffer of its own, x stays readable (from=-4 shortcuts, routes)
                u = a["keep"][1]
                outs[i] = View(u.buf, u.ch_off, u.c)
                assert outs[i].ptr == a["u"] and a["ucs"] == u.buf.shape[-1] and u.c == src.c
            else:
                # in place: layer i - 1's output is scaled after its conv wrote it; nothing reads the unscaled tensor
                assert kind == "se", (i, kind)
                outs[i] = src
                scaled[i - 1] = a["scale"]
        else:
            raise AssertionError("layer type %s in the detect graph" % t)
    assert k == len(steps)
    st.outs, st.conv_of, st.s2d_of, st.se_of, st.scaled = outs, conv_of, s2d_of, se_of, scaled


def check_s2d_step(st, i):
    a = st.plan["steps"][st.s2d_of[i]][1]
    src = st.outs[i - 1]
    assert a["x"] == src.ptr and a["xcs"] == src.buf.shape[-1] and a["c"] == src.c
    xs = a["xs"]
    c4 = 4 * src.c
    return dict(bits=bitwise(interior(xs, 0, c4), s2d(src.interior())),
                pad_zero=bool((xs[..., c4:] == 0).all()))


def check_first(st):
    model = st.model
    kind, a = st.plan["steps"][st.conv_of[0]]
    wt, scale, bias, _ = model._folded(0, torch.device("cuda"))
    r = {}
    r["w_bits"] = torch.equal(a["w"], wt * scale.view(-1, 1, 1, 1)) and torch.equal(a["b"], bias)
    r["slope"] = a["slope"] == slope(model, 0)
    r["fold"] = fold_ratio(model, 0)
    xs = a["xs"]
    cout = a["cout"]
    assert xs.shape[-1] == rup(4 * cout, 64)
    b, _, h, w = st.x.shape
    acc = Acc()
    for b0, b1 in chunks(b, h * w * cout * 8 * 10):
        first_check(interior(xs, 0, 4 * cout)[b0:b1], st.x[b0:b1], a["w"], bias, slope(model, 0), acc)
    r.update(acc.result())
    r["xs_pad_zero"] = bool((xs[..., 4 * cout:] == 0).all())
    if st.stash is not None:
        st.stash["first"] = dict(x=st.x[:2].clone(), got=interior(xs, 0, 4 * cout)[:2].clone(), w=a["w"], b=bias,
                                 slope=slope(model, 0))
    return r


def scaled_want(want, e, t, s):
    """a bf16 conv output that an in-place SE then multiplied by its fp32 scale s [B, c]: the conv's own rounding (half a
    bf16 ulp of |want| + e + t, plus e + t) carried through the multiply, whose fp32 rounding adds U |want s|; the SE's
    bf16 rounding is the half ulp bf16_check allows"""
    s = s.double().view(s.shape[0], 1, 1, -1)
    w = want * s
    return w, (HALF_BF16 * (want.abs() + e + t) + e + t) * s, U * w.abs()


def check_se_step(st, i):
    """an eval SE step on its own buffers.  se_fwd: m, p, s and u against float64 of x (the SE bounds of the training
    step), u's halo zero.  se (in place, x overwritten): s against float64 of the kernel's own channel sums"""
    kind, a = st.plan["steps"][st.se_of[i]]
    fc = st.model.module_list[i].fc
    w1, w2 = a["w1"].double(), a["w2"].double()
    r = dict(kind=kind, w_bits=torch.equal(a["w1"], fc[0].weight.detach().float())
             and torch.equal(a["w2"], fc[2].weight.detach().float()))
    if kind == "se":
        b = a["sums"].numel() // a["c"]
        r["s"] = ratio(a["scale"].view(b, a["c"]), *se_block_s_ref(a["sums"].view(b, a["c"]), w1, w2, a["h"] * a["w"]))
        return r
    se = types.SimpleNamespace(h=a["h"], w=a["w"], c=a["c"], cr=a["cr"], m=a["m"], p=a["p"], s=a["s"])
    x, u = st.outs[i - 1].interior(), st.outs[i].interior()
    rr, refs = se_fwd_ratios(se, x, u, w1, w2)
    r.update(rr)
    r["halo_u"] = halo_zero(st.outs[i].buf)
    if st.stash is not None and i in st.keep:
        st.stash[("se", i)] = dict(x=x.clone(), s=a["s"].clone(), u=u.clone(), refs=refs)
    return r


def conv_offsets(k, taps):
    if k == 3:
        return [(t // 3 - 1, t % 3 - 1) for t in range(taps)]
    if k == 2:
        return [(t // 2 - 1, t % 2 - 1) for t in range(taps)]
    return [(0, 0)]


def check_conv(st, i):
    model, plan = st.model, st.plan
    a = plan["steps"][st.conv_of[i]][1]
    desc = a["desc"]
    L = ryolo_lib()
    r = {}
    # inputs: the graph's wiring
    s2d_layer = i == 1 or i in st.s2d_of
    if s2d_layer:
        # layer 1 reads the buffer the first layer wrote; the other stride-2 layers the copy of ryolo_space_to_depth
        xs = plan["steps"][st.s2d_of[i] if i in st.s2d_of else st.conv_of[0]][1]["xs"]
        assert desc.ksize == 2 and a["x"] == xs.data_ptr() and desc.cin_stride == xs.shape[-1]
        x = interior(xs, 0, desc.cin)
    else:
        src = st.outs[i - 1]
        assert a["x"] == src.ptr and desc.cin == src.c and desc.cin_stride == src.buf.shape[-1]
        x = src.interior()
    assert desc.stride == 1                                  # every stride-2 layer runs on a space-to-depth copy
    assert (desc.in_h, desc.in_w) == tuple(x.shape[1:3])
    k = abs(desc.ksize)
    taps, cin_pad = k * k, rup(desc.cin, 64)
    cout = desc.cout
    cout_pad = a["w"].numel() // (2 * taps * cin_pad)
    pk = a["w"].view(BF16).view(taps, cout_pad, cin_pad)
    # weight pack, bias buffer, slope, folding
    r["w_bits"] = bitwise(pk, packed_want(model, i, s2d_layer, taps, cout_pad, cin_pad))
    _, scale, bias, _ = model._folded(i, torch.device("cuda"))
    bias_pad = torch.zeros(cout_pad, dtype=torch.float32, device=bias.device)
    bias_pad[:cout] = bias
    r["b_bits"] = torch.equal(a["b"], bias_pad)
    if scale is not None:
        r["fold"] = fold_ratio(model, i)
    slope_ = slope(model, i)
    r["slope"] = bool(desc.has_act) == (slope_ is not None) and (slope_ is None or desc.slope == slope_)
    # residual: the layer the [shortcut] names
    res = None
    if desc.has_residual:
        frm = int(model.module_defs[i + 1]["from"])
        rv = st.outs[i + 1 + frm if frm < 0 else frm]
        assert a["r"] == rv.ptr and desc.res_stride == rv.buf.shape[-1] and rv.c == cout
        res = rv.interior()
    else:
        assert a["r"] is None
    head = desc.out_dtype == L.DT_F32
    up = bool(desc.upsample2x)
    oi = i if not up and not desc.has_residual else i + 1
    out = st.outs[oi]
    sc = getattr(st, "scaled", {}).get(oi)         # an in-place SE scaled this output after the conv wrote it
    if sc is not None:
        assert not head and not up
        sc = sc.view(desc.batch, cout)
    n = taps * cin_pad // 16
    mats = [(dy, dx, pk[t, :cout, :desc.cin].double().t().contiguous())
            for t, (dy, dx) in enumerate(conv_offsets(k, taps))]
    b64 = bias.double()
    oh, ow = desc.in_h, desc.in_w
    acc = Acc()
    heads = []
    copies = True
    per_img = 8 * (4 * (oh + 2) * (ow + 2) * desc.cin + 12 * oh * ow * cout)
    keep = st.stash is not None and i in st.keep
    kept = []
    for b0, b1 in chunks(desc.batch, per_img):
        s, mag = tapsum(x[b0:b1], mats, oh, ow)
        e = n * 2.0 ** -23 * mag
        if head:
            got = out[b0:b1].permute(0, 2, 3, 1)
            heads.append(f32_check(got, s + b64, e)["max"])
        else:
            want, t = conv_want(s, b64, slope_, res[b0:b1] if res is not None else None)
            if sc is not None:
                want, e, t = scaled_want(want, e, t, sc[b0:b1])
            y = out.interior()[b0:b1]
            if up:
                base = y[:, ::2, ::2]
                copies = copies and all(bitwise(y[:, ry::2, rx::2], base) for ry in range(2) for rx in range(2))
                y = base
            acc.add(y, want, e, t)
        if keep:
            kept.append((s, mag))
        del s, mag, e
    if head:
        r["max"] = float(torch.tensor(heads, dtype=F64).max())
    else:
        r.update(acc.result())
    if up:
        r["up_copies"] = copies
    if keep:
        st.stash[i] = dict(s=torch.cat([p[0] for p in kept]), mag=torch.cat([p[1] for p in kept]), n=n, bias=b64,
                           slope=slope_, res=res.clone() if res is not None else None, out=out, up=up, head=head)
    r.update(kind="head" if head else ("s2d" if s2d_layer else "k%d" % k), cout=cout, grid="%dx%d" % (oh, ow))
    return r


def check_buffers(st):
    """every halo zero; in every activation buffer the channels no producer owns are zero"""
    owned = {}
    for i, v in st.outs.items():
        if isinstance(v, View):
            owned.setdefault(id(v.buf), (v.buf, []))[1].append((v.off, v.off + v.c))
    bufs = [b for b, _ in owned.values()]
    bufs += [a["xs"] for kind, a in st.plan["steps"] if kind in ("s2d", "first")]
    ok = all(halo_zero(b) for b in bufs)
    for buf, ranges in owned.values():
        mask = torch.ones(buf.shape[-1], dtype=torch.bool, device=buf.device)
        for lo, hi in ranges:
            mask[lo:hi] = False
        ok = ok and bool((buf[..., mask] == 0).all())
    concat = sorted({buf.shape[-1] for buf, rs in owned.values() if len({r for r in rs}) > 1})
    return ok, concat
