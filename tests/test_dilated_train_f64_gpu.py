"""Every kernel launch of one bf16 training step of the multi-branch dilated graph (cfg/yolov3-m.cfg, m_model()) against
float64 of the inputs it actually received, at three shapes: batch 2 at 416 x 416 (the cfg's size: grids 13 / 26 / 52,
ragged phases at every dilation, block 108 13^2 -> 7^2), batch 3 at 352 x 608 (a letterboxed 16:9 frame: h != w, so an
index map with rows and columns swapped cannot pass; an odd batch, so GEMM tiles straddle images; block 108 11 x 19 ->
6 x 10) and batch 2 at 128 x 160 (small phase images; block 108 4 x 5 -> 2 x 3).  A dense random cotangent G per head
(loss = sum (p * G)) reaches all 16 heads.

The blocks this graph shares with yolov3 (convs, BatchNorm statistics, bn_act_fwd / bn_act_bwd, wgrad, dgrad, heads,
head bias sums) are checked by checked_step.py with the bounds of test_train_step_f64_gpu.py (see its docstring:
E = n 2^-23 A per conv, half a bf16 ulp + E for bf16 outputs, E + 2^-24 |want| for fp32 ones, L 2^-24 sum |terms| for
reductions).  What this graph adds, checked here:

  weight_from forward   a linear conv on the owner's bf16 weight.  1x1: y = bf16(S + res) within the conv bound plus
                        2^-24 (A + |res|) for the fp32 residual add; heads: fp32 output with no bias.  Dilated (dh, dw):
                        ryolo_dilate_split equals phase_split bit for bit (zero fill, halo, padding channels); the conv
                        on the phase images, merged back, is within the conv bound (n = 9 cin_pad / 16) of the float64
                        dilated conv of the unsplit input; the merge (+ shortcut) is one rounding of phase_merge(zp) + res.
                        The forward of these blocks is checked right after its launches (plan._linear_fwd wrapped on the
                        instance), since the phase buffers are shared by every dilated block of a shape.
  weight_from backward  bn_act_bwd with has_bn = has_act = 0: dz = dy bit for bit.  The wgrad ADDS into the owner's dW:
                        its increment (after - before, exact in float64) is within E of wgrad_plan + 2^-24 |want| +
                        2^-24 |dW after| (the add into the arena).  Dilated: the split of dz bit for bit, the wgrad on the
                        phase images (wgrad_plan of batch dh dw, ceil(h / dh), ceil(w / dw)) against the float64 dilated
                        weight gradient of the unsplit dz and x, sum_p dz(p) x(p + d o (k - 1)); the phase dgrad, merged,
                        against the float64 dilated transposed conv; the merge into the source gradient bit for bit,
                        bf16(prior + merge) when it accumulates; the channels and halo outside the gradient view untouched.
  owners                dW sees 1 + (number of weight_from users) increments; Conv2d.weight.grad equals dW bit for bit;
                        the final dW is within the sum of the per-use bounds of the float64 sum over all uses; the users'
                        own Conv2d / BatchNorm2d get no gradient.
  block 108             3x3 / stride 2 on an odd grid (zero-insert path): z against the float64 stride-2 conv,
                        ryolo_zero_insert2x bit for bit (dz at the even pixels, zeros elsewhere), the wgrad on dz_up
                        against torch's float64 stride-2 weight gradient, the dgrad against float64 conv_transpose2d with
                        the output padding that restores the odd input size.
  block 109             bias + PReLU without BatchNorm: scale 1 and shift = bias bit for bit, y = act(z + bias); backward
                        dz = dy act'(z + bias) (the kink at z + bias: the fp32 u = fma(z, 1, bias) has the sign of the
                        exact sum, so no element is ambiguous), d bias = sum dz and d slope under the bn_chain bound.

No dilated dgrad of this cfg accumulates (each dilated conv's source gradient has that merge as its only writer), so the
bound self-test also runs ryolo_dilate_merge with accumulate = 1 on the step's own phase gradient and source gradient
buffer.

Measured on an H100 80GB HBM3 (132 SMs, power limit 700 W, 1980 MHz max SM clock), seeds as below.  `pytest -s` prints
one line per block (each kernel's worst |err| / bound); the worst per launch kind over the three shapes (block):
  dilated (36)      conv z 0.984 (240), split / merge bitwise; wgrad increment 0.223 (114 at 128 x 160); dgrad 0.962 (224)
  weight_from 1x1   y 0.994 (239); wgrad increment 0.172 (115); dgrad 0.996 (179)
  weight_from heads fp32 z 0.102 (209); wgrad increment 0.114 (121); dgrad 0.991 (132)
  owners            conv z 0.994, bn_act_fwd / bn_act_bwd 0.996, wgrad increment 0.569 (80 at 128 x 160); final dW
                    against the float64 sum of all uses <= 0.26 (78); 3 / 5 / 7 increments for 75-81 / 87-93 / 99-105
  block 108         z 0.909, dz 0.995, zero-insert bitwise, wgrad 0.213, dgrad 0.941
  block 109         z 0.989, y 0.996, dz 0.932, d bias 0.095, d slope 0.001, wgrad 0.331, dgrad 0.984
Bias ratios (mean signed error) stay <= 0.16.  Bugs put in fail by a factor >= 2 (bitwise checks) and otherwise >= 996:
the last ragged phase column dropped from a (1, 8) wgrad 1.7e3, (dh, dw) swapped in the dgrad 9.6e3, one of seven uses
missing from owner 100 1.0e3, block 109's kink at z 996, a bias on a weight_from head 6.2e3.  Whole file: 18 s."""
import ctypes
import traceback

import pytest
import torch

from builders import m_model, phase_merge, phase_split, ryolo_lib
from checked_step import (Step, check_block_bwd, conv_updates, dy_of, dz_checks, outside_untouched, run_step, slope_of,
                          snapshot)
from f64_refs import (BF16, F64, TINY, U, bad_entries, bf16_check, bitwise, bn_chain, check_z, conv_taps, dil_conv,
                      dil_wgrad_ref, f32_check, gemm_sms, halo_zero, interior, nchw, nhwc, passed, rup, s2_refs,
                      sum_check, tapsum, vint, wgrad_ratio, wgrad_ref)
from helpers import init_darknet_weights, wgrad_plan

pytestmark = pytest.mark.gpu

SHAPES = [(2, 416, 416), (3, 352, 608), (2, 128, 160)]
BUG_OWNER = 100          # owner whose per-use weight gradients the bound self-test keeps (seven uses, 256 x 128 x 9)


def psplit(x, dh, dw):
    """phase_split of an NHWC tensor: [B, H, W, C] -> [B dh dw, ceil(H / dh), ceil(W / dw), C]"""
    return nhwc(phase_split(nchw(x), dh, dw))


def pmerge(xp, b, h, w, dh, dw):
    return nhwc(phase_merge(nchw(xp), b, h, w, dh, dw))


# ---------------------------------------------------------------------------------------------------------------
# checks of the launches yolov3 does not have
def merge_check(got, prior, v, acc):
    """the merge of a phase gradient v into the source gradient: bf16(prior + v) when it accumulates, else v"""
    return bitwise(got, (prior.float() + v.float()).to(BF16) if acc else v.to(BF16))


def bias_act_bwd_check(z, d, dz_got, sums, bias, slope, chain, kink_at_z=False):
    """bn_act_bwd with has_bn = 0: du = d * act'(u), u = fma(z, 1, bias) (its fp32 rounding keeps the sign of the exact
    sum), dz = bf16(du); d bias = sum du, d slope = sum over u <= 0 of d u (fp32 u).  kink_at_z: the branch decided by z
    (a plausible bug)."""
    c = z.shape[-1]
    z64, d64 = z.double().reshape(-1, c), d.double().reshape(-1, c)
    u64 = z64 + bias.double()
    pos = (z64 if kink_at_z else u64) > 0
    du = torch.where(pos, d64, d64 * float(slope))
    r = bf16_check(dz_got.reshape(-1, c), du, 0.0, U * du.abs())
    r["dbias"] = sum_check(sums[:c], du.sum(0), chain["sums"] + 1, du.abs().sum(0))
    ds = d64 * u64.float().double()
    r["dslope"] = float((sums[2 * c].double() - ds[~pos].sum()).abs() / (chain["slope"] * U * ds[~pos].abs().sum() + TINY))
    return r


def inc_bound(want, mag, after, plan_w):
    """bound of one wgrad's increment of a shared dW: E of its split-K chain, half an fp32 ulp of the result and of the
    add into the arena"""
    n = plan_w["updates"] + plan_w["ksplit"]
    return n * 2.0 ** -23 * mag + U * want.abs() + U * after.double().abs()


def wgrad_record(st, blk, got, snap, want, mag, plan_w):
    """the wgrad of a block whose dW is shared (an owner or a weight_from user): the increment, recorded per owner;
    otherwise the plain split-K check"""
    if "dw" not in snap:
        return wgrad_ratio(got, want, mag, plan_w)
    owner = blk.owner if blk.owner is not None else blk.i
    before = snap["dw"][:, :blk.cout, :got.shape[2]]
    inc = got.double() - before.double()
    bound = inc_bound(want, mag, got, plan_w)
    o = st.owners.setdefault(owner, dict(n=0, want=0.0, bound=0.0, uses=[]))
    o["n"] += 1
    o["want"] = o["want"] + want
    o["bound"] = o["bound"] + bound
    o["uses"].append(blk.i)
    if owner == BUG_OWNER:
        st.stash.setdefault("uses", {})[blk.i] = (want.clone(), bound.clone())
    return float(((inc - want).abs() / (bound + TINY)).max())


def _w64(st, blk):
    i = blk.owner if blk.owner is not None else blk.i
    return st.model.module_list[i].Conv2d.weight.detach().to(BF16).double()


def check_linear_fwd(st, blk):
    """a weight_from block's forward (not a head), right after its launches"""
    w64 = _w64(st, blk)
    x = vint(blk.src)
    res = vint(blk.res) if blk.res is not None else None
    y = interior(blk.y.buf, blk.y.ch_off, blk.cout)
    n = conv_updates(blk)
    r = {}
    if blk.dil is None:
        want, mag = tapsum(x, conv_taps(w64), blk.oh, blk.ow)
        t = 0.0
        if res is not None:
            want = want + res.double()
            t = U * (mag + res.double().abs())
        rr = bf16_check(y, want, n * 2.0 ** -23 * mag, t)
        r["y"], r["y_bias"] = rr["max"], rr["bias"]
        return r
    dh, dw = blk.dil
    r["split_bits"] = bitwise(interior(blk.xp, 0, blk.cin), psplit(x, dh, dw))
    r["split_halo"] = halo_zero(blk.xp) and bool((blk.xp[..., blk.cin:] == 0).all())
    got = pmerge(interior(blk.zp, 0, blk.cout), st.batch, blk.oh, blk.ow, dh, dw)
    want, mag = dil_conv(x, w64, dh, dw)
    rz = check_z(got, want, mag, n)
    r["z"], r["z_bias"] = rz["max"], rz["bias"]
    r["merge_bits"] = bitwise(y, (got.float() + res.float()).to(BF16) if res is not None else got)
    return r


def fwd_heads(st):
    """the weight_from heads: fp32 output of the owner's weight, no bias"""
    for blk in st.plan.blocks:
        if not (blk.is_head and blk.owner is not None):
            continue
        want, mag = tapsum(vint(blk.src), conv_taps(_w64(st, blk)), blk.oh, blk.ow)
        got = blk.out.detach().permute(0, 2, 3, 1)
        e = conv_updates(blk) * 2.0 ** -23 * mag
        st.fwd_lin[blk.i] = {"z": f32_check(got, want, e)["max"]}
        if "head" not in st.stash:
            bias = st.model.module_list[blk.i].Conv2d.bias.detach().double()
            st.stash["head"] = dict(got=got.clone(), want=want, e=e, bias=bias)


def check_bwd(st, blk, orig):
    """snapshot -> the production _backward_block -> checks; blocks of the yolov3 kinds go to test_train_step_f64_gpu"""
    plain = blk.owner is None and blk.i not in st.owner_of_users and (blk.is_head or blk.has_bn) and \
        not (blk.stride == 2 and not blk.s2d)
    if plain:
        return check_block_bwd(st, blk, orig)
    r, snap = {}, {}
    try:
        snap = snapshot(st, blk)
        if blk.owner is not None or blk.i in st.owner_of_users:
            snap["dw"] = blk.dw.clone()
    except Exception:
        r["error"] = traceback.format_exc()
    orig(blk)
    if "error" in r:
        return r
    try:
        _own_bwd_checks(st, blk, snap, r)
    except Exception:
        r["error"] = traceback.format_exc()
    return r


def _own_bwd_checks(st, blk, snap, r):
    model = st.model
    dev = st.x.device
    w64 = _w64(st, blk)
    if blk.is_head or blk.has_bn:
        dz = dz_checks(st, blk, snap, r)
    else:
        dz = interior(blk.z, 0, blk.cout)
        dy, r["dy_mode"] = dy_of(st.plan, blk)          # read after the block, which does not write it
        if blk.owner is not None:        # linear: dz = dy, the shortcut gradient (+)= dy
            r["dz_bits"] = bitwise(dz, dy.to(BF16))
        else:                            # block 109: bias + PReLU
            chain = bn_chain(st.batch, blk.oh, blk.ow, blk.cout)
            slope = slope_of(model, blk)
            bias = model.module_list[blk.i].Conv2d.bias.detach()
            z = snap["z"].to(dev)
            rb = bias_act_bwd_check(z, dy, dz, blk.bsums, bias, slope, chain)
            r["dz"], r["dz_bias"], r["dbeta"], r["dslope"] = rb["max"], rb["bias"], rb["dbias"], rb["dslope"]
            st.stash["b109"] = dict(z=z, dy=dy, dz=dz.clone(), sums=blk.bsums.clone(), bias=bias, slope=slope,
                                    chain=chain)
        if blk.gres is not None:
            r["gres_bits"] = bitwise(vint(blk.gres), (snap["gres_prior"].to(dev).float() + dy).to(BF16) if blk.gres_acc
                                       else dy.to(BF16))
        r["dz_halo"] = halo_zero(blk.z)
    x = vint(blk.src)
    prior = snap["prior"].to(dev) if blk.gsrc_acc else None
    got_dw = blk.dw[:, :blk.cout, :blk.cin]
    sms = gemm_sms()
    if blk.dil is not None:
        dh, dw = blk.dil
        b, h, w = st.batch, blk.src.h, blk.src.w
        r["split_bits"] = bitwise(interior(blk.zp, 0, blk.cout), psplit(dz, dh, dw))
        wr, wm = dil_wgrad_ref(x, dz, dh, dw)
        plan_w = wgrad_plan(3, blk.cin_pad, blk.cout_pad, blk.nb, blk.hp, blk.wp, sms)
        r["wgrad"] = wgrad_record(st, blk, got_dw, snap, wr, wm, plan_w)
        v = pmerge(interior(blk.dxp, 0, blk.cin), b, h, w, dh, dw)
        want, mag = dil_conv(dz, w64, dh, dw, adjoint=True)
        n = 9 * rup(blk.cout, 64) // 16
        rd = check_z(v, want, mag, n)
        r["dgrad"], r["dgrad_bias"] = rd["max"], rd["bias"]
        r["merge_bits"] = merge_check(vint(blk.gsrc), prior, v, blk.gsrc_acc)
        if (h % dh or w % dw) and max(dh, dw) > st.stash.get("dil_d", 0):     # the widest ragged dilation
            st.stash["dil_d"] = max(dh, dw)
            st.stash["dil"] = dict(i=blk.i, x=x.clone(), dz=dz.clone(), dh=dh, dw=dw, got=got_dw.clone(),
                                   before=snap["dw"][:, :blk.cout, :blk.cin].clone(), plan=plan_w, v=v.clone(),
                                   dxp=blk.dxp.clone(), w64=w64, n=n, gbuf=blk.gsrc.buf.clone(), gsrc=blk.gsrc)
    elif blk.stride == 2:
        # zero-insert path: dz on the even pixels of the input grid, zeros elsewhere
        up = interior(blk.dz_up, 0, blk.cout)
        want_up = torch.zeros_like(up)
        want_up[:, ::2, ::2] = dz
        r["zero_insert_bits"] = bitwise(up, want_up) and halo_zero(blk.dz_up)
        st.stash["zi"] = dict(up=up.clone(), dz=dz.clone())
        gw, gwm, want, mag = s2_refs(x, dz, w64)
        plan_w = wgrad_plan(3, blk.cin_pad, blk.cout_pad, st.batch, blk.src.h, blk.src.w, sms)
        r["wgrad"] = wgrad_record(st, blk, got_dw, snap, gw, gwm, plan_w)
        n = 9 * rup(blk.cout, 64) // 16
        t = 0.0
        if blk.gsrc_acc:
            want = want + prior.double()
            t = U * (mag + prior.double().abs())
        rd = bf16_check(vint(blk.gsrc), want, n * 2.0 ** -23 * mag, t)
        r["dgrad"], r["dgrad_bias"] = rd["max"], rd["bias"]
    else:
        p = (blk.k - 1) // 2
        wr, wm = wgrad_ref(x, dz, [(kh - p, kw - p) for kh in range(blk.k) for kw in range(blk.k)])
        plan_w = wgrad_plan(blk.k, blk.cin_pad, blk.cout_pad, st.batch, blk.src.h, blk.src.w, sms)
        r["wgrad"] = wgrad_record(st, blk, got_dw, snap, wr, wm, plan_w)
        want, mag = tapsum(dz, conv_taps(w64, mirror=True), blk.src.h, blk.src.w)
        n = blk.k * blk.k * rup(blk.cout, 64) // 16
        t = 0.0
        if blk.gsrc_acc:
            want = want + prior.double()
            t = U * (mag + prior.double().abs())
        rd = bf16_check(vint(blk.gsrc), want, n * 2.0 ** -23 * mag, t)
        r["dgrad"], r["dgrad_bias"] = rd["max"], rd["bias"]
    r["outside_untouched"] = outside_untouched(st, blk, snap)


# ---------------------------------------------------------------------------------------------------------------
def _lin_fwd(st, blk):
    try:
        st.fwd_lin[blk.i] = check_linear_fwd(st, blk)
    except Exception:
        st.fwd_lin[blk.i] = {"error": traceback.format_exc()}


def _prepare(st):
    """the weight_from heads' forward checks, and the owners whose dW the weight_from blocks add into"""
    fwd_heads(st)
    st.owner_of_users = {b.owner for b in st.plan.blocks if b.owner is not None}


def m_step(batch, h, w, seed):
    """the checked step (after the warm-up step that builds the plan whose _linear_fwd is wrapped)"""
    dev = torch.device("cuda")
    model = init_darknet_weights(m_model(), seed=seed).to(dev).train()
    st = Step(model, torch.rand(batch, 3, h, w, generator=torch.Generator().manual_seed(seed + 1)).to(dev))
    st.owners, st.fwd_lin = {}, {}
    run_step(st, seed + 2, prepare=_prepare, linear_fwd=_lin_fwd, block_check=check_bwd, gw_bits=False)
    st.fwd.update(st.fwd_lin)
    after_backward(st)
    return st


def after_backward(st):
    """the gathers into .grad, the owners' totals"""
    plan, model = st.plan, st.model
    # every parameter's .grad is its arena slot bit for bit (dW reshaped for the conv weights); weight_from blocks' own
    # modules get none
    st.grad_bits, st.grad_none = [], []
    by = {b.i: b for b in plan.blocks}
    for name, p in model.named_parameters():
        parts = name.split(".")
        key = (int(parts[1]), ".".join(parts[2:]))
        slot = plan.param_slots.get(key)
        if slot is None:
            st.grad_none.append((name, p.grad is None))
            continue
        off, n, shape = slot
        ok = p.grad is not None and torch.equal(p.grad, plan.garena[off:off + n].view(shape))
        blk = by.get(key[0])
        if ok and key[1] == "Conv2d.weight" and blk is not None and blk.i > 0 and not blk.s2d:
            ok = torch.equal(p.grad, blk.dw[:, :blk.cout, :blk.cin].reshape(blk.k, blk.k, blk.cout, blk.cin)
                             .permute(2, 3, 0, 1))
        st.grad_bits.append((name, ok))
    st.owner_final = {}
    for i, o in st.owners.items():
        blk = by[i]
        final = blk.dw[:, :blk.cout, :blk.cin].double()
        users = sum(b.owner == i for b in plan.blocks)
        st.owner_final[i] = dict(n=o["n"], want_n=1 + users,
                                 ratio=float(((final - o["want"]).abs() / (o["bound"] + TINY)).max()))
        if i == BUG_OWNER:
            st.stash["owner"] = dict(final=final, want=o["want"], bound=o["bound"])


KEYS = ("z", "z_bias", "mean", "invstd", "y", "y_bias", "dz", "dz_bias", "dbeta", "dgamma", "dslope", "wgrad", "dgrad",
        "dgrad_bias", "dbias")


def _kind(blk):
    if blk.is_head:
        return "head" if blk.owner is None else "head<%d" % blk.owner
    if blk.dil is not None:
        return "d%dx%d<%d" % (blk.dil[0], blk.dil[1], blk.owner)
    if blk.owner is not None:
        return "k%d<%d" % (blk.k, blk.owner)
    if blk.stride == 2 and not blk.s2d:
        return "s2zi"
    return "s2d" if blk.s2d else "k%d" % blk.k


def _print_table(st, tag):
    print("\n[%s] whole step with checks %.1f s" % (tag, st.t_total))
    worst = {}
    for blk in st.plan.blocks:
        f, b = st.fwd.get(blk.i, {}), st.bwd.get(blk.i, {})
        cols = ["%-9s" % _kind(blk), "%4d" % blk.cout, "%2dx%-2d" % (blk.oh, blk.ow)]
        for src, tag_ in ((f, "f:"), (b, "b:")):
            for key in KEYS:
                if isinstance(src.get(key), float):
                    cols.append("%s %.3f" % (key, src[key]))
                    if not worst.get(tag_ + key, (-1.0,))[0] >= src[key]:
                        worst[tag_ + key] = (src[key], blk.i)
            if "error" in src:
                cols.append("ERROR")
        print("[%s] %3d " % (tag, blk.i) + "  ".join(cols))
    print("[%s] worst: %s" % (tag, ", ".join("%s %.3f (%d)" % (k, v, i) for k, (v, i) in sorted(worst.items()))))
    print("[%s] owners: %s" % (tag, ", ".join("%d: %d uses %.3f" % (i, o["n"], o["ratio"])
                                              for i, o in sorted(st.owner_final.items()))))


@pytest.fixture(scope="module", params=SHAPES, ids=["b2_416", "b3_352x608", "b2_128x160"])
def step(request):
    batch, h, w = request.param
    st = m_step(batch, h, w, 31)
    _print_table(st, "m%dx%dx%d" % (batch, h, w))
    return st


# ---------------------------------------------------------------------------------------------------------------
def test_covers_every_launch(step):
    plan = step.plan
    heads = [b for b in plan.blocks if b.is_head]
    assert len(heads) == 16 and sum(b.owner is None for b in heads) == 4
    assert sorted(b.i for b in heads if b.owner is None) == [81, 93, 105, 110]
    assert sum(b.dil is not None for b in plan.blocks) == 36
    zi = [b.i for b in plan.blocks if b.stride == 2 and not b.s2d]
    assert zi == [108], zi
    assert set(step.fwd) == {b.i for b in plan.blocks}
    by = {b.i: b for b in plan.blocks}
    ops = plan.sched.ops(plan)
    missing = []
    for kind, i, flag in ops:
        r = step.bwd.get(i, {})
        if kind == "head":
            ok = "dz_bits" in r
        elif kind == "bnact":
            ok = "dz" in r or "dz_bits" in r
        elif kind == "wgrad":
            ok = "wgrad" in r
        elif kind == "dgrad":
            # a dilated dgrad: the split of dz, the phase dgrad and the merge; the zero-insert path of block 108
            ok = "dgrad" in r and (by[i].dil is None or ("split_bits" in r and "merge_bits" in r)) and \
                (i != 108 or "zero_insert_bits" in r)
        else:
            ok = False                   # a launch kind this file does not know
        if not ok:
            missing.append((kind, i, flag))
    assert not missing, missing
    assert {k for k, _, _ in ops} == {"head", "bnact", "wgrad", "dgrad"}
    assert sum(k == "dgrad" and by[i].dil is not None for k, i, _ in ops) == 36
    assert sum(k == "head" for k, _, _ in ops) == 16


def test_forward_kernels_vs_float64(step):
    assert step.nbt_ok and step.fwd_halo
    assert step.im2col == dict(bits=True, pad_zero=True, halo=True), step.im2col
    bad = [p[:2] for p in step.packs if not p[2]]
    assert not bad, bad
    bad = bad_entries(step.fwd)
    assert not bad, bad
    assert step.fwd[109]["fixed_stats"]


def test_backward_kernels_vs_float64(step):
    bad = bad_entries(step.bwd)
    assert not bad, bad
    for i, r in step.bwd.items():
        if "near_zero_u" in r:
            assert r["near_zero_u"] <= max(64, r["n_elems"] // 100000), (i, r["near_zero_u"])


def test_shared_weights(step):
    plan = step.plan
    owners = sorted({b.owner for b in plan.blocks if b.owner is not None})
    assert len(owners) == 21
    want_uses = {**{i: 3 for i in range(75, 82)}, **{i: 5 for i in range(87, 94)}, **{i: 7 for i in range(99, 106)}}
    got = {i: o["n"] for i, o in step.owner_final.items()}
    assert got == want_uses, got
    assert all(o["n"] == o["want_n"] for o in step.owner_final.values())
    bad = {i: o["ratio"] for i, o in step.owner_final.items() if not o["ratio"] <= 1.0}
    assert not bad, bad
    assert all(ok for _, ok in step.grad_bits), [n for n, ok in step.grad_bits if not ok]
    assert all(is_none for _, is_none in step.grad_none), [n for n, is_none in step.grad_none if not is_none]
    for b in plan.blocks:
        if b.owner is not None:
            seq = step.model.module_list[b.i]
            for mod in ("Conv2d", "BatchNorm2d"):
                if hasattr(seq, mod):
                    assert all(p.grad is None for p in getattr(seq, mod).parameters()), (b.i, mod)


def test_bounds_reject_plausible_bugs(step):
    """each bug, put into a reference or a stored tensor, fails the check that guards it"""
    s = step.stash
    out = {}
    # the last ragged phase row / column of a dilated wgrad dropped
    d = s["dil"]
    dh, dw = d["dh"], d["dw"]
    inc = d["got"].double() - d["before"].double()
    want, mag = dil_wgrad_ref(d["x"], d["dz"], dh, dw)
    bound = inc_bound(want, mag, d["got"], d["plan"])
    assert float(((inc - want).abs() / bound).max()) <= 1.0
    h, w = d["x"].shape[1], d["x"].shape[2]
    mask = torch.ones_like(d["dz"], dtype=F64)
    if w % dw:
        mask[:, :, (w // dw) * dw:] = 0        # phase column wp - 1 exists only for the phases rx < w % dw
    else:
        mask[:, (h // dh) * dh:] = 0
    lost, _ = dil_wgrad_ref(d["x"], d["dz"].double() * mask, dh, dw)
    out["ragged phase edge dropped from wgrad"] = float(((inc - lost).abs() / bound).max())
    # (dh, dw) swapped in the dgrad's index map
    want, mag = dil_conv(d["dz"], d["w64"], dh, dw, adjoint=True)
    assert passed(check_z(d["v"], want, mag, d["n"]))
    want_sw, mag_sw = dil_conv(d["dz"], d["w64"], dw, dh, adjoint=True)
    out["dgrad with (dh, dw) swapped"] = check_z(d["v"], want_sw, mag_sw, d["n"])["max"]
    # the merge with accumulate = 1, run on the step's own phase gradient into a copy of the source gradient buffer
    # (which holds the step's final gradient there): correct against bf16(prior + merge), fails against an overwrite
    L = ryolo_lib()
    g = d["gsrc"]
    buf = d["gbuf"].clone()
    buf[:, 1:-1, 1:-1, g.ch_off:g.ch_off + g.c] = torch.randn(buf.shape[0], buf.shape[1] - 2, buf.shape[2] - 2, g.c,
                                                              device=buf.device, generator=torch.Generator(
                                                                  device=buf.device).manual_seed(9)).to(BF16)
    prior = interior(buf, g.ch_off, g.c).clone()
    L.check(L.lib.ryolo_dilate_merge(L.ptr(d["dxp"]), d["dxp"].shape[-1], d["x"].shape[0], h, w, g.c, dh, dw, None, 0,
                                     1, ctypes.c_void_p(buf.data_ptr() + 2 * g.ch_off), buf.shape[-1],
                                     L.stream_ptr(buf.device)), "dilate_merge")
    torch.cuda.synchronize()
    got = interior(buf, g.ch_off, g.c)
    assert merge_check(got, prior, d["v"], True)
    out["merge overwrites instead of accumulating"] = 2.0 if not merge_check(got, prior, d["v"], False) else 0.0
    # one branch use missing from an owner's gradient
    o = s["owner"]
    uses = s["uses"]
    j = sorted(uses)[len(uses) // 2]
    wj, bj = uses[j]
    out["owner gradient missing one use"] = float(((o["final"] - (o["want"] - wj)).abs() / (o["bound"] - bj)).max())
    # zero-insert at the odd pixels
    zi = s["zi"]
    up_odd = torch.zeros_like(zi["up"])
    n_odd = up_odd[:, 1::2, 1::2].shape
    up_odd[:, 1::2, 1::2] = zi["dz"][:, :n_odd[1], :n_odd[2]]
    out["zero-insert at the odd pixels"] = 0.0 if bitwise(zi["up"], up_odd) else 2.0
    # block 109: the PReLU kink taken at z instead of z + bias
    k = s["b109"]
    args = (k["z"], k["dy"], k["dz"], k["sums"], k["bias"], k["slope"], k["chain"])
    assert passed(bias_act_bwd_check(*args))
    out["block 109 kink at z"] = bias_act_bwd_check(*args, kink_at_z=True)["max"]
    # a bias added to a weight_from head
    hd = s["head"]
    assert f32_check(hd["got"], hd["want"], hd["e"])["max"] <= 1.0
    out["bias on a weight_from head"] = f32_check(hd["got"], hd["want"] + hd["bias"], hd["e"])["max"]
    print("\n[bite] " + ", ".join("%s %.3g" % kv for kv in out.items()))
    bad = {kk: v for kk, v in out.items() if not v > 1.0}
    assert not bad, bad
