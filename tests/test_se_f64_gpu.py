"""Every kernel of the bf16 training step and of the detect forward of the reference's squeeze-excitation recipes against
float64 of the inputs each launch received: cfg/HRSC+/yolov3_512_se.cfg with HRSC+/hyp.txt and cfg/ICDAR/yolov3_608_se.cfg
with ICDAR/hyp.txt, both at the recipes' batch 4 and arc 'defaultpw' (train.py keeps the BCE positive weights obj_pw
3.941 and cls_pw 1.446 for arcs containing 'pw').  Both recipes are single-class (classes=1): the loss has no class term
and the class column's cotangent is exactly 0, so cls_pw reaches no kernel on these graphs.

Training step (checked_step.run_step, the real loss: loss.compute_loss, the fused path), at se512 (4 x 512^2), se512
at 4 x 416^2 (grids 13 / 26 / 52: odd SE spans, inside the recipe's multi-scale range 384-640) and se608 (4 x 608^2),
on loss_f64.make_targets (matched rows on every head, two rows on one cell, one row outside the map):
  every launch      checked_step's forward_checks and check_block_bwd with the bounds of test_train_step_f64_gpu: im2col
                    and the weight packs bit for bit, conv z, BN statistics and running statistics, bn_act_fwd,
                    bn_act_bwd, wgrad, dgrad, the head's fp32 z, the head dz bit for bit, the head bias sums, the .grad
                    gathers bit for bit (the SE weights' too), every halo zero
  SE                ryolo_se_fwd post hoc and ryolo_se_bwd through the wrapped plan._se_bwd (checked_step.check_se_bwd),
                    both on their own inputs; the producing block's bn_act_bwd is checked on the gx the SE left, which is
                    what it reads.  Bounds (U = 2^-24, the fp32 unit roundoff; f64_refs.se_fwd_refs / se_bwd_refs):
    m, ds           L U sum|terms| (+ U |m| for the division), L = the longest fp32 addition chain of the launch: the
                    pixels one thread adds in its span, the lanes of a channel, the spans (f64_refs.se_chain mirrors
                    se_nsplit in csrc/se.cu)
    p, dhid         (n + 1) U |W| |v|, n terms; dhid also carries da's 3 U relative error; dm carries dhid's error
                    through W1^T
    s               s (1 - s) (cr + 1) U |W2| |relu(p)| + 4 U s   (expf, the add and the division)
    gW1, gW2        (B + 1) U sum_b |a||b| plus the propagated error of da / dhid
    u, gx           half a bf16 ulp of the float64 result + the fp32 terms (3 U each), and no rounding bias:
                    |mean((got - want) sign(want))| <= 2^-12 rms(want)
  loss, cotangent   loss_f64 (the bounds of test_multiclass_f64_gpu, which carry lw = 1 + (pw - 1) t) at obj_pw 3.941
Wiring, through the plan's pointers: the 1x1 conv after each SE reads u, each `from=-4` shortcut adds x, the SE inputs
36 / 61 live in the concat buffers of routes 118 / 106 and their gx has three writers (the concat consumer's dgrad
first, the shortcut gradient and the SE accumulating).

Detect forward (eval, CUDA-graph replay on a second input) at se512 4 x 512^2, se512 2 x 288 x 512 (the letterbox of a
16:9 frame, oh != ow) and se608 4 x 608^2: every conv with check_conv, every se_fwd step with check_se_step (the SE
bounds above), check_buffers and the decode within 2^-20 M of f64_refs.decode_ref.  The in-place eval SE
(ryolo_se_block, used when nothing reads the SE's input again, never in the reference's cfgs) runs at batch 4 at the
(c, h, w) of all 20 SEs of both cfgs: the channel sums within their own chain (f64_refs.se_block_chain: the pixels a
thread adds, then one atomicAdd per thread and row block in any order), s from the kernel's sums as above (the mean's
fp32 1 / hw carried through W1), u as above, halo and padding channels untouched; and once through map_plan on a small
graph where the eval plan takes it (check_conv then bounds the conv output the SE scaled in place).

Measured on an H100 80GB HBM3 (132 SMs, power limit 700 W, 1980 MHz max SM clock), seeds as below; worst |err| / bound
per kernel kind over all launches (layer in parentheses), se512 / se512 at 416 / se608:
  conv z, bn_act_fwd, bn_act_bwd, dgrad   0.996 / 0.996 / 0.996 (half a bf16 ulp at the bottom of a binade, see
                     test_train_step_f64_gpu); BN sums 0.122 / 0.134 / 0.115, finalize 0.571 / 0.561 / 0.589, running
                     0.020 / 0.021 / 0.024; wgrad 0.454 / 0.529 / 0.501; d beta, d gamma <= 0.095; d slope <= 0.002
  heads              fp32 z 0.168 / 0.144 / 0.162; dgrad 0.993 / 0.994 / 0.993; wgrad <= 0.112; bias sums 0.079 / 0.108 /
                     0.097; dz bit for bit
  SE forward         m 0.093 / 0.105 / 0.090; p 0.002; s 0.408 / 0.463 / 0.331; u 0.996, bias <= 0.075
  SE backward        ds 0.040 / 0.053 / 0.040; dm 0.002; gW1 0.002; gW2 0.465 / 0.476 / 0.399; gx 0.996, bias <= 0.017
  loss, cotangent    lobj 0.030 / 0.023 / 0.023, lcls 0 and lreg < 0.001; objectness <= 0.248, regression columns
                     <= 0.471, class column 0; up to 2 rows per cell, 14 / 14 / 18 matched rows outside the map
  detect             se512 / letterbox / se608: convs <= 0.996, heads <= 0.124; se_fwd m <= 0.096, s <= 0.404, u 0.996
                     (bias <= 0.465); decode <= 0.204
  ryolo_se_block     sums 0.035, s 0.003, u 0.996 (bias 0.122) over the 6 distinct shapes of the 40 SEs; through the eval
                     plan: the conv output it scaled 0.952, s 0.188
Two runs print the same ratios except the in-place SE's channel sums, whose atomicAdd order varies (0.034 / 0.035).
Bugs put in (test_bounds_reject_plausible_bugs), worst |err| / bound at se512: conv i + 1 reading x instead of u 3.8e4;
the from=-4 residual taken as u 6.7e6; bn_act_bwd of the SE's producer fed gx from before the SE 1.2e6; the concat
consumer's dgrad accumulating onto gx 1.7e8; the 1x1 dgrad accumulating into gu 258; the SE's gx without dm / hw 1.8e6,
or overwritten 2.8e6; eval se_fwd applying image 0's s to every image 1.98 (1.54 at se608); u rounded toward zero
(bias) 8.7; obj_pw taken as 1 1.4e6.  No kernel needed a change.  Whole file: 29 s."""
import os
import time
import types

import pytest
import torch

from builders import REF_CFG, in_dir, pkg
from checked_step import (Run, Step, bn_bwd_check, check_buffers, check_conv, check_first, check_s2d_step, check_se_step,
                          map_plan, run_step, ses_of)
from f64_refs import (BF16, U, bad_entries, bf16_check, bn_act_fwd_ref, check_z, conv_taps, decode_ref, halo_zero, ratio,
                      rtz_bf16, se_block_chain, se_block_s_ref, se_bwd_refs, sum_check, tapsum, vint)
from helpers import cfg_conv, init_darknet_weights
from loss_f64 import cot_check, fused_loss, loss64, loss_checks, make_targets, read_hyp, record_head_grads

pytestmark = pytest.mark.gpu

RECIPES = {"HRSC+": ("cfg/HRSC+/yolov3_512_se.cfg", "cfg/HRSC+/hyp.txt"),
           "ICDAR": ("cfg/ICDAR/yolov3_608_se.cfg", "cfg/ICDAR/hyp.txt")}
STEPS = {"se512": ("HRSC+", 4, 512, 512), "se512_416": ("HRSC+", 4, 416, 416), "se608": ("ICDAR", 4, 608, 608)}
DETECT = {"se512": ("HRSC+", 4, 512, 512), "se512_letterbox": ("HRSC+", 2, 288, 512), "se608": ("ICDAR", 4, 608, 608)}
ARC = "defaultpw"
KEEP_SE = 37            # the SE whose input (layer 36) lives in a concat buffer: its stored tensors feed the bug test


def make_model(recipe, seed):
    """the recipe's Darknet as train.py builds it (hyp from hyp.txt, arc 'defaultpw', model.nc / model.hyp set)"""
    cfg, hyp_path = RECIPES[recipe]
    hyp = read_hyp(os.path.join(REF_CFG, hyp_path))
    with in_dir(REF_CFG):                  # the SE cfgs name their anchor files relative to the reference root
        m = pkg().Darknet(cfg, hyp, arc=ARC)
    m.hyp, m.nc = hyp, 1
    return init_darknet_weights(m, seed=seed), hyp


# ---------------------------------------------------------------------------------------------------------------
def se_step(name, seed=51):
    recipe, batch, h, w = STEPS[name]
    dev = torch.device("cuda")
    t0 = time.time()
    model, hyp = make_model(recipe, seed)
    model = model.to(dev).train()
    st = Step(model, torch.rand(batch, 3, h, w, generator=torch.Generator().manual_seed(seed + 1)).to(dev))
    st.nc, st.hyp, st.cot = 1, hyp, {}
    st.targets = make_targets(model, 1, batch, h, w, seed + 2)
    k = KEEP_SE
    # the producing block of x (layer k - 1), the 1x1 conv reading u, the 3x3 conv adding x, and the concat consumer
    # whose dgrad writes gx first: their stored tensors feed test_bounds_reject_plausible_bugs
    st.keep_se = {k}
    st.keep_fwd = {k + 1, k + 2}

    def prepare(st):
        se = next(s for s in ses_of(st.plan) if s.i == k)
        prod = next(b for b in st.plan.blocks if getattr(b, "se", None) is se)
        cons = [b for b in st.plan.blocks if b.gsrc is not None and b.gsrc.buf is se.gx.buf and b.gsrc.c > se.x.c]
        st.keep_bwd = {prod.i, k + 1} | {b.i for b in cons}
        st.stash["se_io"] = dict(x=vint(se.x).clone(), u=vint(se.u).clone(), prod=prod.i,
                                 cons=[b.i for b in cons])
    run_step(st, loss=lambda st, ps: fused_loss(st, ps, hyp), head_grads=record_head_grads, prepare=prepare)
    # the gradients the buffers of gu and the concat hold at the end of the step: what a dgrad that wrongly accumulates
    # would find there at the next step
    se = next(s for s in ses_of(st.plan) if s.i == k)
    cons = st.stash["se_io"]["cons"]
    st.stash["end"] = dict(gu=vint(se.gu).clone(),
                           gcons=vint(next(b for b in st.plan.blocks if b.i == cons[0]).gsrc).clone() if cons else None)
    loss_checks(st)
    st.t_total = time.time() - t0
    _print_step(name, st)
    return st


KINDS = (("f", ("z", "z_bias", "mean", "invstd", "sums", "finalize", "running", "y", "y_bias")),
         ("se f", ("m", "p", "s", "u_max", "u_bias")),
         ("se b", ("ds", "dm", "gw1", "gw2", "gx_max", "gx_bias")),
         ("b", ("dz", "dz_bias", "dbeta", "dgamma", "dslope", "wgrad", "dgrad", "dgrad_bias", "dbias")))


def _print_step(name, st):
    tag = "[se step %s %dx%dx%d]" % (name, st.batch, st.h, st.w)
    print("\n%s whole step with checks %.1f s" % (tag, st.t_total))
    ses = {se.i for se in ses_of(st.plan)}
    heads = {b.i for b in st.plan.blocks if b.is_head}
    worst = {}
    for pre, keys in KINDS:
        src = st.bwd if pre.endswith("b") else st.fwd
        for i, r in src.items():
            if (i in ses) != pre.startswith("se"):
                continue
            for key in keys:
                v = r.get(key)
                if isinstance(v, float):
                    kk = "%s%s:%s" % ("head " if i in heads else "", pre, key)
                    if not worst.get(kk, (-1.0,))[0] >= v:
                        worst[kk] = (v, i)
    print("%s worst |err| / bound per kind (layer): %s" % (tag, ", ".join("%s %.3f (%d)" % (k, v, i)
                                                                          for k, (v, i) in sorted(worst.items()))))
    print("%s loss value / bound: %s" % (tag, ", ".join("%s %.3f" % kv for kv in st.loss_r.items())))
    for i, r in st.cot_r.items():
        print("%s head %d cotangent / bound: obj %.3f  class column %.3f  regression columns %.3f  zeros %s  "
              "(%d matched cells)" % (tag, i, r["obj"], r["cls"], r["reg"], r["zero"], r["matched_cells"]))
    print("%s rows: up to %d per cell, %d matched rows outside the map" % (tag, st.max_rows_per_cell, st.border_rows))


# ---------------------------------------------------------------------------------------------------------------
def decode_ratio(got, want, mag):
    r = (got.double() - want).abs() / (mag * 2.0 ** -20)
    r = torch.where(got.double() == want, torch.zeros_like(r), r)
    return float(r.max()) if not bool(r.isnan().any()) else float("nan")


def run_detect(name, seed=53):
    """the eval forward replayed as a CUDA graph on a second input; every conv and SE step, the buffers and the decode
    against float64"""
    recipe, batch, h, w = DETECT[name]
    dev = torch.device("cuda")
    t0 = time.time()
    model, hyp = make_model(recipe, seed)
    model = model.to(dev).eval()
    model.use_cuda_graph = True
    xa, xb = (torch.rand(batch, 3, h, w, generator=torch.Generator().manual_seed(seed + s)).to(dev) for s in (1, 2))
    st = Run(name, model)
    with torch.no_grad():
        io_a = model(xa)[0].clone()
        st.io, _ = model(xb)
    torch.cuda.synchronize()
    st.replayed = model._graph is not None and model.replayed_kernels == 2 * model._graph_kernels
    st.io_changed = not torch.equal(io_a, st.io)
    st.plan, st.x, st.stash, st.keep = model._plan, model._x_static, {}, {KEEP_SE}
    st.x_is_xb = torch.equal(st.x, xb)
    map_plan(st)
    convs = sorted(st.conv_of)
    st.res = {0: check_first(st)}
    for i in convs[1:]:
        st.res[i] = check_conv(st, i)
    st.s2d = {i: check_s2d_step(st, i) for i in st.s2d_of}
    st.se = {i: check_se_step(st, i) for i in st.se_of}
    st.buffers_ok, _ = check_buffers(st)
    st.decode, off = [], 0
    for (li, p), yi in zip(st.plan["heads"], model.yolo_layers):
        layer = model.module_list[yi]
        want, mag = decode_ref(p, layer.anchors.float(), float(layer.stride), float(hyp["context_factor"]), 1)
        st.decode.append(decode_ratio(st.io[:, off:off + want.shape[1]], want, mag))
        off += want.shape[1]
        del want, mag
    st.io_rows = off == st.io.shape[1]
    st.t_total = time.time() - t0
    tag = "[se detect %s %dx%dx%d]" % (name, batch, h, w)
    worst = {}
    for i, r in list(st.res.items()) + list(st.se.items()):
        kind = "first" if i == 0 else r["kind"]
        for key in ("max", "bias", "m", "p", "s", "u_max", "u_bias"):
            if isinstance(r.get(key), float) and not worst.get((kind, key), (-1.0,))[0] >= r[key]:
                worst[(kind, key)] = (r[key], i)
    print("\n%s %.1f s; worst |err| / bound per kind (layer): %s; decode %s" % (
        tag, st.t_total, ", ".join("%s %s %.3f (%d)" % (k[0], k[1], v, i) for k, (v, i) in sorted(worst.items())),
        ", ".join("%.3f" % v for v in st.decode)))
    return st


_CACHE = {}


def _get(kind, name):
    key = (kind, name)
    if key not in _CACHE:
        _CACHE[key] = se_step(name) if kind == "step" else run_detect(name)
    return _CACHE[key]


@pytest.fixture(scope="module", params=list(STEPS))
def step(request):
    return _get("step", request.param)


# ---------------------------------------------------------------------------------------------------------------
def test_recipes_keep_the_positive_weights():
    """the hyp files as train.py reads them, with arc 'defaultpw' leaving obj_pw / cls_pw in place (train.py:43-45)"""
    for recipe, iou_t in (("HRSC+", 0.5), ("ICDAR", 0.3)):
        hyp = read_hyp(os.path.join(REF_CFG, RECIPES[recipe][1]))
        assert hyp["obj_pw"] == 3.941 and hyp["cls_pw"] == 1.446 and hyp["iou_t"] == iou_t and hyp["batch_size"] == 4
        assert abs(hyp["ang_t"] - 3.1415926 / 12) < 1e-12
    assert "pw" in ARC and "default" in ARC


def test_se_wiring(step):
    plan = step.plan
    ses = ses_of(plan)
    assert len(ses) == 20
    by_i = {b.i: b for b in plan.blocks}
    for se in ses:
        prod = next(b for b in plan.blocks if getattr(b, "se", None) is se)
        assert prod.y is se.x and prod.gy is se.gx and prod.i == se.i - 1 - (prod.res is not None), se.i
        conv1 = by_i[se.i + 1]
        assert conv1.k == 1 and conv1.src is se.u and conv1.gsrc is se.gu, se.i
        conv3 = by_i[se.i + 2]
        assert conv3.fuse_res and conv3.res is se.x and conv3.gres is se.gx, se.i
        assert se.u.buf.data_ptr() != se.x.buf.data_ptr()
    for i in (37, 62):
        se = next(s_ for s_ in ses if s_.i == i)
        assert se.x.buf.shape[-1] > se.x.c                       # x lives in the concat buffer of route 118 / 106
        concat = [b for b in plan.blocks if b.gsrc is not None and b.gsrc.buf is se.gx.buf and b.gsrc.c > se.x.c]
        assert len(concat) == 1 and not concat[0].gsrc_acc        # the concat consumer's dgrad writes gx first ...
        assert by_i[i + 2].gres_acc and se.gx_acc                # ... the shortcut gradient and the SE accumulate
    # every SE input is also a shortcut source, whose gradient (the 3x3 block's bn_act_bwd) comes first: the SE accumulates
    assert all(s_.gx_acc for s_ in ses)


def test_covers_every_launch(step):
    """every launch of the backward schedule and every forward block and SE tied to a check; every eval step too"""
    st = step
    plan = st.plan
    ses = {se.i for se in ses_of(plan)}
    assert set(st.fwd) == {b.i for b in plan.blocks} | ses and len(plan.blocks) == 75
    missing = []
    for kind, i, flag in plan.sched.ops(plan):
        r = st.bwd.get(i, {})
        ok = {"head": "dz_bits" in r and "dbias" in r, "bnact": "dz" in r, "wgrad": "wgrad" in r,
              "dgrad": "dgrad" in r, "se": "ds" in r and "gx_max" in r and "gw_bits" in r}.get(kind, False)
        if not ok:
            missing.append((kind, i, flag))
    assert not missing, missing
    ops = plan.sched.ops(plan)
    assert {k for k, _, _ in ops} == {"head", "bnact", "wgrad", "dgrad", "se"}
    assert {i for k, i, _ in ops if k == "se"} == ses
    for i in ses:
        assert {"m", "p", "s", "u_max", "u_bias", "halo_u"} <= set(st.fwd[i]), i
    name = next(n for n, s in _CACHE.items() if s is st)[1]
    if name in DETECT:
        dt = _get("detect", name)
        kinds = [k for k, _ in dt.plan["steps"]]
        assert set(kinds) == {"first", "conv", "s2d", "se_fwd"}, set(kinds)
        assert kinds.count("se_fwd") == 20 and len(dt.se) == 20
        assert sorted(dt.res) == sorted(dt.conv_of) and len(dt.res) == 75
        checked = set(dt.conv_of.values()) | set(dt.s2d_of.values()) | set(dt.se_of.values())
        assert checked == set(range(len(kinds)))


def test_training_step_kernels_vs_float64(step):
    st = step
    assert st.fwd_halo and st.nbt_ok
    assert st.im2col == dict(bits=True, pad_zero=True, halo=True), st.im2col
    assert all(p[2] for p in st.packs), [p[:2] for p in st.packs if not p[2]]
    bad = bad_entries(st.fwd) + bad_entries(st.bwd)
    assert not bad, bad
    for i, r in st.bwd.items():
        if "near_zero_u" in r:
            assert r["near_zero_u"] <= max(64, r["n_elems"] // 100000), (i, r["near_zero_u"])


def test_se_forward_kernels_vs_float64(step):
    ses = {se.i for se in ses_of(step.plan)}
    bad = bad_entries({i: r for i, r in step.fwd.items() if i in ses})
    assert not bad, bad


def test_se_backward_kernels_vs_float64(step):
    ses = {se.i for se in ses_of(step.plan)}
    assert ses <= set(step.bwd)
    bad = bad_entries({i: r for i, r in step.bwd.items() if i in ses})
    assert not bad, bad
    assert all(step.bwd[i]["acc"] == 1 for i in ses)


def test_loss_and_head_cotangent_vs_float64(step):
    st = step
    assert st.masks_equal
    assert st.max_rows_per_cell >= 2 and st.border_rows > 0
    bad = {k: v for k, v in st.loss_r.items() if not v <= 1.0}
    assert not bad, (bad, st.loss_r)
    for i, r in st.cot_r.items():
        assert r["zero"] and r["matched_cells"] > 0, (i, r)
        assert r["obj"] <= 1.0 and r["cls"] <= 1.0 and r["reg"] <= 1.0, (i, r)


@pytest.mark.parametrize("name", list(DETECT))
def test_detect_forward_vs_float64(name):
    dt = _get("detect", name)
    assert dt.replayed and dt.io_changed and dt.x_is_xb and dt.io_rows
    bad = [(i, k, r[k]) for i, r in dt.res.items() for k in ("max", "bias") if k in r and not r[k] <= 1.0]
    bad += [(i, k) for i, r in dt.res.items() for k in ("w_bits", "b_bits", "slope", "up_copies") if k in r and not r[k]]
    bad += bad_entries({i: {k: v for k, v in r.items() if k != "kind"} for i, r in dt.se.items()})
    assert not bad, bad
    assert dt.buffers_ok and all(v["bits"] and v["pad_zero"] for v in dt.s2d.values())
    assert all(v <= 1.0 for v in dt.decode), dt.decode
    # wiring: conv i + 1 reads u, the from=-4 residual of conv i + 2 is x (map_plan asserts the pointers)
    for i, k in dt.se_of.items():
        a = dt.plan["steps"][k][1]
        assert dt.plan["steps"][dt.conv_of[i + 1]][1]["x"] == a["u"]
        assert dt.plan["steps"][dt.conv_of[i + 2]][1]["r"] == a["x"]


# ---------------------------------------------------------------------------------------------------------------
# ryolo_se_block: the in-place eval SE
def se_block_case(b, h, w, c, w1, w2, seed):
    """ryolo_se_block on a padded-NHWC bf16 x with 64 channels beyond c; returns the checks"""
    from rotate_yolov3_b200 import layout as L
    lib, dev = pkg()._lib, torch.device("cuda")
    g = torch.Generator().manual_seed(seed)
    cs = c + 64
    mu = torch.randn(c, generator=g) * 0.5
    x = (torch.randn(b, c, h, w, generator=g) + mu.view(1, c, 1, 1)).to(dev)
    buf = L.to_padded_nhwc(x, cs)
    buf[:, 1:-1, 1:-1, c:] = torch.randn(b, h, w, 64, generator=g).to(dev).to(BF16)     # not the SE's channels
    before = buf.clone()
    x = buf[:, 1:-1, 1:-1, :c].clone()
    cr = w1.shape[0]
    sums = torch.full((b * c,), float("nan"), device=dev)
    scale = torch.full((b * c,), float("nan"), device=dev)
    st = lib.lib.ryolo_se_block(lib.ptr(buf), cs, b, h, w, c, lib.ptr(w1), lib.ptr(w2), cr, lib.ptr(sums), lib.ptr(scale),
                                lib.stream_ptr(dev))
    assert st == 0, lib.last_error()
    torch.cuda.synchronize()
    xd = x.double()
    r = {"sums": sum_check(sums.view(b, c), xd.sum((1, 2)), se_block_chain(h, w, c), xd.abs().sum((1, 2)))}
    s = scale.view(b, c)
    r["s"] = ratio(s, *se_block_s_ref(sums.view(b, c), w1.double(), w2.double(), h * w))
    u64 = xd * s.double().view(b, 1, 1, c)
    ru = bf16_check(buf[:, 1:-1, 1:-1, :c], u64, 3 * U * u64.abs())
    r["u_max"], r["u_bias"] = ru["max"], ru["bias"]
    r["untouched"] = torch.equal(buf[..., c:], before[..., c:]) and halo_zero(buf)
    return r, dict(x=x, s=s, u=buf[:, 1:-1, 1:-1, :c].clone(), u64=u64)


def test_se_block_in_place_vs_float64():
    """ryolo_se_block at batch 4 at the (c, h, w) of all 20 SEs of both cfgs, with each SE's own weights"""
    shapes = {}
    for name in ("se512", "se608"):
        dt = _get("detect", name)
        for i, k in dt.se_of.items():
            a = dt.plan["steps"][k][1]
            shapes.setdefault((a["c"], a["h"], a["w"]), []).append((name, i, a["w1"], a["w2"]))
    assert sum(len(v) for v in shapes.values()) == 40
    out, worst = {}, {}
    for n, ((c, h, w), uses) in enumerate(sorted(shapes.items())):
        for name, i, w1, w2 in uses:
            r, _ = se_block_case(4, h, w, c, w1, w2, seed=100 + i)
            out[(name, i)] = r
            for k, v in r.items():
                if isinstance(v, float) and not worst.get(k, (-1.0,))[0] >= v:
                    worst[k] = (v, "%s %d (%dx%dx%d)" % (name, i, c, h, w))
    print("\n[se block] %d shapes; worst: %s" % (len(shapes), ", ".join("%s %.3f (%s)" % (k, v, i)
                                                                         for k, (v, i) in sorted(worst.items()))))
    bad = bad_entries(out)
    assert not bad, bad


def test_se_block_in_place_through_the_eval_plan():
    """a graph whose [se] input nothing reads again: the eval plan takes the in-place kernel, map_plan maps the scaled
    output as layer i - 1's, check_conv bounds that conv's output through the scale, check_se_step the scale"""
    text = ("[net]\nwidth=64\nheight=48\nchannels=3\n\n" + cfg_conv(32, 3) + cfg_conv(64, 3, 2) +
            "[se]\nchannels=64\n\n" + cfg_conv(32, 1) + cfg_conv(64, 3) + "[shortcut]\nfrom=-3\nactivation=linear\n\n" +
            cfg_conv(14, 1, bn=0, act="linear") +
            "[yolo]\nmask = 0-1\nanchors = ara 900 / 5.0 / -45, 45\nclasses=1\nnum=2\n\n")
    model = init_darknet_weights(pkg().Darknet(text, {"context_factor": 1.0}), seed=5).cuda().eval()
    x = torch.rand(2, 3, 48, 64, generator=torch.Generator().manual_seed(6)).cuda()
    st = Run("se in place", model)
    with torch.no_grad():
        model(x)
    torch.cuda.synchronize()
    st.plan, st.x, st.stash = model._plan, x, None
    map_plan(st)
    assert [k for k, _ in st.plan["steps"]].count("se") == 1 and list(st.se_of) == [2] and list(st.scaled) == [1]
    res = {0: check_first(st)}
    for i in sorted(st.conv_of)[1:]:
        res[i] = check_conv(st, i)
    res[2] = check_se_step(st, 2)
    bad = bad_entries({i: {k: v for k, v in r.items() if k not in ("kind", "cout", "grid")} for i, r in res.items()})
    assert not bad, bad
    assert check_buffers(st)[0]
    # the residual of the shortcut is the scaled tensor; a bound that ignored the scale fails
    assert st.plan["steps"][st.conv_of[4]][1]["r"] == st.outs[1].ptr
    print("\n[se block graph] conv 1 (scaled in place) %.3f, s %.3f" % (res[1]["max"], res[2]["s"]))
    st.scaled = {}
    assert check_conv(st, 1)["max"] > 1.0


# ---------------------------------------------------------------------------------------------------------------
def bn_bwd_check_ref(bn, dy):
    """the stored bn_act_bwd launch of a block checked against float64 with dy as the gradient it read: worst ratio of
    dz, d beta and d gamma"""
    r, _ = bn_bwd_check(bn["z"], dy, bn["dz"], bn["sums"], bn["mean"], bn["invstd"], bn["sc"], bn["sh"], bn["slope"],
                        bn["chain"])
    return max(r["max"], r["dbeta"], r["dgamma"])


def test_bounds_reject_plausible_bugs(step):
    """each bug, put into a stored tensor or a reference, fails the check that guards it; the factors are printed"""
    st = step
    k = KEEP_SE
    io, end = st.stash["se_io"], st.stash["end"]
    out = {}
    # conv k + 1 (the 1x1 after the SE) computed from x instead of u
    z = st.stash[("z", k + 1)]
    assert check_z(z["got"], z["want"], z["mag"], z["n"])["max"] <= 1.0
    blk = next(b for b in st.plan.blocks if b.i == k + 1)
    w64 = st.model.module_list[k + 1].Conv2d.weight.detach().to(BF16).double()
    want_x, mag_x = tapsum(io["x"], conv_taps(w64), blk.oh, blk.ow)
    out["conv i+1 reads x instead of u"] = check_z(z["got"], want_x, mag_x, z["n"])["max"]
    # the from=-4 residual taken as u
    y = st.stash[("y", k + 2)]
    want_y, t = bn_act_fwd_ref(y["z"], y["sc"], y["sh"], y["slope"], y["res"])
    assert bf16_check(y["got"], want_y, 0.0, t)["max"] <= 1.0
    want_y, t = bn_act_fwd_ref(y["z"], y["sc"], y["sh"], y["slope"], io["u"])
    out["from=-4 residual taken as u"] = bf16_check(y["got"], want_y, 0.0, t)["max"]
    # bn_act_bwd of the SE-producing block fed gx from before the SE added into it
    bn, se_k = st.stash[("bn", io["prod"])], st.stash[("se", k)]
    rb = bn_bwd_check_ref(bn, bn["dy"])
    assert rb <= 1.0, rb
    out["bn_act_bwd fed gx before the SE"] = bn_bwd_check_ref(bn, se_k["gx_old"].float())
    # the concat consumer's dgrad accumulating onto gx instead of writing it first
    d = st.stash[("dgrad", io["cons"][0])]
    assert not d["acc"]
    want, mag = tapsum(d["dz"], conv_taps(d["w64"], mirror=True), d["h"], d["w"])
    e = d["n"] * 2.0 ** -23 * mag
    assert bf16_check(d["got"], want, e)["max"] <= 1.0
    out["concat dgrad accumulates onto gx"] = bf16_check((d["got"].float() + end["gcons"].float()).to(BF16), want, e)["max"]
    # the 1x1 dgrad accumulating into gu
    d = st.stash[("dgrad", k + 1)]
    assert not d["acc"]
    want, mag = tapsum(d["dz"], conv_taps(d["w64"], mirror=True), d["h"], d["w"])
    e = d["n"] * 2.0 ** -23 * mag
    assert bf16_check(d["got"], want, e)["max"] <= 1.0
    out["1x1 dgrad accumulates into gu"] = bf16_check((d["got"].float() + end["gu"].float()).to(BF16), want, e)["max"]
    # the SE backward's gx without dm / hw, and overwritten instead of accumulated
    B, se = st.batch, next(s for s in ses_of(st.plan) if s.i == k)
    s_ = se.s.view(B, se.c)
    gxr = se_k["refs"]["gx"]
    gus = se_k["gu"].float() * s_.view(B, 1, 1, se.c)
    out["SE gx without dm / hw"] = bf16_check((se_k["gx_old"].float() + gus).to(BF16), *gxr)["max"]
    out["SE gx overwritten"] = bf16_check((gus + (se.dm.view(B, se.c) / (se.h * se.w)).view(B, 1, 1, se.c)).to(BF16),
                                          *gxr)["max"]
    # eval se_fwd applying image 0's s to every image; u rounded toward zero
    name = next(n for n, s in _CACHE.items() if s is st)[1]
    if name in DETECT:
        e_ = _get("detect", name).stash[("se", k)]
        c = e_["x"].shape[-1]
        s0 = e_["s"].view(-1, c)
        assert bf16_check(e_["u"], *e_["refs"]["u"])["max"] <= 1.0
        out["eval se_fwd with image 0's s"] = bf16_check((e_["x"].float() * s0[0]).to(BF16), *e_["refs"]["u"])["max"]
        out["eval u rounded toward zero (bias)"] = bf16_check(rtz_bf16(e_["x"].float() * s0.view(-1, 1, 1, c)),
                                                              *e_["refs"]["u"])["bias"]
    # obj_pw taken as 1 in the objectness cotangent (the float64 loss at obj_pw 1)
    c = st.stash["cot"]
    assert cot_check(c["got"], c["want"], c["m"], c["ncell"])["obj"] <= 1.0
    hyp = st.model.hyp
    st.model.hyp = dict(hyp, obj_pw=1.0)
    try:
        p64 = [p.double().requires_grad_(True) for p in c["p32"]]
        comps, _ = loss64(p64, st.targets.double(), st.model, st.model.hyp)
        sum(comps).sum().backward()
    finally:
        st.model.hyp = hyp
    out["obj_pw taken as 1"] = cot_check(c["got"], p64[-1].grad, c["m"], c["ncell"])["obj"]
    print("\n[se bugs %s] |err| / bound: %s" % (name, ", ".join("%s %.3g" % kv for kv in out.items())))
    bad = {k_: v for k_, v in out.items() if not v > 1.0}
    assert not bad, bad


def test_se_kernels_first_writer_accumulate_and_relu_at_zero():
    """ryolo_se_bwd alone: gx as the first writer and accumulating (the reference graphs only accumulate), and hidden units
    with p == 0 exactly (a zero row of W1) pass no gradient, like torch's relu backward"""
    from rotate_yolov3_b200 import layout as L
    lib, dev = pkg()._lib.lib, torch.device("cuda")
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
    P, st = pkg()._lib.ptr, pkg()._lib.stream_ptr(dev)
    assert lib.ryolo_se_fwd(P(x), 256, P(u), 256, B, h, w, c, P(w1), P(w2), cr, P(m), P(p), P(s), P(ws), ws.numel(), st) == 0
    assert lib.ryolo_se_bwd(P(gu), 256, P(x), 256, P(gx), 256, 0, B, h, w, c, P(w1), P(w2), cr, P(m), P(p), P(s), P(ds), P(dm),
                            P(gw1), P(gw2), P(ws), ws.numel(), st) == 0
    torch.cuda.synchronize()
    se = types.SimpleNamespace(h=h, w=w, c=c, cr=cr, m=m, p=p, s=s, ds=ds, dm=dm)
    xi, gui = x[:, 1:-1, 1:-1], gu[:, 1:-1, 1:-1]
    r = bf16_check(gx[:, 1:-1, 1:-1], *se_bwd_refs(se, gui, xi, None, w1.double(), w2.double(), gw1, gw2)["gx"])
    assert r["max"] <= 1 and r["bias"] <= 1, r                     # first writer
    gx_old = gx.clone()
    assert lib.ryolo_se_bwd(P(gu), 256, P(x), 256, P(gx), 256, 1, B, h, w, c, P(w1), P(w2), cr, P(m), P(p), P(s), P(ds), P(dm),
                            P(gw1), P(gw2), P(ws), ws.numel(), st) == 0
    torch.cuda.synchronize()
    r = bf16_check(gx[:, 1:-1, 1:-1], *se_bwd_refs(se, gui, xi, gx_old[:, 1:-1, 1:-1], w1.double(), w2.double(), gw1,
                                                   gw2)["gx"])
    assert r["max"] <= 1 and r["bias"] <= 1, r                     # accumulating
    assert halo_zero(gx) and halo_zero(u)
    assert bool((p.view(B, cr)[:, 3] == 0).all())
    assert bool((gw1.view(cr, c)[3] == 0).all()) and bool((gw2.view(c, cr)[:, 3] == 0).all())
    assert float(gw1.view(cr, c).abs().sum()) > 0
