"""The bf16 training step and the detect forward of multi-class models against float64 of the inputs each kernel
received: cfgs.yolov3_cfg(classes=15) at batch 2 x 608^2 (the bench graph with 1512-filter heads) and
cfgs.yolov3_cfg(classes=22, width=416, height=320) at batch 3 (2016-filter heads, the widest the training backward
takes; an odd batch, h != w, grids 10 x 13, 20 x 26, 40 x 52).  The single-class files run 504-filter heads only: here
the head convs have a partial last N tile (1512) or fill the 2048-wide one, the head wgrad runs at cout_pad 1536 / 2048,
the head dgrad at K = 1536 / 2048, head_grad_nchw_kernel needs its opt-in shared tile, and the decode its direct path.

Training step, with the real loss (compute_loss, the fused path) on targets that reach every branch of it: classes
0, nc - 1 and between, five per image, two rows on one cell (the scatter chains), one target on the right border (its
rows fall outside every map: the fused path gathers 0 for them and writes nothing; the reference would raise).
  every launch       checked_step's forward_checks and check_block_bwd (the bounds of test_train_step_f64_gpu), on the
                     cotangent the loss produced: conv z, BN statistics, bn_act_fwd / bn_act_bwd, wgrad, dgrad; at the
                     heads fp32 z, the head cotangent bit for bit as RN-bf16 with its padding channels and halo zero,
                     the bias sums under head_bias_chain, wgrad_ratio at cout_pad 1536 / 2048, the dgrad at K = 1536 / 2048
  loss and cotangent a float64 restatement of _compute_loss_masked (its target assignment, _sparse_terms, _obj_term; in
                     loss_f64, shared with test_se_f64_gpu) on
                     the same fp32 heads, differentiated by float64 autograd; the fp32 assignment equals the float64
                     one.  Bounds, U = 2^-24:
                       objectness channel  8 U scale (|1 - t| + lw (s + |s - 1|)): expf, 1 + e, the division, s - 1,
                                           the sum, the scale and its rounding (loss.cu obj_bce_bwd_kernel)
                       matched cells       (16 + rows on the cell) U sum over the rows of M_row: 16 fp32 roundings in
                                           torch's autograd of one row term, one fmaf per row in the scatter.  M_row:
                                           class cls / (cnt nc) (s + t); xy reg / (2 cnt) (s + |t ng|) s (the fp32
                                           target offset t ng - floor(t ng) carries U of the cell index; 1 - s in the
                                           sigmoid backward carries U s); wh giou reg / cnt e^x a (|d iou / dw| terms
                                           taken apart); theta 2 reg / cnt (|atan x| + |a| + |t|) / (1 + x^2)
                       every other element exactly 0, in the kernel's output and in float64
                       loss value          lobj 8 U sum M_l + (cells) 2^-53 sum M_l + U |lobj| (fp32 terms, the double
                                           sums of ordered_sum_add_kernel, the float conversion); lcls / lreg (16 + n + 8)
                                           U sum M over their n row terms (a worst-case sequential fp32 sum)
  coverage           test_covers_every_launch ties every entry of sched.ops and every forward block to a check.
Detect forward (eval, CUDA-graph replay) of the same two models and of nc = 23 at batch 1 x 320 x 416 (2088-filter
heads, which training refuses at plan build): every conv launch with checked_step's eval-forward checks, the decode
(direct path, no = 21 / 28 / 29) within 2^-20 M of f64_refs.decode_ref, and detect_postprocess_classes on the io
equal bit for bit to the per-image per-class pipeline (check_equals_per_class_pipeline).  The bound self-test puts five bugs in.

Measured on an H100 80GB HBM3 (132 SMs, power limit 700 W, 1980 MHz max SM clock), seeds as below; worst ratio per
kernel (block), nc = 15 / nc = 22:
  heads, training    fp32 z 0.185 (105) / 0.158 (105); wgrad 0.141 (81) / 0.142 (81); dgrad 0.987 (105) / 0.985 (105);
                     bias sums 0.094 (81) / 0.130 (81); dz bit for bit, padding and halo zero
  other blocks       conv z, bn_act_fwd, bn_act_bwd, dgrad 0.996 (half a bf16 ulp at the bottom of a binade, see
                     test_train_step_f64_gpu); wgrad 0.684 (104) / 0.615 (92); d beta / d gamma <= 0.128; d slope 0.003
  head cotangent     objectness 0.157 / 0.204; class columns 0.185 / 0.181; regression columns 0.365 / 0.622 (81);
                     every other element 0; up to 2 rows per cell, 10 / 6 matched rows outside the map
  loss value         lobj 0.016 / 0.009; lcls, lreg and the total < 0.001 (their sequential-sum bounds are loose; a
                     wrong class column moves lcls by O(1))
  detect             heads 0.133 / 0.139 / 0.110 (nc = 23) at layer 105; other convs <= 0.996; decode <= 0.197;
                     post-processing bit for bit (4000 / 6000 / 2000 selected at cap 2000)
Bugs put in, worst |err| / bound: the one-hot shifted by one column 7.7e6; the scatter dropping row columns >= 16 9.9e5;
the head bias without its last 8-channel group 8.8e5; a nonzero padding channel of the head dz fails its bitwise check;
the decode reading class scores with the nc = 1 row stride 4.6e14.  No kernel needed a change.  Whole file: 19 s."""
import time

import pytest
import torch

from builders import check_equals_per_class_pipeline, pkg
from checked_step import (Run, Step, check_block_bwd, check_buffers, check_conv, check_first, check_s2d_step, map_plan,
                          run_step)
from f64_refs import bad_entries, decode_ref, halo_zero, head_bias_chain, sum_check
from helpers import init_darknet_weights
from loss_f64 import cot_check, fused_loss, loss64, loss_checks, make_targets, record_head_grads

pytestmark = pytest.mark.gpu

MODELS = {"nc15": (15, 2, 608, 608), "nc22": (22, 3, 320, 416)}
NC_EVAL_ONLY = (23, 1, 320, 416)          # 2088-channel heads: eval runs them, training refuses them at plan build
HYP = {"giou": 0.1, "cls": 27.76, "cls_pw": 1.0, "obj": 20.35, "obj_pw": 1.0, "iou_t": 0.5, "ang_t": 3.1415926 / 12,
       "reg": 1.0, "context_factor": 1.0}
CONF, NMS_T, CAP = 0.5, 0.5, 2000


def make_model(nc, h, w, seed):
    from rotate_yolov3_b200 import cfgs
    m = pkg().Darknet(cfgs.yolov3_cfg(width=w, height=h, classes=nc), {"context_factor": 1.0}, arc="default")
    m.hyp, m.nc = HYP, nc                  # train.py sets both before compute_loss
    return init_darknet_weights(m, seed=seed)


# ---------------------------------------------------------------------------------------------------------------
def mc_step(name, seed=41):
    nc, batch, h, w = MODELS[name]
    dev = torch.device("cuda")
    t0 = time.time()
    model = make_model(nc, h, w, seed).to(dev).train()
    st = Step(model, torch.rand(batch, 3, h, w, generator=torch.Generator().manual_seed(seed + 1)).to(dev))
    st.nc = nc
    st.targets = make_targets(model, nc, batch, h, w, seed + 2)
    st.cot = {}

    def block_check(st, blk, orig):
        r = check_block_bwd(st, blk, orig)
        if blk.is_head and "pad" not in st.stash:
            st.stash["pad"] = dict(dz=blk.dz.clone(), cout=blk.cout)
        return r
    run_step(st, loss=lambda st, ps: fused_loss(st, ps, HYP), head_grads=record_head_grads, block_check=block_check)
    # the first head's bias sum, kept for the bound self-test
    hd = next(b for b in st.plan.blocks if b.is_head)
    g = st.g_nhwc[hd.i].double()
    st.stash["bias"] = dict(got=st.plan.garena[hd.gb_off:hd.gb_off + hd.cout].clone(), want=g.sum((0, 1, 2)),
                            mag=g.abs().sum((0, 1, 2)), chain=head_bias_chain(st.batch, hd.oh, hd.ow))
    loss_checks(st)
    st.t_total = time.time() - t0
    _print_table(st)
    return st


def _print_table(st):
    tag = "[mc %s]" % ("nc%d %dx%dx%d" % (st.nc, st.batch, st.h, st.w))
    print("\n%s whole step with checks %.1f s" % (tag, st.t_total))
    worst = {}
    for blk in st.plan.blocks:
        f, b = st.fwd.get(blk.i, {}), st.bwd.get(blk.i, {})
        kind = "head" if blk.is_head else ("s2d" if blk.s2d else "k%d" % blk.k)
        cols = ["%-4s" % kind, "%4d" % blk.cout, "%2dx%-2d" % (blk.oh, blk.ow)]
        for src, t_ in ((f, "f:"), (b, "b:")):
            for key in ("z", "z_bias", "mean", "invstd", "y", "y_bias", "dz", "dz_bias", "dbeta", "dgamma", "dslope",
                        "wgrad", "dgrad", "dgrad_bias", "dbias"):
                if isinstance(src.get(key), float):
                    cols.append("%s %.3f" % (key, src[key]))
                    k = ("head " if blk.is_head else "") + t_ + key
                    if not worst.get(k, (-1.0,))[0] >= src[key]:
                        worst[k] = (src[key], blk.i)
            if "error" in src:
                cols.append("ERROR")
        if blk.is_head or blk.i in (0, 1):
            print("%s %3d " % (tag, blk.i) + "  ".join(cols))
    print("%s worst: %s" % (tag, ", ".join("%s %.3f (%d)" % (k, v, i) for k, (v, i) in sorted(worst.items()))))
    print("%s loss value / bound: %s" % (tag, ", ".join("%s %.3f" % kv for kv in st.loss_r.items())))
    for i, r in st.cot_r.items():
        print("%s head %d cotangent / bound: obj %.3f  class columns %.3f  regression columns %.3f  zeros %s  "
              "(%d matched cells)" % (tag, i, r["obj"], r["cls"], r["reg"], r["zero"], r["matched_cells"]))
    print("%s rows: up to %d per cell, %d matched rows outside the map" % (tag, st.max_rows_per_cell, st.border_rows))


# ---------------------------------------------------------------------------------------------------------------
def run_detect(nc, batch, h, w, seed=43):
    """the eval forward replayed as a CUDA graph, every conv launch and the decode against float64, the class-aware
    post-processing against the per-image per-class pipeline"""
    dev = torch.device("cuda")
    t0 = time.time()
    model = make_model(nc, h, w, seed).to(dev).eval()
    model.use_cuda_graph = True
    xa, xb = (torch.rand(batch, 3, h, w, generator=torch.Generator().manual_seed(seed + s)).to(dev) for s in (1, 2))
    st = Run("nc%d" % nc, model)
    st.nc = nc
    with torch.no_grad():
        io_a = model(xa)[0].clone()
        st.io, _ = model(xb)
    torch.cuda.synchronize()
    st.replayed = model._graph is not None and model.replayed_kernels == 2 * model._graph_kernels
    st.io_changed = not torch.equal(io_a, st.io)
    st.plan, st.x, st.stash = model._plan, model._x_static, None
    map_plan(st)
    convs = sorted(st.conv_of)
    st.res = {0: check_first(st)}
    for i in convs[1:]:
        st.res[i] = check_conv(st, i)
    st.s2d = {i: check_s2d_step(st, i) for i in st.s2d_of}
    st.buffers_ok, _ = check_buffers(st)
    # decode: io within 2^-20 M of the float64 decode of the actual head buffers (direct path: nc + 6 > 8)
    st.decode, off = [], 0
    for (li, p), yi in zip(st.plan["heads"], model.yolo_layers):
        layer = model.module_list[yi]
        want, mag = decode_ref(p, layer.anchors.float(), float(layer.stride), 1.0, nc)
        got = st.io[:, off:off + want.shape[1]]
        st.decode.append(decode_ratio(got, want, mag))
        if off == 0:
            st.dec = dict(p=p.clone(), got=got.clone(), anchors=layer.anchors.float(), stride=float(layer.stride))
        off += want.shape[1]
        del want, mag
    st.io_rows = off == st.io.shape[1]
    res, st.kept = check_equals_per_class_pipeline(st.io, CONF, NMS_T, CAP)
    st.selected = int(res["counts"].sum())
    st.t_total = time.time() - t0
    tag = "[mc detect nc%d %dx%dx%d]" % (nc, batch, h, w)
    heads = [i for i in convs if st.res[i].get("kind") == "head"]
    print("\n%s %.1f s; heads %s; worst conv %.3f, bias %.3f; decode %s; %d selected, %d kept" % (
        tag, st.t_total, ", ".join("%d (cout %d): %.3f" % (i, st.res[i]["cout"], st.res[i]["max"]) for i in heads),
        max(r["max"] for i, r in st.res.items() if i), max(r.get("bias", 0.0) for r in st.res.values()),
        ", ".join("%.3f" % v for v in st.decode), st.selected, st.kept))
    return st


def decode_ratio(got, want, mag):
    ratio = (got.double() - want).abs() / (mag * 2.0 ** -20)
    ratio = torch.where(got.double() == want, torch.zeros_like(ratio), ratio)
    return float(ratio.max()) if not bool(ratio.isnan().any()) else float("nan")


_CACHE = {}


def _get(kind, name):
    key = (kind, name)
    if key not in _CACHE:
        if kind == "step":
            _CACHE[key] = mc_step(name)
        else:
            _CACHE[key] = run_detect(*(MODELS[name] if name in MODELS else NC_EVAL_ONLY))
    return _CACHE[key]


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(MODELS))
def test_covers_every_launch(name):
    st, dt = _get("step", name), _get("detect", name)
    nc, batch, h, w = MODELS[name]
    plan = st.plan
    heads = [b for b in plan.blocks if b.is_head]
    assert [b.cout for b in heads] == [72 * (nc + 6)] * 3 and {b.cout_pad for b in heads} == {1536 if nc == 15 else 2048}
    assert [(b.oh, b.ow) for b in heads] == [(h // s, w // s) for s in (32, 16, 8)]
    assert [b.cin for b in heads] == [1024, 512, 256]
    assert set(st.fwd) == {b.i for b in plan.blocks} and len(plan.blocks) == 75
    missing = []
    for kind, i, flag in plan.sched.ops(plan):
        r = st.bwd.get(i, {})
        ok = {"head": "dz_bits" in r and "dbias" in r, "bnact": "dz" in r, "wgrad": "wgrad" in r,
              "dgrad": "dgrad" in r}.get(kind, False)
        if not ok:
            missing.append((kind, i, flag))
    assert not missing, missing
    ops = plan.sched.ops(plan)
    assert {k for k, _, _ in ops} == {"head", "bnact", "wgrad", "dgrad"}
    for b in heads:
        assert {"dz_bits", "dz_pad_zero", "dbias", "wgrad", "dgrad", "gw_bits"} <= set(st.bwd[b.i]), b.i
    assert set(st.cot_r) == {b.i for b in heads}
    # detect: every conv of the graph, the three heads at this width, the decode on its direct path
    assert sorted(dt.res) == sorted(dt.conv_of) and len(dt.res) == 75
    assert [r["cout"] for r in dt.res.values() if r.get("kind") == "head"] == [72 * (nc + 6)] * 3
    assert nc + 6 > 8 and len(dt.decode) == 3 and dt.io_rows and dt.io.shape[-1] == nc + 6
    assert dt.replayed and dt.io_changed


@pytest.mark.parametrize("name", list(MODELS))
def test_training_step_kernels_vs_float64(name):
    st = _get("step", name)
    assert st.fwd_halo
    assert st.im2col == dict(bits=True, pad_zero=True, halo=True), st.im2col
    assert all(p[2] for p in st.packs), [p[:2] for p in st.packs if not p[2]]
    bad = bad_entries(st.fwd) + bad_entries(st.bwd)
    assert not bad, bad
    for i, r in st.bwd.items():
        if "near_zero_u" in r:
            assert r["near_zero_u"] <= max(64, r["n_elems"] // 100000), (i, r["near_zero_u"])


@pytest.mark.parametrize("name", list(MODELS))
def test_loss_and_head_cotangent_vs_float64(name):
    st = _get("step", name)
    assert st.masks_equal
    # the targets reach what they are there for: chained rows on a cell, rows outside the map, classes 0 and nc - 1
    assert st.max_rows_per_cell >= 2 and st.border_rows > 0
    cls = st.targets[:, 1].long()
    assert int(cls.min()) == 0 and int(cls.max()) == st.nc - 1
    bad = {k: v for k, v in st.loss_r.items() if not v <= 1.0}
    assert not bad, (bad, st.loss_r)
    for i, r in st.cot_r.items():
        assert r["zero"] and r["matched_cells"] > 0, (i, r)
        assert r["obj"] <= 1.0 and r["cls"] <= 1.0 and r["reg"] <= 1.0, (i, r)


@pytest.mark.parametrize("name", list(MODELS) + ["nc23"])
def test_detect_forward_vs_float64(name):
    """every conv launch (the three fp32 heads at 72 (nc + 6) filters among them), the decode on the direct path and
    the class-aware post-processing; nc23: 2088-channel heads, which training refuses, run in eval"""
    dt = _get("detect", name)
    bad = [(i, k, r[k]) for i, r in dt.res.items() for k in ("max", "bias") if k in r and not r[k] <= 1.0]
    bad += [(i, k) for i, r in dt.res.items() for k in ("w_bits", "b_bits", "slope", "up_copies") if k in r and not r[k]]
    assert not bad, bad
    assert dt.buffers_ok and all(v["bits"] and v["pad_zero"] for v in dt.s2d.values())
    assert all(v <= 1.0 for v in dt.decode), dt.decode
    assert dt.selected > 0 and dt.kept > 0
    if name == "nc23":
        assert [r["cout"] for r in dt.res.values() if r.get("kind") == "head"] == [2088] * 3


def test_training_refuses_2088_channel_heads_before_any_launch():
    nc, batch, h, w = NC_EVAL_ONLY
    model = make_model(nc, h, w, 5).cuda().train()
    x = torch.rand(batch, 3, h, w, device="cuda")
    lib = pkg()._lib.lib
    torch.cuda.synchronize()
    c0 = lib.ryolo_launch_count()
    with pytest.raises(NotImplementedError, match="limited to 2048 channels"):
        model(x)
    assert lib.ryolo_launch_count() == c0
    assert model._tplan is None


def test_bounds_reject_plausible_bugs():
    """each bug, put into a stored tensor or a reference, fails the check that guards it"""
    st, dt = _get("step", "nc22"), _get("detect", "nc22")
    out = {}
    c = st.stash["cot"]
    ok = cot_check(c["got"], c["want"], c["m"], c["ncell"])
    assert ok["cls"] <= 1.0 and ok["reg"] <= 1.0 and ok["obj"] <= 1.0 and ok["zero"]
    # the class one-hot shifted by one column (the float64 loss with tcls + 1)
    p64 = [p.double().requires_grad_(True) for p in c["p32"]]
    comps, _ = loss64(p64, st.targets.double(), st.model, HYP, shift_cls=1)
    sum(comps).sum().backward()
    out["one-hot shifted by one column"] = cot_check(c["got"], p64[-1].grad, c["m"], c["ncell"])["cls"]
    # the scatter dropping the row columns >= 16: those columns of the matched cells keep the objectness kernel's 0
    got = c["got"].clone()
    got[..., 16:][c["ncell"] > 0] = 0.0
    out["scatter drops columns >= 16"] = cot_check(got, c["want"], c["m"], c["ncell"])["cls"]
    # the head bias gradient missing its last 8-channel group
    b = st.stash["bias"]
    assert sum_check(b["got"], b["want"], b["chain"], b["mag"]) <= 1.0
    gb = b["got"].clone()
    gb[-8:] = 0.0
    out["head bias without its last 8 channels"] = sum_check(gb, b["want"], b["chain"], b["mag"])
    # a nonzero padding channel of the head dz (2016 = 63 * 32 has none: the 1512-channel heads, zcs 1536)
    d = _get("step", "nc15").stash["pad"]
    dz = d["dz"].clone()
    assert bool((dz[..., d["cout"]:] == 0).all()) and halo_zero(dz)
    dz[1, 3, 4, d["cout"] + 5] = 1.0
    out["nonzero padding channel of the head dz"] = 0.0 if bool((dz[..., d["cout"]:] == 0).all()) else 2.0
    # decode reading the class scores with the nc = 1 row stride (anchor a's column k at channel 7 a + k)
    e = dt.dec
    p = e["p"]
    bs, ch, ny, nx = p.shape
    no = dt.nc + 6
    na = ch // no
    assert decode_ratio(e["got"], *decode_ref(p, e["anchors"], e["stride"], 1.0, dt.nc)) <= 1.0
    pb = p.view(bs, na, no, ny, nx).clone()
    for k in range(6, no):
        src = torch.arange(na, device=p.device) * 7 + k
        pb[:, :, k] = p[:, src.clamp(max=ch - 1)]
    out["decode with the nc = 1 row stride"] = decode_ratio(e["got"], *decode_ref(pb.view(bs, ch, ny, nx), e["anchors"],
                                                                                     e["stride"], 1.0, dt.nc))
    print("\n[bite] " + ", ".join("%s %.3g" % kv for kv in out.items()))
    bad = {k: v for k, v in out.items() if not v >= 2.0}
    assert not bad, bad
