"""Every kernel launch of the bf16 detect forward at 608 x 608, batch 32, against float64 of the inputs it actually
received.

The forward is the one bench.py's detect workload times: Darknet-53 / YOLOv3 (cfgs.yolov3_cfg(): 75 convs, 504-filter
heads, 768- and 384-channel concat buffers) with init_darknet_weights(seed=1) (randomised BN statistics and PReLU
slopes), in eval mode and replayed as one CUDA graph.  It is called on x_a, then on a different x_b; after the second
call every buffer of model._plan holds what the graph replay wrote for x_b.  Each step of the plan is mapped back to the
tensors its pointers address (the image, the first layer's space-to-depth buffer, a ryolo_space_to_depth copy, a view,
a concat slice, the shortcut source, the fp32 head), so each launch is checked post hoc on its own inputs; no upstream
layer is recomputed.  The graph's wiring is checked on the way: the input of conv i is the output of layer i - 1, the
residual is the layer the [shortcut] names, the producers of a concat buffer sit at their route offsets.

  weight pack    every packed operand == torch's bf16(w * scale) (L.s2d_weight for the stride-2 layers), zero padded,
                 bit for bit; the kernel's bias buffer == _folded's bias; the first layer's fp32 operand == w * scale
  BN folding     _folded's fp32 scale and bias against a float64 restatement of utils/torch_utils.py:45-69, bounded by
                 their fp32 roundings: scale = gamma / sqrt(var + eps): eps to fp32 and the add (2 U of var + eps, halved
                 by the square root), the square root, the division: 3 U |scale|; bias = beta - mean * scale: the 3 U of
                 the scale carried by the product, the multiply, the subtraction: U (4 |mean * scale| + |bias|)
  first layer    conv_first_s2d_fwd: float64 of the fp32 image with bf16(wf), + bias, PReLU, rearranged by a plain reshape
                 into the space-to-depth layout; e = 4 * 2^-23 A + 2^-16 A (four k16 updates, the hi + lo image)
  conv           all 74 conv_bn_act_fwd launches with the packed operand as the GEMM matrix: want = act(S + bias) + res,
                 E = n * 2^-23 A, n = taps * cin_pad / 16, T = U (2 (|S| + |bias|) + |act| + |res|) (bias add, PReLU
                 multiply, residual add); bf16 outputs  |got - want| <= 2^-8 (|want| + E + T) + E + T  and
                 |mean((got - want) sign(want))| <= 2^-12 rms(want); up-sampled outputs: the four replicas bitwise equal,
                 each within the bound; fp32 heads  |got - want| <= E + 2^-24 |want|
  buffers        every halo zero after all writes; the channels of a buffer no producer owns are zero; a concat
                 producer that wrote into its neighbour's channels fails the neighbour's check (the checks read the
                 final state, and a clobbered earlier producer is also caught by the s2d copy made from it)
  s2d            ryolo_space_to_depth bit for bit against a plain reshape
  decode         io within 2^-20 M of f64_refs.decode_ref on the actual head buffers
  whole forward  (bench shape) the replay's io and heads == an eager forward on x_b, bit for bit; each of the 32 images
                 == a batch-1 forward of that image, bit for bit (the tile width depends on cout only and there is no
                 split-K, so no accumulation order depends on the batch: the cheap exact check of the large offsets)

A second parametrisation runs checks 1-5 at batch 3 on H x W = 352 x 608 (the letterbox of a 16:9 frame: grids
11 x 19, 22 x 38, 44 x 76; oh != ow in the head staging and the up-sampling).  A last test puts nine plausible bugs
into stored tensors or references and requires each check to fail.

Measured on an H100 80GB HBM3 (132 SMs, power limit 400 W, 1980 MHz max SM clock), seeds as below, two runs bitwise
identical.  `pytest -s` prints one line per launch (worst |err| / bound, the no-bias ratio and the folding ratio); the
worst ratio per kernel over the launches (layer in parentheses), batch 32 at 608^2 / batch 3 at 352 x 608:
  conv_first_s2d_fwd        0.992 / 0.990 (0), bias 0.007 / 0.007
  conv_bn_act_fwd, bf16     0.996 / 0.996 (2), bias 0.072 (67) / 0.052 (70); the s2d layers <= 0.993 (1)
  up-sampled (84, 96)       0.993 / 0.990 (96), bias 0.009 / 0.028; replicas bitwise equal
  fp32 heads                0.115 / 0.101 (105)
  BN folding                0.947 (90); packs, bias buffers and slopes bit for bit
  decode                    0.203 / 0.191;  ryolo_space_to_depth bit for bit;  halos zero
  whole forward             replay == eager, and each image == its batch-1 forward, bit for bit
The bf16 ratios just under 1 are half an ulp at the bottom of a binade: every bf16 output is the correctly rounded
float64 result up to E + T.  Bugs put in (test_bounds_reject_plausible_bugs), worst |err| / bound: an up-sample
replica left zero 255 (and the replicas differ); a concat producer 32 channels off 1.7e5; the shortcut from the
previous block's source 4845; the neighbouring layer's PReLU slope 230; BN folding without eps 45 on the layer where it
shows least (it fails on all 72 BN layers); the first layer's image with its hi half only 90; round-toward-zero conv
output 1.9 (bias 9.0); the bias missing on a head's second 256-filter tile 5239; image 31 one pixel row off 9779.
Whole file: 12 s (4.1 s for the batch-32 forward, its checks and the 33 whole-forward runs)."""
import time

import pytest
import torch

from checked_step import (Acc, Run, check_buffers, check_conv, check_first, check_s2d_step, conv_want, first_check,
                          fold_ratio, map_plan, slope)
from f64_refs import BF16, bf16_check, bitwise, decode_ref, f32_check, interior, passed, rtz_bf16, yolov3_heads
from helpers import init_darknet_weights

pytestmark = pytest.mark.gpu

SHAPES = {"bench": (32, 608, 608), "letterbox": (3, 352, 608)}
X_SEEDS = (0, 5)           # x_a (bench.py's rank-0 image) and x_b


def check_decode(st):
    """io against float64 _decode_ref of the actual head buffers"""
    model = st.model
    heads = yolov3_heads(1)
    off = 0
    worst = 0.0
    for (li, p), (anchors, _, stride), yi in zip(st.plan["heads"], heads, model.yolo_layers):
        layer = model.module_list[yi]
        assert torch.equal(layer.anchors.float(), anchors) and layer.stride == stride
        want, mag = decode_ref(p, anchors, stride, 1.0, 1)
        rows = want.shape[1]
        got = st.io[:, off:off + rows].double()
        ratio = (got - want).abs() / (mag * 2.0 ** -20)
        ratio = torch.where(got == want, torch.zeros_like(ratio), ratio)
        worst = max(worst, float(ratio.max())) if not bool(ratio.isnan().any()) else float("nan")
        off += rows
        del want, mag, got, ratio
    assert off == st.io.shape[1]
    return worst


def run_forward(name, stash):
    """bench.py's wl_detect model and graph replay at the given shape, then every check on the plan's buffers"""
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import cfgs
    batch, h, w = SHAPES[name]
    t0 = time.time()
    dev = torch.device("cuda")
    model = pkg.Darknet(cfgs.yolov3_cfg(), {"context_factor": 1.0}, arc="default")
    init_darknet_weights(model, seed=1)
    model = model.cuda().eval()
    model.use_cuda_graph = True
    xa, xb = (torch.rand(batch, 3, h, w, generator=torch.Generator().manual_seed(s)).to(dev) for s in X_SEEDS)
    st = Run(name, model)
    with torch.no_grad():
        io_a = model(xa)[0].clone()
        st.io, _ = model(xb)
    torch.cuda.synchronize()
    st.t_fwd = time.time() - t0
    st.replayed = model._graph is not None and model.replayed_kernels == 2 * model._graph_kernels
    st.io_changed = not torch.equal(io_a, st.io)
    del io_a
    st.plan = model._plan
    st.x = model._x_static
    st.x_is_xb = torch.equal(st.x, xb)
    st.stash = {} if stash else None
    map_plan(st)
    convs = sorted(st.conv_of)
    if stash:
        res = [i for i in convs if i > 0 and st.plan["steps"][st.conv_of[i]][1]["desc"].has_residual]
        ups = [i for i in convs if i > 0 and st.plan["steps"][st.conv_of[i]][1]["desc"].upsample2x]
        hds = [li for li, _ in st.plan["heads"]]
        st.picks = dict(res=res[-1], res_prev=res[-2], up=ups[0], head=hds[0])
        st.keep = {res[-1], ups[0], hds[0]}
    st.res = {}
    st.res[0] = check_first(st)
    for i in convs[1:]:
        st.res[i] = check_conv(st, i)
    st.s2d = {i: check_s2d_step(st, i) for i in st.s2d_of}
    st.buffers_ok, st.concat_widths = check_buffers(st)
    st.decode = check_decode(st)
    torch.cuda.synchronize()
    st.t_checks = time.time() - t0
    if name == "bench":
        whole_forward(st, xb)
    st.t_total = time.time() - t0
    _print_table(st)
    return st


def whole_forward(st, xb):
    """the replay against an eager forward, and each image against a batch-1 forward, bit for bit"""
    model = st.model
    io_g = st.io.clone()
    heads_g = [p.clone() for _, p in st.plan["heads"]]
    model.use_cuda_graph = False
    with torch.no_grad():
        io_e, _ = model(xb)
    torch.cuda.synchronize()
    st.eager_io = torch.equal(io_e.view(torch.int32), io_g.view(torch.int32))
    st.eager_heads = all(torch.equal(p.view(torch.int32), g.view(torch.int32))
                         for (_, p), g in zip(st.plan["heads"], heads_g))
    del io_e
    bad = []
    with torch.no_grad():
        for b in range(xb.shape[0]):
            io1, _ = model(xb[b:b + 1])
            same = torch.equal(io1[0].view(torch.int32), io_g[b].view(torch.int32))
            same = same and all(torch.equal(p[0].view(torch.int32), g[b].view(torch.int32))
                                for (_, p), g in zip(model._plan["heads"], heads_g))
            if not same:
                bad.append(b)
    torch.cuda.synchronize()
    st.batch1_bad = bad
    st.io = io_g


def _print_table(st):
    tag = "[detect %s]" % st.name
    print("\n%s forward %.1f s, per-kernel checks done at %.1f s, total %.1f s"
          % (tag, st.t_fwd, st.t_checks, st.t_total))
    for i in sorted(st.res):
        r = st.res[i]
        kind = "first" if i == 0 else r["kind"]
        cols = ["%3d %-5s" % (i, kind)]
        if i:
            cols.append("%4d %-7s" % (r["cout"], r["grid"]))
        cols.append("max %.3f" % r["max"])
        if "bias" in r:
            cols.append("bias %.3f" % r["bias"])
        if "fold" in r:
            cols.append("fold %.3f" % r["fold"])
        for key in ("w_bits", "b_bits", "slope", "up_copies"):
            if key in r and not r[key]:
                cols.append("%s FAILED" % key)
        print(tag + " " + "  ".join(cols))
    print("%s decode worst |err| / (2^-20 M) %.3f; s2d copies bitwise: %s" %
          (tag, st.decode, all(v["bits"] for v in st.s2d.values())))


@pytest.fixture(scope="module")
def bench():
    return run_forward("bench", stash=True)


@pytest.fixture(scope="module")
def letterbox():
    return run_forward("letterbox", stash=False)


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SHAPES))
def test_covers_the_whole_forward(request, name):
    st = request.getfixturevalue(name)
    kinds = [k for k, _ in st.plan["steps"]]
    assert set(kinds) == {"first", "conv", "s2d"}, set(kinds)
    assert "se" not in kinds and "maxpool" not in kinds          # neither block is in this graph
    assert kinds.count("first") == 1 and kinds.count("conv") == 74 and kinds.count("s2d") == 4
    assert sorted(st.res) == sorted(st.conv_of) and len(st.res) == 75
    assert sorted(st.s2d) == [5, 12, 37, 62] and 1 not in st.s2d_of
    assert sum(r.get("kind") == "head" for r in st.res.values()) == 3
    assert sum("up_copies" in r for r in st.res.values()) == 2
    assert st.concat_widths == [384, 768]
    assert st.replayed and st.io_changed and st.x_is_xb


@pytest.mark.parametrize("name", list(SHAPES))
def test_weight_pack_and_bn_folding(request, name):
    st = request.getfixturevalue(name)
    bad = [(i, k) for i, r in st.res.items() for k in ("w_bits", "b_bits", "slope") if k in r and not r[k]]
    assert not bad, bad
    folds = {i: r["fold"] for i, r in st.res.items() if "fold" in r}
    assert len(folds) == 72
    worst = max(folds.values())
    print("[detect %s] BN folding: worst ratio %.3f (layer %d)" % (name, worst, max(folds, key=folds.get)))
    assert worst <= 1.0, worst


@pytest.mark.parametrize("name", list(SHAPES))
def test_first_layer_vs_float64(request, name):
    st = request.getfixturevalue(name)
    r = st.res[0]
    assert r["max"] <= 1.0 and r["bias"] <= 1.0 and r["xs_pad_zero"], r


@pytest.mark.parametrize("name", list(SHAPES))
def test_conv_launches_vs_float64(request, name):
    st = request.getfixturevalue(name)
    bad = []
    for i, r in st.res.items():
        if i == 0:
            continue
        for k in ("max", "bias"):
            if k in r and not r[k] <= 1.0:                     # NaN fails
                bad.append((i, k, r[k]))
        if "up_copies" in r and not r["up_copies"]:
            bad.append((i, "up_copies"))
    assert not bad, bad
    assert st.buffers_ok


@pytest.mark.parametrize("name", list(SHAPES))
def test_space_to_depth_and_decode(request, name):
    st = request.getfixturevalue(name)
    assert all(v["bits"] and v["pad_zero"] for v in st.s2d.values()), st.s2d
    assert st.decode <= 1.0, st.decode


def test_whole_forward_bitwise(bench):
    assert bench.eager_io and bench.eager_heads
    assert not bench.batch1_bad, bench.batch1_bad


def test_bounds_reject_plausible_bugs(bench):
    """each check, applied to a stored tensor or a reference with one plausible bug put in, fails"""
    st = bench
    pk = st.picks
    found = {}

    def conv_result(i, got=None, res=None, slope=None, want_fn=None):
        d = st.stash[i]
        want, t = conv_want(d["s"], d["bias"], d["slope"] if slope is None else slope,
                            d["res"] if res is None else res)
        if want_fn is not None:
            want = want_fn(want)
        y = d["out"].interior() if got is None else got
        if d["up"]:
            y = y[:, ::2, ::2]
        acc = Acc()
        acc.add(y, want, d["n"] * 2.0 ** -23 * d["mag"], t)
        return acc.result()

    # the stored checks pass before any bug is put in
    for i in (pk["res"], pk["up"]):
        assert passed(conv_result(i)), i
    # one up-sample replica left zero
    u = st.stash[pk["up"]]
    y = u["out"].interior().clone()
    y[:, 1::2, 1::2] = 0
    y0 = y[:, ::2, ::2]
    copies = float(all(bitwise(y[:, ry::2, rx::2], y0) for ry in range(2) for rx in range(2)))
    # the bound on the zeroed replica (1, 1) itself
    found["up_replica_zero"] = {"replicas_equal": copies, "max": conv_result(pk["up"], got=y[:, 1:, 1:])["max"]}
    # a concat producer shifted by 32 channels
    v = u["out"]
    assert v.off + 32 + v.c <= v.buf.shape[-1]
    found["concat_shift_32"] = conv_result(pk["up"], got=interior(v.buf, v.off + 32, v.c))
    # the shortcut taken from the wrong layer: the one the previous shortcut adds (from = -6 instead of -3)
    prev = st.stash[pk["res"]]
    j = pk["res_prev"] + 1
    wrong_v = st.outs[j + int(st.model.module_defs[j]["from"])]
    assert wrong_v.ptr != st.plan["steps"][st.conv_of[pk["res"]]][1]["r"]
    wrong = wrong_v.interior()
    assert wrong.shape == prev["res"].shape
    found["shortcut_wrong_layer"] = conv_result(pk["res"], res=wrong)
    # the neighbouring layer's PReLU slope
    s_next = slope(st.model, pk["res"] - 1)
    assert s_next != prev["slope"]
    found["neighbour_slope"] = conv_result(pk["res"], slope=s_next)
    # BN folding without eps, on every BN layer: the worst and the count
    folds = {i: fold_ratio(st.model, i, drop_eps=True) for i in st.res if "fold" in st.res[i]}
    found["fold_without_eps"] = {"least": min(folds.values())}
    n_eps = sum(f > 1.0 for f in folds.values())
    # the first layer's image with only its hi half
    f = st.stash["first"]
    found["first_hi_only"] = first_check(f["got"], f["x"].to(BF16).float(), f["w"], f["b"], f["slope"]).result()
    assert passed(first_check(f["got"], f["x"], f["w"], f["b"], f["slope"]).result())
    # round-toward-zero conv output
    d = st.stash[pk["res"]]
    want, t = conv_want(d["s"], d["bias"], d["slope"], d["res"])
    v32 = want.float()
    e = d["n"] * 2.0 ** -23 * d["mag"]
    assert passed(bf16_check(v32.to(BF16), want, e, t))
    found["rtz_output"] = bf16_check(rtz_bf16(v32), want, e, t)
    del want, t, v32, e
    # the bias missing on the second 256-filter tile of a head
    h = st.stash[pk["head"]]
    got = h["out"].permute(0, 2, 3, 1).clone()
    assert f32_check(got, h["s"] + h["bias"], h["n"] * 2.0 ** -23 * h["mag"])["max"] <= 1.0
    got[..., 256:] -= h["bias"][256:].float()
    found["head_bias_tile2"] = f32_check(got, h["s"] + h["bias"], h["n"] * 2.0 ** -23 * h["mag"])
    # image 31 shifted by one pixel row
    y = d["out"].interior().clone()
    y[31] = torch.roll(y[31], 1, 0)
    found["image31_row_shift"] = conv_result(pk["res"], got=y)
    for name, r in found.items():
        print("[bite] %-22s %s" % (name, {k: round(v, 3) for k, v in r.items()}))
    print("[bite] BN folding without eps fails on %d of %d BN layers" % (n_eps, len(folds)))
    assert found["up_replica_zero"]["replicas_equal"] == 0.0 and found["up_replica_zero"]["max"] > 1.0
    assert found["rtz_output"]["bias"] > 1.0, found["rtz_output"]
    for name in ("concat_shift_32", "shortcut_wrong_layer", "neighbour_slope", "fold_without_eps", "first_hi_only",
                 "head_bias_tile2", "image31_row_shift"):
        assert not passed(found[name]), (name, found[name])
