"""Every kernel launch of one bf16 training step at 608 x 608 against float64 of the inputs it actually received.

The step is the one bench.py measures: Darknet-53 / YOLOv3 (cfgs.yolov3_cfg(): 75 convs, 504-filter heads, 768- and
384-channel concat buffers) run by train_path.TrainPlan, here at batch 2 so that GEMM tiles straddle the image boundary of
the flat pixel index.  A dense random cotangent G per head (loss = sum (p * G)) reaches all 504 head channels.

Forward: after model(x) every buffer a forward kernel wrote is still there, so each launch is checked post hoc on the
plan's own input buffers (the im2col columns, a view, a concat slice, the space-to-depth copy): im2col bit for bit, the
multi-tensor weight pack bit for bit against ryolo_conv_pack_weights_ex, the raw conv z, the fp32 heads, the batch
statistics (two-pass float64) with the running-statistics update, and bn_act_fwd / bn_act_fwd_s2d.  Backward:
plan._backward_block is wrapped (instance attribute) so that what each block overwrites is snapshotted, the production
code runs unchanged, and its outputs are checked right after: bn_act_bwd (dz, d beta, d gamma, d slope, the shortcut
gradient), the split-K weight gradient and its gather, the dgrad (mode-1 operands; mode-3 operands with ksize -2 and the
depth_to_space pass) including the accumulate flag and the channels outside the gradient view.  No graph sits between a
kernel and its reference, so no PReLU kink crossing blurs a check and the bounds are the single-kernel ones:

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
                 part and the 8 parts (f64_refs.bn_chain mirrors mk_pieces).  d slope: a thread adds all 8 channels,
                 then a 5-level butterfly and the 8 warps.  Head bias (head_grad_nchw_kernel): 5-level warp sum,
                 rows_per_block * ceil(nx / 32) chunk sums per block, ordered_rows_add_kernel: ceil(blocks / 8) + 8, one
                 add into the zeroed gradient.
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
import pytest
import torch

from checked_step import Step, bn_bwd_check, run_step
from f64_refs import (BF16, F64, STAT_TOL, U, bf16_check, bn_act_fwd_ref, check_z, conv_taps, passed, rtz_bf16, tapsum,
                      wgrad_ratio, wgrad_ref)
from helpers import init_darknet_weights

pytestmark = pytest.mark.gpu

BATCH = 2
SIZE = 608
MOMENTUM_DEFAULT = 0.1


def _keep_sets(st):
    """blocks whose tensors the bound self-test reuses: small grids only"""
    bl = st.plan.blocks
    k3 = [b for b in bl if b.k == 3 and not b.s2d and b.i > 0]
    acc1 = [b for b in bl if b.k == 1 and not b.s2d and not b.is_head and b.gsrc_acc]
    res = [b for b in bl if b.fuse_res]
    up = [b for b in bl if b.fuse_up and b.gy.ch_off + 32 + b.cout <= b.gy.cs]
    st.keep_fwd = {res[-1].i}
    st.keep_bwd = {k3[-1].i, acc1[-1].i, up[0].i}
    st.picks = dict(k3=k3[-1].i, acc1=acc1[-1].i, res=res[-1].i, up=up[0].i)


@pytest.fixture(scope="module")
def step():
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import cfgs
    dev = torch.device("cuda")
    model = pkg.Darknet(cfgs.yolov3_cfg(), {"context_factor": 1.0}, arc="default")
    init_darknet_weights(model, seed=1)
    model = model.to(dev).train()
    x = torch.rand(BATCH, 3, SIZE, SIZE, generator=torch.Generator().manual_seed(2)).to(dev)
    st = run_step(Step(model, x), 3, prepare=_keep_sets)
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
    from rotate_yolov3_b200 import _lib as lib
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
