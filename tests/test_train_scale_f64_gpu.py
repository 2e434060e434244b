"""Every kernel launch of the bf16 training step against float64 of its own inputs at the shapes it trains at: the eleven
sizes of `train.py --multi-scale` at base 608 (448 ... 768 in steps of 32: head grids 14 ... 24 at stride 32, odd ones
included, 56 ... 96 at stride 8) at batch 3, and the benchmark's batch 64 at 608^2 and at the recipe's largest size 768^2.

Bounds: those of test_train_step_f64_gpu.py's docstring, unchanged (E = n 2^-23 A per conv, half a bf16 ulp + E for bf16
outputs with the rounding-bias test, L 2^-24 sum |terms| for reductions, every ratio <= 1 so that a NaN fails), with n
and L from each launch's own schedule at its batch and grid (wgrad_plan, bn_chain, head_bias_chain).

Batch 3 runs checked_step.run_step as the 608 test does, and the eval forward at the same sizes the per-launch checks of
test_detect_forward_f64_gpu.py.  Batch 64 fills the card (at 768^2 the activation pool alone is 69.4 GB); run_step checks
the same launches there, over image chunks of at most BUDGET float64 bytes: the forward post hoc, the backward inside the
_backward_block wrapper on the live buffers, with only what a block overwrites copied to host memory first, and every
full reduction (wgrad, BN sums, d gamma / d beta / d slope, head bias) summed in float64 over chunks.

bn_act_bwd's dz bound leaves out the elements whose PReLU branch is ambiguous (u within four fp32 ulps of 0); z is bf16,
so in a channel every z equal to the bf16 value nearest -shift / scale drops out together: up to 0.01 % of a block's
elements are allowed here (820 of 26 M at 3 x 736^2, block 1), against 0.001 % at the one 608 shape of
test_train_step_f64_gpu.py.

The schedule table shows what the batch-64 shapes reach that batch 2 / 3 does not: longer split-K chains and more BN
pieces per CTA, and at 64 x 768^2 an im2col buffer of 2.43e9 elements (past 2^31 - 1), checked past element 2^31 up to its last interior pixel.
The last test puts plausible bugs into tensors these runs kept and requires each check to fail."""
import gc
import time

import pytest
import torch
import torch.nn.functional as F

from checked_step import Step, check_block_bwd, chunks, plan_layout, ref_bytes, run_step, schedule_rows
from f64_refs import (BF16, F64, bitwise, bn_chain, check_z, gemm_sms, interior, passed, sum_check, vint, wgrad_ratio,
                      wgrad_ref)
from helpers import init_darknet_weights, wgrad_plan

SIZES = list(range(448, 769, 32))        # train.py:52-54 at img_size 608: 608 * (0.75 ... 1.25), multiples of 32
SWEEP_BATCH = 3
BIG = (608, 768)
BIG_BATCH = 64
BUDGET = 2e9                             # float64 working set of one chunk of images
H100_SMS = 132
ODD = 480                                # the size of the stale-tile bug: grid 15 at stride 32
I31 = 2 ** 31 - 1


def _model(device="cpu"):
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import cfgs
    m = pkg.Darknet(cfgs.yolov3_cfg(), {"context_factor": 1.0}, arc="default")
    init_darknet_weights(m, seed=1)
    return m.to(device)


def _ratio_ok(v):
    return v <= 1.0                      # NaN fails


def bad_results(fwd, bwd):
    bad = []
    for part in (fwd, bwd):
        for i, r in part.items():
            for k, v in r.items():
                if k == "error":
                    bad.append((i, k, v[-800:]))
                elif k in ("dy_mode", "near_zero_u", "n_elems", "wgrad_rw", "mean_over_std"):
                    continue
                elif (isinstance(v, bool) and not v) or (isinstance(v, float) and not _ratio_ok(v)):
                    bad.append((i, k, v))
            if "near_zero_u" in r:      # see the docstring
                if r["near_zero_u"] > max(64, r["n_elems"] // 10000):
                    bad.append((i, "near_zero_u", r["near_zero_u"]))
    return bad


KINDS = (("conv z", "fwd", ("z",)), ("z bias", "fwd", ("z_bias",)), ("bn stats", "fwd", ("sums", "mean", "invstd",
         "finalize", "running")), ("bn_act_fwd", "fwd", ("y", "y_bias")), ("bn_act_bwd dz", "bwd", ("dz", "dz_bias")),
         ("d beta/gamma/slope", "bwd", ("dbeta", "dgamma", "dslope")), ("wgrad", "bwd", ("wgrad",)),
         ("dgrad", "bwd", ("dgrad", "dgrad_bias")), ("head bias", "bwd", ("dbias",)))


def worst_per_kind(fwd, bwd):
    out = {}
    for name, part, keys in KINDS:
        d = fwd if part == "fwd" else bwd
        vals = [(v, i) for i, r in d.items() for k, v in r.items() if k in keys and isinstance(v, float)]
        if vals:
            out[name] = max(vals, key=lambda t: (t[0] != t[0], t[0]))     # NaN first
    return out


def _print_worst(tag, res):
    print("%s worst |err| / bound per kernel kind: %s" % (tag, ", ".join(
        "%s %.3f (%d)" % (k, v, i) for k, (v, i) in worst_per_kind(res.fwd, res.bwd).items())))


class Res:
    """what a checked step leaves behind: results, schedule rows and a few kept tensors -- no plan, no model"""


def _keep_step(st, sms):
    res = Res()
    for k in ("fwd", "bwd", "im2col", "packs", "nbt_ok", "fwd_halo", "stash", "t_total", "max_ratio"):
        setattr(res, k, getattr(st, k))
    res.rows = schedule_rows(st.plan, sms)
    res.s2d = sorted(b.i for b in st.plan.blocks if b.s2d)
    res.stride2 = sorted(b.i for b in st.plan.blocks if b.stride == 2)
    res.n_blocks = len(st.plan.blocks)
    res.modes = {r["dy_mode"] for r in st.bwd.values() if "dy_mode" in r}
    res.acc = any(b.gsrc is not None and b.gsrc_acc for b in st.plan.blocks)
    res.d2s = any(b.s2d and not b.dxs_direct for b in st.plan.blocks)
    return res


def _release():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------
# batch 3 at the eleven recipe sizes: training step and eval forward
def _eval_forward(model, size):
    from checked_step import Run, check_buffers, check_conv, check_first, check_s2d_step, map_plan
    dev = torch.device("cuda")
    model.eval()
    model.use_cuda_graph = True
    x = torch.rand(SWEEP_BATCH, 3, size, size, generator=torch.Generator().manual_seed(5)).to(dev)
    st = Run("eval%d" % size, model)
    with torch.no_grad():
        model(x)
    torch.cuda.synchronize()
    st.plan, st.x, st.stash = model._plan, model._x_static, None
    map_plan(st)
    out = {0: check_first(st)}
    for i in sorted(st.conv_of)[1:]:
        out[i] = check_conv(st, i)
    s2d_ = {i: check_s2d_step(st, i) for i in st.s2d_of}
    ok, concat = check_buffers(st)
    return dict(res=out, s2d=s2d_, buffers_ok=ok, concat=concat, steps=[k for k, _ in st.plan["steps"]])


@pytest.fixture(scope="module")
def sweep():
    dev = torch.device("cuda")
    out = {}
    t0 = time.time()
    for size in SIZES:
        model = _model(dev).train()
        x = torch.rand(SWEEP_BATCH, 3, size, size, generator=torch.Generator().manual_seed(2)).to(dev)

        def prepare(st):
            if size == ODD:        # the conv output of the last 1024-filter block on the 15 x 15 grid
                blk = [b for b in st.plan.blocks if b.oh == 15 and not b.is_head and b.cout == 1024][-1]
                st.keep_fwd = {blk.i}
        st = run_step(Step(model, x), 3, prepare=prepare)
        res = _keep_step(st, torch.cuda.get_device_properties(0).multi_processor_count)
        del st
        res.eval = _eval_forward(model, size)
        del model, x
        _release()
        out[size] = res
        _print_worst("[scale %d x %d^2]" % (SWEEP_BATCH, size), res)
        print("[scale %d x %d^2] train step with checks %.1f s" % (SWEEP_BATCH, size, res.t_total))
    print("[scale] sweep %.1f s" % (time.time() - t0))
    return out


# ---------------------------------------------------------------------------------------------------------------
# batch 64 at 608^2 and 768^2, chunked
def needed_bytes(size):
    """device bytes of the checked batch-64 step: the activation pool and the parameter-sized state of its plan, the
    model's parameters, gradients and optimizer-free autograd copies, one dense cotangent, the chunk budget twice"""
    model = _model()
    shared = {}
    plan, pool = plan_layout(model.train(), BIG_BATCH, size, size, shared=shared)
    state = sum(t.numel() * t.element_size() for t in shared.values())
    params = sum(p.numel() for p in model.parameters()) * 4
    cot = sum(b.out.numel() * 4 for b in plan.blocks if b.is_head)
    return dict(pool=pool, total=pool + state + 3 * params + cot + 2 * int(BUDGET))


def _big_step(size):
    dev = torch.device("cuda")
    need = needed_bytes(size)
    free, total = torch.cuda.mem_get_info()
    if free < need["total"]:
        pytest.skip("64 x %d^2 checked step needs %.2f GB of device memory (pool %.2f GB), %.2f GB free"
                    % (size, need["total"] / 1e9, need["pool"] / 1e9, free / 1e9))
    torch.cuda.reset_peak_memory_stats()
    model = _model(dev).train()
    x = torch.rand(BIG_BATCH, 3, size, size, generator=torch.Generator().manual_seed(2)).to(dev)

    def prepare(st):
        plan = st.plan
        # a split-K wgrad of batch 64 (a short last split where there is one) whose operands are small enough to keep
        k3 = sorted((b for b in plan.blocks if b.k == 3 and not b.s2d and not b.is_head and b.i > 0),
                    key=lambda b: b.src.h * b.src.w * b.cin)
        sms = gemm_sms()
        plans = {b.i: wgrad_plan(3, b.cin_pad, b.cout_pad, BIG_BATCH, b.src.h, b.src.w, sms) for b in k3}
        pick = min(k3, key=lambda b: (plans[b.i]["ksplit"] == 1, not plans[b.i]["short_last"], b.src.h))
        st.pick, st.pick_plan = pick, plans[pick.i]
        st.stash["bn"] = dict(z=interior(pick.z, 0, pick.cout).clone(), sums=pick.sums.clone(),
                              l=bn_chain(BIG_BATCH, pick.oh, pick.ow, pick.cout)["sums"])
        # the first interior element of the im2col past index 2^31 (its image kept on the host)
        col = plan.col
        per = col[0].numel()
        b, rem = divmod(2 ** 31, per)
        if b < BIG_BATCH:
            y, x_ = divmod(rem // col.shape[3] + 1, col.shape[2])
            if y < 1:
                y, x_ = 1, 1
            elif x_ < 1:
                x_ = 1
            elif x_ > size:
                y, x_ = y + 1, 1
            if y > size:
                b, y, x_ = b + 1, 1, 1
            st.stash["col"] = dict(b=b, y=y, x=x_, c=0, col=col[b].cpu(), img=st.x[b].cpu(),
                                   index=b * per + (y * col.shape[2] + x_) * col.shape[3])

    def block_check(st, blk, orig):
        r = check_block_bwd(st, blk, orig)
        if blk is st.pick:      # the picked wgrad's operands and result (st.keep_bwd would keep its other launches' too)
            st.stash["wgrad"] = dict(x=vint(blk.src).clone(), dz=interior(blk.z, 0, blk.cout).clone(),
                                     offs=[(kh - 1, kw - 1) for kh in range(3) for kw in range(3)],
                                     got=blk.dw[:, :blk.cout, :blk.cin].clone(), plan=st.pick_plan)
        return r
    t0 = time.time()
    st = run_step(Step(model, x), 3, budget=BUDGET, prepare=prepare, block_check=block_check)
    res = _keep_step(st, torch.cuda.get_device_properties(0).multi_processor_count)
    res.checked_offsets = st.checked_offsets
    res.seconds = time.time() - t0
    del st, model, x
    _release()
    res.peak = torch.cuda.max_memory_allocated()
    res.need, res.free, res.card = need, free, total
    _print_worst("[scale %d x %d^2]" % (BIG_BATCH, size), res)
    print("[scale %d x %d^2] step with chunked checks %.1f s; peak max_memory_allocated %.2f GB (card %.1f GB, %.2f GB "
          "free before, %.2f GB estimated)" % (BIG_BATCH, size, res.seconds, res.peak / 1e9, total / 1e9, free / 1e9,
                                               need["total"] / 1e9))
    return res


@pytest.fixture(scope="module")
def big608(sweep):
    return _big_step(608)


@pytest.fixture(scope="module")
def big768(big608):
    return _big_step(768)


# ---------------------------------------------------------------------------------------------------------------
# host-side: recipe sizes, buffer arithmetic, chunk planner, schedule coverage at 132 SMs
def test_recipe_sizes_and_grids():
    assert len(SIZES) == 11 and SIZES[0] == 448 and SIZES[-1] == 768 and all(s % 32 == 0 for s in SIZES)
    assert [s // 32 for s in SIZES] == list(range(14, 25))
    assert {15, 17, 21, 23} <= {s // 32 for s in SIZES}
    assert [s // 8 for s in SIZES] == list(range(56, 97, 4))


def test_big_buffer_sizes():
    """the im2col and layer-0 z buffers of the batch-64 plans against the element and byte limits of 32-bit offsets"""
    m = _model().train()
    shared = {}
    p608, _ = plan_layout(m, 64, 608, 608, shared=shared)
    p768, need768 = plan_layout(m, 64, 768, 768, shared=shared)
    col608, col768 = p608.col, p768.col
    assert tuple(col608.shape) == (64, 610, 610, 64) and col608.numel() == 1524121600
    assert 2 * col608.numel() > I31 and col608.numel() <= I31            # 3.05 GB: past 2^31 bytes only
    assert tuple(col768.shape) == (64, 770, 770, 64) and col768.numel() == 2428518400 > I31
    z0 = p768.blocks[0].z
    assert tuple(z0.shape) == (64, 770, 770, 32) and 2 * z0.numel() == 2428518400
    assert 69.0e9 < need768 < 70.0e9
    rows = schedule_rows(p768, H100_SMS)
    assert max(r["max_offset"] for r in rows) == col768.numel() - 1


def test_chunk_planner():
    for batch, per_img, budget in ((64, 1.89e9, 2e9), (64, 3e7, 2e9), (3, 1e9, 2e9), (64, 5e9, 2e9), (1, 1.0, 1.0),
                                   (17, 1.0e8, 4.5e8)):
        cl = chunks(batch, per_img, budget)
        assert cl[0][0] == 0 and cl[-1][1] == batch and all(a[1] == b[0] for a, b in zip(cl, cl[1:]))
        assert all(b1 > b0 for b0, b1 in cl)
        assert all((b1 - b0) * per_img <= budget or b1 - b0 == 1 for b0, b1 in cl)
        assert len(cl) == -(-batch // max(1, min(batch, int(budget // per_img))))
    # one image of every forward reference of the 64 x 768^2 step fits the budget; of the backward ones, all but the
    # dgrad of layer 1 (its zero-inserted dz on the 768^2 grid), which fits the margin needed_bytes reserves
    m = _model().train()
    plan, _ = plan_layout(m, 64, 768, 768)
    per = {k: max(ref_bytes(b).get(k, 0) for b in plan.blocks) for k in ("fwd", "wgrad", "dgrad")}
    print("[scale 64x768] float64 bytes per image, worst block: %s" % per)
    assert per["fwd"] <= BUDGET and per["wgrad"] <= BUDGET, per
    assert max(ref_bytes(b)["dgrad"] for b in plan.blocks if b.i > 1) <= BUDGET < per["dgrad"] <= 2 * BUDGET, per


def coverage(big, small):
    """what the batch-64 launches reach that no batch-2/3 launch does (rows of schedule_rows)"""
    def launches(rows, key):
        return [r[key] for r in rows if key in r]
    out = dict(
        per_split=(max(w["per_split"] for w in launches(big, "wgrad")), max(w["per_split"] for w in launches(small, "wgrad"))),
        ksplit_new=sorted({w["ksplit"] for w in launches(big, "wgrad")} - {w["ksplit"] for w in launches(small, "wgrad")}),
        bn_per_cta=(max(p["per_cta"] for p in launches(big, "bn_bwd") + launches(big, "bn_fwd")),
                    max(p["per_cta"] for p in launches(small, "bn_bwd") + launches(small, "bn_fwd"))),
        head_rpb=(max(h[0] for h in launches(big, "head_bias")), max(h[0] for h in launches(small, "head_bias"))),
        past_ring=sum(c["per_cta"] > c["staging"] for k in ("fwd", "dgrad") for c in launches(big, k)),
        max_offset=max(r["max_offset"] for r in big))
    return out


def assert_coverage(cov):
    assert cov["per_split"][0] > cov["per_split"][1], cov
    assert cov["ksplit_new"], cov
    assert cov["bn_per_cta"][0] > cov["bn_per_cta"][1], cov
    assert cov["past_ring"] > 0, cov


def test_schedule_coverage_mirror():
    """the coverage claims from the plans' geometry on an H100 SXM (132 SMs), without a device"""
    m = _model().train()
    shared = {}
    small = schedule_rows(plan_layout(m, 2, 608, 608, shared=shared)[0], H100_SMS)
    for s in SIZES:
        small += schedule_rows(plan_layout(m, SWEEP_BATCH, s, s, shared=shared)[0], H100_SMS)
    for size in BIG:
        big = schedule_rows(plan_layout(m, BIG_BATCH, size, size, shared=shared)[0], H100_SMS)
        cov = coverage(big, small)
        assert_coverage(cov)
        assert (cov["max_offset"] > I31) == (size == 768), cov


# ---------------------------------------------------------------------------------------------------------------
# the device
@pytest.mark.gpu
def test_sweep_covers_every_launch(sweep):
    for size, r in sweep.items():
        assert r.n_blocks == 75 and len(r.fwd) == 75, size
        assert len([i for i, b in r.bwd.items() if "wgrad" in b]) == 75, size
        # every recipe size is a multiple of 32: every stride-2 block runs on the space-to-depth copy
        assert r.s2d == r.stride2 == [1, 5, 12, 37, 62], (size, r.s2d, r.stride2)
        assert r.modes == {0, 1, 2} and r.acc and r.d2s, size
        assert r.im2col == dict(bits=True, pad_zero=True, halo=True), (size, r.im2col)
        assert len(r.packs) == 149 and all(p[2] for p in r.packs), size
        assert r.nbt_ok and r.fwd_halo, size


@pytest.mark.gpu
def test_sweep_train_step_vs_float64(sweep):
    bad = {size: bad_results(r.fwd, r.bwd) for size, r in sweep.items()}
    assert not any(bad.values()), {s: b[:5] for s, b in bad.items() if b}


@pytest.mark.gpu
def test_sweep_eval_forward_vs_float64(sweep):
    for size, r in sweep.items():
        ev = r.eval
        assert ev["steps"].count("first") == 1 and ev["steps"].count("conv") == 74 and ev["steps"].count("s2d") == 4
        assert sorted(ev["s2d"]) == [5, 12, 37, 62] and all(v["bits"] and v["pad_zero"] for v in ev["s2d"].values())
        assert ev["buffers_ok"] and ev["concat"] == [384, 768], size
        bad = [(i, k, v) for i, x in ev["res"].items() for k, v in x.items()
               if (k in ("max", "bias", "fold") and not _ratio_ok(v))
               or (k in ("w_bits", "b_bits", "slope", "up_copies", "xs_pad_zero") and not v)]
        assert not bad, (size, bad[:5])
        print("[scale eval %d x %d^2] worst conv ratio %.3f, worst bias %.3f" % (
            SWEEP_BATCH, size, max(x["max"] for x in ev["res"].values()),
            max(x.get("bias", 0.0) for x in ev["res"].values())))


@pytest.mark.gpu
@pytest.mark.parametrize("size", BIG)
def test_batch64_step_vs_float64(request, size):
    r = request.getfixturevalue("big%d" % size)
    assert r.n_blocks == 75 and len(r.fwd) == 75 and len([i for i, b in r.bwd.items() if "wgrad" in b]) == 75
    assert r.modes == {0, 1, 2} and r.acc and r.d2s
    assert r.s2d == r.stride2 == [1, 5, 12, 37, 62]
    assert r.im2col == dict(bits=True, pad_zero=True, halo=True), r.im2col
    assert len(r.packs) == 149 and all(p[2] for p in r.packs)
    assert r.nbt_ok and r.fwd_halo
    bad = bad_results(r.fwd, r.bwd)
    assert not bad, bad[:5]


def _print_rows(tag, rows):
    print("%s blk kind grid   | conv fwd tiles/CTA (ring) | dgrad tiles/CTA | wgrad ksplit x per_split (last) | "
          "bn pieces/CTA x rows | head rows/blk | max offset" % tag)
    for r in rows:
        f, d, w = r["fwd"], r.get("dgrad"), r["wgrad"]
        cols = ["%3d %-4s %3dx%-3d" % (r["i"], r["kind"], r["grid"][0], r["grid"][1]),
                "%7d %4d/CTA (%d)" % (f["tiles"], f["per_cta"], f["staging"]),
                "%4d/CTA (%d)" % (d["per_cta"], d["staging"]) if d else "      -     ",
                "%3d x %4d (%4d)" % (w["ksplit"], w["per_split"], w["last"])]
        if "bn_bwd" in r:
            cols.append("%3d x %d / %3d x %d" % (r["bn_fwd"]["per_cta"], 1, r["bn_bwd"]["per_cta"], r["bn_bwd"]["rows"]))
        else:
            cols.append("head %d rows x %d blocks" % r["head_bias"])
        cols.append("%.3e" % r["max_offset"])
        print(tag + " " + " | ".join(cols))


@pytest.mark.gpu
def test_schedule_coverage(sweep, big608, big768):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    small = schedule_rows(plan_layout(_model().train(), 2, 608, 608)[0], sms)
    for r in sweep.values():
        small += r.rows
    for size, big in ((608, big608), (768, big768)):
        _print_rows("[scale 64x%d]" % size, big.rows)
        cov = coverage(big.rows, small)
        print("[scale 64x%d] coverage against batch 2 / 3: %s" % (size, cov))
        assert_coverage(cov)
    n_col, off_col = big768.checked_offsets["col"]
    print("[scale 64x768] im2col: %d elements, checked up to element offset %d" % (n_col, off_col))
    assert n_col > I31 and 2 ** 31 < off_col < n_col


@pytest.mark.gpu
def test_bounds_reject_bugs_at_the_new_shapes(sweep, big608, big768):
    found = {}
    # split-K weight gradient at batch 64: the last (shorter) split's partial lost, the last image left out
    wg = big768.stash["wgrad"]
    pw = wg["plan"]
    assert pw["ksplit"] > 1, pw
    want, mag = wgrad_ref(wg["x"], wg["dz"], wg["offs"])
    assert wgrad_ratio(wg["got"], want, mag, pw) <= 1.0
    b, h, w = wg["dz"].shape[:3]
    flat = torch.zeros(b * (h + 2) * (w + 2), dtype=F64, device=want.device)
    flat[64 * (pw["ksplit"] - 1) * pw["per_split"]:] = 1.0
    mask = flat.view(b, h + 2, w + 2)[:, 1:-1, 1:-1, None]
    lost, _ = wgrad_ref(wg["x"], wg["dz"].double() * mask, wg["offs"])
    found["lost_last_split"] = {"max": wgrad_ratio(wg["got"], want - lost, mag, pw)}
    last, _ = wgrad_ref(wg["x"][-1:], wg["dz"][-1:], wg["offs"])
    found["wgrad_without_last_image"] = {"max": wgrad_ratio(wg["got"], want - last, mag, pw)}
    # BN sums over 63 of 64 images
    bn = big768.stash["bn"]
    z64 = bn["z"].double().reshape(64, -1, bn["z"].shape[-1])
    c = z64.shape[-1]
    s_all, a_all = z64.sum((0, 1)), z64.abs().sum((0, 1))
    assert sum_check(bn["sums"][:c], s_all, bn["l"], a_all) <= 1.0
    found["bn_sum_63_images"] = {"max": sum_check(bn["sums"][:c], z64[:63].sum((0, 1)), bn["l"], a_all)}
    # one im2col element past index 2^31 of the 64 x 768^2 buffer
    cs = big768.stash["col"]
    assert cs["index"] > 2 ** 31
    want_col = F.unfold(cs["img"][None], 3, padding=1).view(1, 27, 768, 768).permute(0, 2, 3, 1).to(BF16)[0]
    got_col = cs["col"][1:-1, 1:-1, :27].clone()
    assert bitwise(got_col, want_col)
    got_col[cs["y"] - 1, cs["x"] - 1, cs["c"]] += 1.0
    found["im2col_past_2^31"] = {"bits": bitwise(got_col, want_col)}
    # the odd grid: a conv output whose last partial M tile (128 padded pixels) is left stale
    zc = next(v for k, v in sweep[ODD].stash.items() if k[0] == "z")
    assert passed(check_z(zc["got"], zc["want"], zc["mag"], zc["n"]))
    got = zc["got"].clone()
    b, hh, ww = got.shape[:3]
    np_ = b * (hh + 2) * (ww + 2)
    assert np_ % 128, np_
    stale = 0
    for p in range(np_ // 128 * 128, np_):
        img, rem = divmod(p, (hh + 2) * (ww + 2))
        y, x = divmod(rem, ww + 2)
        if 1 <= y <= hh and 1 <= x <= ww and img > 0:
            got[img, y - 1, x - 1] = zc["got"][0, y - 1, x - 1]        # what the tile held for another image
            stale += 1
    assert stale > 0
    found["stale_last_m_tile"] = check_z(got, zc["want"], zc["mag"], zc["n"])
    for name, r in found.items():
        print("[scale bite] %-26s %s" % (name, {k: (round(v, 3) if isinstance(v, float) else v) for k, v in r.items()}))
    for name, r in found.items():
        assert not passed(r), (name, r)
    assert found["lost_last_split"]["max"] > 1 and found["wgrad_without_last_image"]["max"] > 1
