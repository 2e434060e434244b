"""Same inputs, same bits: the fixed-order reductions of the bf16 training step, and their float64 accuracy.

The training step adds every multi-CTA reduction in a fixed order -- BN statistics and BN backward sums (per-CTA partial
rows, then bn_sums_reduce_kernel), split-K weight gradients (the last split adds the splits in split order), the
objectness loss sum and the head bias gradient (ordered_sum_add_kernel / ordered_rows_add_kernel) and matched loss rows
that share a cell (rows_scatter_add_kernel) -- so its numbers do not depend on the order in which CTAs finish.

Kernel level: each reduction runs three times on identical inputs, the last time next to a stream of large bf16 matmuls
on a second stream (the CTAs then finish in a different order), and the results must be bitwise equal.  Step level:
forward, compute_loss and backward of the yolov3 graph must give identical bits across a rerun, a second model instance,
another stream and CUDA-graph capture / replay.

Float64: the ordered sums must also be accurate, |got - want| <= KAPPA_SUM * sqrt(n_add) * 2^-24 * sum|terms|, with n_add
the longest chain of fp32 additions (per thread, within the CTA, across the CTA partial rows), mirrored from the launch
geometry.  KAPPA_SUM = 2 for every shape, chosen from the first run on an H100 SXM (132 SMs, 700 W): the worst ratio at
KAPPA_SUM = 1 was 0.78 (sum of squares, c = 2048, a 15-add chain), 0.01-0.4 elsewhere.  Taking one CTA's partial row out
of the reference breaks the bound by a factor of thousands.

The one-pass variance E[z^2] - E[z]^2 at mean / std = 8 (E[z^2] / var = 68.5) was measured 1.6e-5 relative to float64
against a bound of 1.4e-4 (the sum bound times that amplification); at mean / std = 0.3 it is 2e-7 to 5e-7."""
import ctypes
import math

import pytest
import torch

from builders import STEP_HYP, assert_same, repeat, ryolo_lib, small_train_model, step_targets
from f64_refs import CASES, Case, bf, gemm_sms

pytestmark = pytest.mark.gpu

KAPPA_SUM = 2.0
U = 2.0 ** -24


# ---------------------------------------------------------------------------------------------------------------
# BN geometry mirror (csrc/bnact.cu rows_per_block, csrc/bnpipe.cuh mk_pieces / pipe_ok)
def bn_geometry(b, h, w, c, cs, sms):
    cgs = c // 8
    pstep = 256 // cgs
    if cs == c:                                     # TMA row pipe: pieces of <= 1280 16-byte items, <= 2 CTAs per SM
        max_px = 1280 // cgs
        ppr = -(-w // max_px)
        px = -(-w // ppr)
        total = b * h * ppr
        per_cta = -(-total // (2 * sms))
        grid = -(-total // per_cta)
        per_thread = -(-total // grid) * -(-px // pstep)
        rpb = None
    else:                                           # direct kernels: a CTA owns rows_per_block image rows
        per_row = w * cgs
        nrows = b * h
        rpb = max(1, min(-(-16384 // per_row), -(-nrows // 592)))
        grid = -(-nrows // rpb)
        per_thread = rpb * -(-w // pstep)
    n_add = per_thread + pstep + -(-grid // 8) + 8
    return dict(pipe=cs == c, grid=grid, rpb=rpb, n_add=n_add)


def bn_stats_call(zb, cs, b, h, w, c, eps=1e-5, momentum=0.1, gamma=None, beta=None, rm=None, rv=None):
    L = ryolo_lib()
    dev = zb.device
    sums = torch.full((2 * c,), 3.0, device=dev)
    mean, inv, sc, sh = (torch.empty(c, device=dev) for _ in range(4))
    gamma = gamma if gamma is not None else torch.ones(c, device=dev)
    beta = beta if beta is not None else torch.zeros(c, device=dev)
    st = L.lib.ryolo_bn_stats_finalize(L.ptr(zb), cs, b, h, w, c, L.ptr(sums), eps, momentum, L.ptr(gamma), L.ptr(beta),
                                       L.ptr(mean), L.ptr(inv), L.ptr(sc), L.ptr(sh), L.ptr(rm) if rm is not None else None,
                                       L.ptr(rv) if rv is not None else None, L.stream_ptr())
    assert st == 0, L.last_error()
    return sums, mean, inv, sc, sh


def sum_ratio(got, want, mag, n_add):
    return float(((got.double() - want).abs() / (KAPPA_SUM * math.sqrt(n_add) * U * mag + 1e-30)).max())


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path,c,cs,b,h,w", [("direct", 64, 128, 2, 30, 40), ("pipe", 64, 64, 2, 50, 200),
                                             ("pipe", 2048, 2048, 2, 5, 6), ("direct", 32, 64, 4, 38, 38)])
def test_bn_stats_finalize_is_bitwise_repeatable(path, c, cs, b, h, w):
    from rotate_yolov3_b200 import layout as Lo
    geo = bn_geometry(b, h, w, c, cs, gemm_sms())
    assert geo["pipe"] == (path == "pipe") and geo["grid"] > 8
    g = torch.Generator().manual_seed(c + h)
    z = bf(torch.randn(b, c, h, w, generator=g) * 1.3 + 0.4).cuda()
    zb = Lo.to_padded_nhwc(z, cs)
    gamma, beta = (0.5 + torch.rand(c, generator=g)).cuda(), torch.randn(c, generator=g).cuda()
    rm0, rv0 = torch.randn(c, generator=g).cuda(), (0.5 + torch.rand(c, generator=g)).cuda()

    def run():
        rm, rv = rm0.clone(), rv0.clone()
        return bn_stats_call(zb, cs, b, h, w, c, gamma=gamma, beta=beta, rm=rm, rv=rv) + (rm, rv)

    sums, mean, inv, sc, sh, rm, rv = repeat(run)
    assert torch.allclose(mean.double(), z.double().mean((0, 2, 3)), atol=1e-5)


def _bwd_inputs(c, b, h, w, up, seed):
    g = torch.Generator().manual_seed(seed)
    z = bf(torch.randn(b, c, h, w, generator=g) * 1.2 + 0.1).cuda()
    oh, ow = (2 * h, 2 * w) if up == 1 else (h, w)
    dy = bf(torch.randn(b, c, oh, ow, generator=g)).cuda()
    mean = (0.1 * torch.randn(c, generator=g)).cuda()
    inv = (0.5 + torch.rand(c, generator=g)).cuda()
    return z, dy, mean, inv


def bn_bwd_call(dyb, dcs, up, zb_master, cs, b, h, w, c, scale, shift, mean, inv, slope, has_act=1, slope_dev=None):
    L = ryolo_lib()
    zb = zb_master.clone()                          # the call overwrites z with dz
    sums = torch.full((2 * c + 1,), 5.0, device="cuda")
    st = L.lib.ryolo_bn_act_bwd(L.ptr(dyb), dcs, up, L.ptr(zb), cs, b, h, w, c, L.ptr(scale), L.ptr(shift), L.ptr(mean),
                                L.ptr(inv), slope, has_act, 1, L.ptr(sums), None, 0, 0,
                                L.ptr(slope_dev) if slope_dev is not None else None, L.stream_ptr())
    assert st == 0, L.last_error()
    return sums, zb


@pytest.mark.parametrize("up,cs_mode", [(0, "pipe"), (0, "direct"), (1, "pipe"), (2, "pipe")])
def test_bn_act_bwd_is_bitwise_repeatable(up, cs_mode):
    """dy modes: 0 plain (on the pipe next to z, or direct loads for a wider buffer), 1 at 2x resolution (upsample
    adjoint), 2 in the space-to-depth layout of a following stride-2 block; sums, slope scalar sums[2c] and dz"""
    from rotate_yolov3_b200 import layout as Lo
    c, b, h, w = 64, 2, 48, 120
    cs = c if cs_mode == "pipe" else 128
    z, dy, mean, inv = _bwd_inputs(c, b, h, w, up, 7 + up)
    zb = Lo.to_padded_nhwc(z, cs)
    if up == 2:
        q = torch.cat([dy[:, :, ry::2, rx::2] for ry in range(2) for rx in range(2)], 1)
        dyb, dcs = Lo.to_padded_nhwc(q, 4 * c), 4 * c
    else:
        dyb, dcs = Lo.to_padded_nhwc(dy, cs), cs
    g = torch.Generator().manual_seed(3)
    scale, shift = (0.5 + torch.rand(c, generator=g)).cuda(), (0.2 * torch.randn(c, generator=g)).cuda()
    sd = torch.tensor([0.13], device="cuda")
    sums, dz = repeat(lambda: bn_bwd_call(dyb, dcs, up, zb, cs, b, h, w, c, scale, shift, mean, inv, 0.0, 1, sd))
    assert float(sums[2 * c]) != 5.0 and torch.isfinite(sums).all()


@pytest.mark.parametrize("name", list(CASES))
def test_wgrad_is_bitwise_repeatable(name):
    c = Case(**CASES[name][0], seed=21)
    assert c.plan()["ksplit"] > 1
    repeat(lambda: (c.run(c.new_dw()),))


def _head_grad_call(g, B, C, ny, nx, cs):
    L = ryolo_lib()
    dst = torch.zeros((B, ny + 2, nx + 2, cs), dtype=torch.bfloat16, device="cuda")
    bias = torch.zeros(C, device="cuda")
    L.check(L.lib.ryolo_head_grad_nchw_to_padded(L.ptr(g), B, C, ny, nx, L.ptr(dst), cs, L.ptr(bias), L.stream_ptr()), "hg")
    return bias, dst


HEAD = (30, 24, 80, 40)          # batch * ny = 2400 > 2048: two image rows per block


def test_head_bias_grad_repeatable_and_vs_float64():
    B, C, ny, nx = HEAD
    rpb = -(-(B * ny) // 2048)
    assert rpb >= 2
    g = torch.randn(B, C, ny, nx, generator=torch.Generator().manual_seed(4)).cuda()
    bias, dst = repeat(lambda: _head_grad_call(g, B, C, ny, nx, 32))
    blocks = -(-ny // rpb) * B
    # chain: 5 shuffle levels, rpb x ceil(nx / 32) adds into the block's row, the rows / 8 + 8 ordered adds, += into bias
    n_add = 5 + rpb * -(-nx // 32) + -(-blocks // 8) + 8 + 1
    g64 = g.double()
    r = sum_ratio(bias, g64.sum((0, 2, 3)), g64.abs().sum((0, 2, 3)), n_add)
    print("[sums] head bias gradient: %d blocks, n_add %d, worst ratio %.4f" % (blocks, n_add, r))
    assert r <= 1.0, r


def _head(B, na, ny, nx, no, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(B, na, ny, nx, no, generator=g) * 3.0).cuda()
    tobj = (torch.rand(B, na, ny, nx, generator=g) < 0.05).float().cuda()
    return x, tobj


def _obj_call(x, tobj, pw):
    L = ryolo_lib()
    B, na, ny, nx, no = x.shape
    strides = (ctypes.c_longlong * 5)(*x.stride())
    out = torch.zeros(1, dtype=torch.float64, device="cuda")
    L.check(L.lib.ryolo_obj_bce_fwd(L.ptr(x), strides, B, na, ny, nx, no, 5, L.ptr(tobj), pw, L.ptr(out), L.stream_ptr()),
            "obj_bce_fwd")
    return (out,)


def test_objectness_sum_repeatable_and_vs_float64():
    x, tobj = _head(4, 3, 76, 76, 7, 8)
    pw = 1.7
    (got,) = repeat(lambda: _obj_call(x, tobj, pw))
    xv, t = x[..., 5].double(), tobj.double()
    lw = 1.0 + (pw - 1.0) * t
    terms = (1.0 - t) * xv + lw * (torch.log1p(torch.exp(-xv.abs())) + (-xv).clamp(min=0))
    mag = ((1.0 - t) * xv).abs() + lw * (torch.log1p(torch.exp(-xv.abs())) + (-xv).clamp(min=0))
    # per cell a handful of fp32 operations (log1pf / expf within 2 ulp); the partials are added in double
    err, bound = abs(float(got) - float(terms.sum())), 8 * U * float(mag.sum())
    print("[sums] objectness: |got - want| %.3e, bound %.3e" % (err, bound))
    assert err <= bound, (err, bound)


def _rows(B, na, ny, nx, n_rows, seed):
    g = torch.Generator().manual_seed(seed)
    cells = torch.stack([torch.randint(0, s, (12,), generator=g) for s in (B, na, ny, nx)], 1)
    pick = torch.randint(0, 12, (n_rows,), generator=g)
    idx = cells[pick].clone()
    mask = torch.ones(n_rows, dtype=torch.uint8)
    mask[torch.randperm(n_rows, generator=g)[:n_rows // 8]] = 0          # masked rows write nothing
    oob = torch.randperm(n_rows, generator=g)[:n_rows // 10]             # rows outside the map (border targets)
    idx[oob[0::4], 3] = nx
    idx[oob[1::4], 2] = -1
    idx[oob[2::4], 0] = B
    idx[oob[3::4], 1] = na
    return idx, mask


def _scatter_call(g0, idx, mask, vals, scale):
    L = ryolo_lib()
    g = g0.clone()
    B, na, ny, nx, no = g.shape
    strides = (ctypes.c_longlong * 5)(*g.stride())
    cols = [idx[:, k].contiguous().cuda() for k in range(4)]
    m8 = mask.cuda()
    L.check(L.lib.ryolo_loss_rows_scatter_add(L.ptr(g), strides, B, na, ny, nx, no, *[L.ptr(cl) for cl in cols], L.ptr(m8),
                                              idx.shape[0], L.ptr(vals), L.ptr(scale), L.stream_ptr()), "scatter")
    return (g,)


def test_rows_scatter_add_repeatable_and_vs_float64():
    B, na, ny, nx, no = 2, 3, 10, 12, 7
    idx, mask = _rows(B, na, ny, nx, 400, 11)
    g0 = torch.randn(B, na, ny, nx, no, generator=torch.Generator().manual_seed(12)).cuda()
    vals = torch.randn(400, no, generator=torch.Generator().manual_seed(13)).cuda()
    scale = torch.tensor([0.37], device="cuda")
    (got,) = repeat(lambda: _scatter_call(g0, idx, mask, vals, scale))
    want, mag = g0.double().clone(), g0.double().abs()
    mult = torch.zeros(B, na, ny, nx, dtype=torch.float64)
    live = 0
    for i in range(idx.shape[0]):
        b, a, y, x = (int(v) for v in idx[i])
        if not mask[i] or not (0 <= b < B and 0 <= a < na and 0 <= y < ny and 0 <= x < nx):
            continue
        live += 1
        v = vals[i].double() * float(scale)
        want[b, a, y, x] += v
        mag[b, a, y, x] += v.abs()
        mult[b, a, y, x] += 1
    assert live > 200 and int(mult.max()) >= 20                 # many rows per cell
    # fp32, row order: one rounding of each product and of each add, bounded by the running magnitude
    bound = (2 * mult.cuda()[..., None] + 1) * U * mag
    assert bool(((got.double() - want).abs() <= bound).all())
    untouched = (mult == 0).cuda()
    assert torch.equal(got[untouched], g0[untouched])


# ---------------------------------------------------------------------------------------------------------------
# float64 accuracy of the BN sums
@pytest.mark.parametrize("name,c,cs,b,h,w,mu", [
    ("few_ctas", 64, 128, 1, 4, 8, 0.3),          # 4 CTAs < 8 reduce parts: some parts are empty
    ("short_last", 64, 128, 1, 601, 16, 0.3),     # 2 rows per CTA, the last CTA has one
    ("c2048_pipe", 2048, 2048, 2, 5, 6, 0.3),     # the full kAccFloats staging
    ("c2048_direct", 2048, 2112, 2, 5, 6, 0.3),
    ("pipe_pieces", 64, 64, 2, 50, 200, 0.3),     # several pieces per row
    ("high_mean", 64, 64, 4, 38, 38, 8.0),        # mean / std = 8: one-pass variance E[z^2] - E[z]^2 cancels
])
def test_bn_stats_vs_float64(name, c, cs, b, h, w, mu):
    from rotate_yolov3_b200 import layout as Lo
    geo = bn_geometry(b, h, w, c, cs, gemm_sms())
    if name == "few_ctas":
        assert geo["grid"] < 8
    if name == "short_last":
        assert geo["rpb"] == 2 and (b * h) % geo["rpb"] != 0
    g = torch.Generator().manual_seed(h + c)
    z = bf(torch.randn(b, c, h, w, generator=g) + mu).cuda()
    zb = Lo.to_padded_nhwc(z, cs)
    eps = 1e-5
    sums, mean, inv, _, _ = bn_stats_call(zb, cs, b, h, w, c, eps=eps)
    torch.cuda.synchronize()
    z64 = z.double()
    s1, s2 = z64.sum((0, 2, 3)), (z64 * z64).sum((0, 2, 3))
    m1, m2 = z64.abs().sum((0, 2, 3)), s2
    r1 = sum_ratio(sums[:c], s1, m1, geo["n_add"])
    r2 = sum_ratio(sums[c:], s2, m2, geo["n_add"])
    n = b * h * w
    var64 = z64.var((0, 2, 3), unbiased=False)                 # float64 reference (Welford on the device)
    var_got = 1.0 / inv.double() ** 2 - eps
    rel = float(((var_got - var64).abs() / var64).max())
    # sum errors amplified by E[z^2] / var (the cancellation), the fp32 finalisation and rsqrtf: a few ulps more
    amp = float((s2 / n / var64).max())
    rel_bound = U * (amp * (2 * KAPPA_SUM * math.sqrt(geo["n_add"]) + 4) + 8)
    print("[sums] BN %s: %s grid %d n_add %d, worst ratio sum %.4f sumsq %.4f; variance rel err %.2e (bound %.2e, "
          "E[z^2]/var %.1f)" % (name, "pipe" if geo["pipe"] else "direct", geo["grid"], geo["n_add"], r1, r2, rel, rel_bound, amp))
    assert r1 <= 1.0 and r2 <= 1.0, (r1, r2)
    assert rel <= rel_bound, (rel, rel_bound)
    assert float(((mean.double() - s1 / n).abs() / (m1 / n)).max()) <= KAPPA_SUM * math.sqrt(geo["n_add"]) * U + 2 * U
    if name == "short_last":
        # sensitivity: the reference without the partial row of one CTA (rows 2k, 2k+1) breaks the bound
        k = geo["grid"] // 2
        zr = z64.permute(0, 2, 1, 3).reshape(b * h, c, w)[2 * k:2 * k + 2]
        r_lost = sum_ratio(sums[c:], s2 - (zr * zr).sum((0, 2)), m2, geo["n_add"])
        r_lost1 = sum_ratio(sums[:c], s1 - zr.sum((0, 2)), m1, geo["n_add"])
        print("[sums] BN reference without CTA %d: worst ratio sum %.1f sumsq %.1f" % (k, r_lost1, r_lost))
        assert r_lost > 1.0 and r_lost1 > 1.0


@pytest.mark.parametrize("cs_mode", ["pipe", "direct"])
def test_bn_bwd_sums_vs_float64(cs_mode):
    """scale 1, shift 0: u = z exactly, so the PReLU mask and the slope term sum(dy * z over z <= 0) are exact in float64;
    zhat = (z - mean) * invstd is rounded in fp32 exactly as the kernel does, its sum of products is then float64"""
    from rotate_yolov3_b200 import layout as Lo
    c, b, h, w = 64, 2, 48, 120
    cs = c if cs_mode == "pipe" else 128
    geo = bn_geometry(b, h, w, c, cs, gemm_sms())
    z, dy, mean, inv = _bwd_inputs(c, b, h, w, 0, 31)
    zb, dyb = Lo.to_padded_nhwc(z, cs), Lo.to_padded_nhwc(dy, cs)
    one, zero = torch.ones(c, device="cuda"), torch.zeros(c, device="cuda")
    slope = 0.125
    sums, _ = bn_bwd_call(dyb, cs, 0, zb, cs, b, h, w, c, one, zero, mean, inv, slope)
    torch.cuda.synchronize()
    du = torch.where(z > 0, dy, dy * slope).double()
    zh = ((z - mean.view(1, -1, 1, 1)) * inv.view(1, -1, 1, 1)).double()       # fp32 ops, as in the kernel
    r1 = sum_ratio(sums[:c], du.sum((0, 2, 3)), du.abs().sum((0, 2, 3)), geo["n_add"])
    r2 = sum_ratio(sums[c:2 * c], (du * zh).sum((0, 2, 3)), (du * zh).abs().sum((0, 2, 3)), geo["n_add"])
    neg = (z <= 0).double()
    sl = (dy.double() * z.double() * neg).sum()
    r3 = sum_ratio(sums[2 * c:], sl.view(1), (dy.double() * z.double() * neg).abs().sum().view(1), geo["n_add"] + 5)
    print("[sums] BN backward %s: n_add %d, worst ratio sum(du) %.4f sum(du*zhat) %.4f slope %.4f"
          % (cs_mode, geo["n_add"], r1, r2, r3))
    assert max(r1, r2, r3) <= 1.0, (r1, r2, r3)


# ---------------------------------------------------------------------------------------------------------------
# step level
def _setup(m):
    m.nc, m.hyp, m.arc = 1, STEP_HYP, "default"
    return m


def _step(m, x, t):
    from rotate_yolov3_b200.loss import compute_loss
    for p in m.parameters():
        p.grad = None
    ps = m(x)
    loss, items = compute_loss(ps, t.clone(), m, STEP_HYP)
    loss.backward()
    out = {"p%d" % k: p.detach().clone() for k, p in enumerate(ps)}
    out["loss"], out["items"] = loss.detach().clone(), items.detach().clone()
    for n, p in m.named_parameters():
        out["grad:" + n] = p.grad.clone()
    for n, buf in m.named_buffers():
        out["buf:" + n] = buf.clone()
    torch.cuda.synchronize()
    return out


def test_training_step_is_bitwise_repeatable():
    m = _setup(small_train_model())
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    x = torch.rand(2, 3, 128, 160, generator=torch.Generator().manual_seed(17)).cuda()
    t = step_targets()
    ref = _step(m, x, t)
    assert float(ref["items"][2]) > 0            # matched rows exist (regression term)
    assert all(torch.isfinite(v).all() for v in ref.values() if v.is_floating_point())
    # 1. the same model again, from the same restored state
    m.load_state_dict(sd0)
    assert_same(ref, _step(m, x, t), "rerun")
    # 2. a second instance: parameters, plan buffers and scratch at other addresses
    m2 = _setup(small_train_model())
    m2.load_state_dict(sd0)
    assert m2.module_list[0].Conv2d.weight.data_ptr() != m.module_list[0].Conv2d.weight.data_ptr()
    assert_same(ref, _step(m2, x, t), "second instance")
    del m2
    # 3. on another stream: per-stream scratch buffers
    m.load_state_dict(sd0)
    side, cur = torch.cuda.Stream(), torch.cuda.current_stream()
    side.wait_stream(cur)
    with torch.cuda.stream(side):
        out = _step(m, x, t)
    cur.wait_stream(side)
    assert_same(ref, out, "side stream")
    # 4. CUDA graphs: the capture step and a replayed step
    m3 = _setup(small_train_model())
    m3.load_state_dict(sd0)
    m3.use_cuda_graph = True
    assert_same(ref, _step(m3, x, t), "graph capture step")
    m3.load_state_dict(sd0)                      # in place: the captured graphs stay valid
    assert_same(ref, _step(m3, x, t), "graph replay")
    assert m3._tplan.replayed_kernels > 0
