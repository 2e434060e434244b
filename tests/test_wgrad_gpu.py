"""wgmma weight gradient (csrc/wgrad.cu) against float64, element by element, on the paths the training step takes.

For bf16-exact x and dz the exact gradient is want = conv2d_weight(x, dz) in float64, and every fp32 addition the kernel
makes can be off by at most half an ulp of the running sum, which is bounded by A = conv2d_weight(|x|, |dz|).  With random
signs the rounding errors add like a random walk, so every entry must satisfy

    |got - want| <= KAPPA * sqrt(n_add) * 2^-24 * A + TINY,     n_add = ceil(K / 16) + ksplit

where K is the padded pixel count (the GEMM's K dimension, whole 64-pixel k-steps), K / 16 the sequential wgmma
accumulations and ksplit the split-K partial sums that the last split adds in split order.  KAPPA = 1 for every shape,
chosen from the first run on an H100 SXM (132 SMs, 700 W): the worst |got - want| / bound over all cases was 0.143
(ksize 2, cin_pad 256, ksplit 4), 0.012-0.064 on the long-K cases.  A k-step of 64 pixels that is lost, or a split that
is added twice, moves entries by O(sqrt(64)) products -- three orders of magnitude above the bound (ratio 1131 in
test_bound_rejects_a_lost_k_step).

wgrad_plan() mirrors the host heuristic of ryolo_conv_wgrad (tile width BN, taps per CTA TG, split count), so that each
case can assert the path it covers and a change to the heuristic cannot silently drop coverage."""
import pytest
import torch

from builders import ryolo_lib
from f64_refs import CASES, U, Case, bf, gemm_sms, ref_wgrad, unpacked, wgrad, worst_ratio
from helpers import wgrad_plan

pytestmark = pytest.mark.gpu

H100_SXM_SMS = 132


def check_plan(plan, want):
    assert plan["bn"] == want["bn"] and plan["tg"] == want["tg"], (plan, want)
    assert plan["ksplit"] > 1, plan                   # every case covers the split-K path on any card
    if gemm_sms() == H100_SXM_SMS:
        for key in ("ksplit", "short_last", "last", "tiles"):
            if key in want:
                assert plan[key] == want[key], (key, plan, want)


@pytest.mark.parametrize("name", list(CASES))
def test_wgrad_vs_float64(name):
    kw, want_plan = CASES[name]
    c = Case(**kw)
    plan = c.plan()
    check_plan(plan, want_plan)
    dw = c.run(c.new_dw())
    torch.cuda.synchronize()
    want, mag = c.ref()
    r = worst_ratio(c.got(dw), want, mag, plan["n_add"])
    print("[wgrad] %s: bn %d tg %d ksplit %d (k-steps %d, %d per split, last %d) n_add %d worst |got-want|/bound %.4f"
          % (name, plan["bn"], plan["tg"], plan["ksplit"], plan["ksteps"], plan["per_split"], plan["last"], plan["n_add"], r))
    assert r <= 1.0, (name, r)
    # padding filters / channels: nothing but zeros was added to them
    full = dw.view(c.k * c.k, c.cout_pad, c.cin_pad)
    assert float(full[:, c.cout:].abs().max() if c.cout_pad > c.cout else 0.0) == 0.0
    assert float(full[:, :, c.cin:].abs().max() if c.cin_pad > c.cin else 0.0) == 0.0


def test_bound_rejects_a_lost_k_step():
    """The same bound, applied to a reference that misses ONE 64-pixel k-step (the last one of split 0), must fail on
    the kernel's output: the bound is tight enough to see a dropped or doubled k-step."""
    kw, _ = CASES["k3_c64_tg3"]
    c = Case(**kw)
    plan = c.plan()
    dw = c.run(c.new_dw())
    torch.cuda.synchronize()
    want, mag = c.ref()
    assert worst_ratio(c.got(dw), want, mag, plan["n_add"]) <= 1.0
    j = plan["per_split"] - 1
    hp, wp = c.h + 2, c.w + 2
    flat = torch.zeros(c.b * hp * wp, dtype=torch.float64, device="cuda")
    flat[64 * j:64 * (j + 1)] = 1.0
    mask = flat.view(c.b, 1, hp, wp)[:, :, 1:-1, 1:-1]
    assert float(mask.sum()) >= 32                    # the k-step lies on interior pixels
    lost, _ = ref_wgrad(c.x, c.dz * mask, c.k)
    r = worst_ratio(c.got(dw), want - lost, mag, plan["n_add"])
    print("[wgrad] reference without k-step %d: worst ratio %.1f" % (j, r))
    assert r > 1.0, r


def test_wgrad_accumulates_into_dw():
    """dw += gradient: a random prefill survives (padding entries bit-exactly), the interior is prefill + gradient"""
    kw, _ = CASES["s2d_c32_tg2"]
    kw = dict(kw, cout=48)                            # cout_pad 64 > cout: padding filters exist
    c = Case(**kw)
    plan = c.plan()
    assert plan["ksplit"] > 1
    pre = torch.randn(c.k * c.k, c.cout_pad, c.cin_pad, generator=torch.Generator().manual_seed(9)).cuda() * 50.0
    dw = c.run(c.new_dw(pre))
    torch.cuda.synchronize()
    want, mag = c.ref()
    pre_u = c.got(pre).double()
    # the final fp32 add of the prefill rounds once more: half an ulp of |prefill + gradient|
    r = worst_ratio(c.got(dw), pre_u + want, mag, plan["n_add"], extra=U * (pre_u + want).abs())
    assert r <= 1.0, r
    full, pfull = dw.view(c.k * c.k, c.cout_pad, c.cin_pad), pre.view(c.k * c.k, c.cout_pad, c.cin_pad)
    assert torch.equal(full[:, c.cout:], pfull[:, c.cout:])
    # s2d: cin = 4 * 32 = 128 = cin_pad, so the channel padding is covered by a 40 -> 64 channel case
    c2 = Case(batch=2, h=40, w=40, cin=40, cout=40, ksize=3, narrow=True, seed=3)
    assert c2.plan()["ksplit"] > 1
    pre2 = torch.randn(9, c2.cout_pad, c2.cin_pad, generator=torch.Generator().manual_seed(10)).cuda()
    dw2 = c2.run(c2.new_dw(pre2))
    torch.cuda.synchronize()
    want2, mag2 = c2.ref()
    p2 = c2.got(pre2).double()
    assert worst_ratio(c2.got(dw2), p2 + want2, mag2, c2.plan()["n_add"], extra=U * (p2 + want2).abs()) <= 1.0
    assert torch.equal(dw2[:, c2.cout:], pre2[:, c2.cout:]) and torch.equal(dw2[:, :, c2.cin:], pre2[:, :, c2.cin:])


def test_wgrad_split_counts_via_reserved_sms():
    """ryolo_set_reserved_sms shrinks the GEMM grid and with it the split count: every split count stays within the
    float64 bound, and repeated launches at one setting are bitwise equal.  The setting is process-global: restored."""
    L = ryolo_lib()
    c = Case(batch=8, h=76, w=76, cin=64, cout=64, ksize=3, seed=4)
    want, mag = c.ref()
    seen = {}
    try:
        for r in (0, 32, 60, 64):
            assert L.lib.ryolo_set_reserved_sms(r) == 0
            plan = c.plan(r)
            assert plan["tg"] == 3 and plan["ksplit"] > 1
            outs = [c.run(c.new_dw()) for _ in range(2)]
            torch.cuda.synchronize()
            assert torch.equal(outs[0], outs[1]), r
            ratio = worst_ratio(c.got(outs[0]), want, mag, plan["n_add"])
            print("[wgrad] reserved %d: %d SMs, ksplit %d, worst ratio %.4f" % (r, gemm_sms(r), plan["ksplit"], ratio))
            assert ratio <= 1.0, (r, ratio)
            seen[plan["ksplit"]] = outs[0]
        assert L.lib.ryolo_set_reserved_sms(100) != 0     # outside the documented 0..64
    finally:
        L.lib.ryolo_set_reserved_sms(0)
    if gemm_sms() == H100_SXM_SMS:
        assert sorted(seen) == [22, 24, 32, 43], sorted(seen)
    assert len(seen) >= 2


def test_wgrad_scratch_growth_and_concurrent_streams():
    """The split-K scratch is per stream and grows on demand.  small -> large (grows it) -> small on one stream without
    synchronising in between; then the same launches on two streams at once.  All results correct, and the streams'
    results bitwise equal.  High-priority streams: a pool the rest of the suite does not draw from, so the scratch of
    the first stream starts at its initial 4 MB."""
    small = Case(batch=2, h=40, w=40, cin=32, cout=32, ksize=3, narrow=True, seed=5)
    large = Case(batch=4, h=76, w=76, cin=256, cout=128, ksize=3, seed=6)     # 9 taps x 14 splits, 128 KB per CTA
    for cs in (small, large):
        assert cs.plan()["ksplit"] > 1
    sp, lp = small.plan(), large.plan()
    per_cta = lambda p: (p["tg"] * p["bn"] // 2) * 256 * 4
    assert sp["tiles"] * sp["ksplit"] * per_cta(sp) < (4 << 20) < lp["tiles"] * lp["ksplit"] * per_cta(lp)
    cur = torch.cuda.current_stream()
    s1, s2 = torch.cuda.Stream(priority=-1), torch.cuda.Stream(priority=-1)
    seq = [small, large, small]
    out1 = [cs.new_dw() for cs in seq]
    s1.wait_stream(cur)
    with torch.cuda.stream(s1):
        for cs, dw in zip(seq, out1):
            cs.run(dw, s1)
    s1.synchronize()
    s3 = torch.cuda.Stream(priority=-1)
    out_a, out_b = [cs.new_dw() for cs in seq], [cs.new_dw() for cs in seq]
    s2.wait_stream(cur)
    s3.wait_stream(cur)
    for cs, da, db in zip(seq, out_a, out_b):
        cs.run(da, s2)
        cs.run(db, s3)
    torch.cuda.synchronize()
    for cs, d1, da, db in zip(seq, out1, out_a, out_b):
        want, mag = cs.ref()
        assert worst_ratio(cs.got(d1), want, mag, cs.plan()["n_add"]) <= 1.0
        assert torch.equal(d1, da) and torch.equal(da, db)


@pytest.mark.parametrize("c_in,cout", [(32, 64), (16, 64), (64, 128)])
def test_stride2_wgrad_space_to_depth_end_to_end(c_in, cout):
    """space_to_depth(x) -> 2x2-tap wgrad at h/2 x w/2 -> unpack mode 2 == float64 gradient of the 3x3/stride-2/pad-1
    conv; the multi-tensor unpack (one job table, as the training step builds it) writes the same bits"""
    L = ryolo_lib()
    from rotate_yolov3_b200 import _lib as lm
    c = Case(batch=4 if c_in < 64 else 2, h=38, w=38, s2d_c=c_in, cout=cout, ksize=2, seed=c_in)
    plan = c.plan()
    assert plan["ksplit"] > 1
    dw = c.run(c.new_dw())
    grad = torch.full((cout, c_in, 3, 3), float("nan"), device="cuda")
    st = L.lib.ryolo_conv_unpack_wgrad(L.ptr(dw), c.cout_pad, c.cin_pad, 2, cout, c_in, 3, L.ptr(grad), L.stream_ptr())
    assert st == 0, L.last_error()
    # the multi form with a second (plain 1x1) job in the same table
    other = torch.randn(1, 64, 64, generator=torch.Generator().manual_seed(1)).cuda()
    g_multi = torch.full_like(grad, float("nan"))
    g_other = torch.full((40, 24, 1, 1), float("nan"), device="cuda")
    jobs = [lm.UnpackJob(dw.data_ptr(), g_multi.data_ptr(), c.cout_pad, c.cin_pad, 2, cout, c_in, 3),
            lm.UnpackJob(other.data_ptr(), g_other.data_ptr(), 64, 64, 0, 40, 24, 1)]
    arr = (lm.UnpackJob * 2)(*jobs)
    raw = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).cuda()
    sizes = [cout * c_in * 9, 40 * 24]
    prefix = torch.tensor([0, sizes[0], sizes[0] + sizes[1]], dtype=torch.int64).cuda()
    st = L.lib.ryolo_conv_unpack_wgrad_multi(L.ptr(raw), 2, L.ptr(prefix), sum(sizes), L.stream_ptr())
    assert st == 0, L.last_error()
    torch.cuda.synchronize()
    want, mag = ref_wgrad(c.x_full, c.dz, 3, stride=2)
    r = worst_ratio(grad, want, mag, plan["n_add"])
    print("[wgrad] s2d end to end C=%d cout=%d: ksplit %d worst ratio %.4f" % (c_in, cout, plan["ksplit"], r))
    assert r <= 1.0, r
    assert torch.equal(g_multi, grad)
    assert torch.equal(g_other.view(40, 24), other[0, :40, :24])


def test_stride2_wgrad_zero_insert_end_to_end():
    """zero_insert2x(dz) -> 3x3 wgrad at input resolution == float64 gradient of the 3x3/stride-2/pad-1 conv"""
    from rotate_yolov3_b200 import layout as Lo
    L = ryolo_lib()
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(12)
    b, cin, cout, h, w = 4, 64, 128, 76, 76
    x = bf(torch.randn(b, cin, h, w, generator=g)).to(dev)
    dz = bf(torch.randn(b, cout, h // 2, w // 2, generator=g)).to(dev)
    cin_pad, cout_pad = 64, 128
    xb = Lo.to_padded_nhwc(x, cin_pad)
    dzb = Lo.to_padded_nhwc(dz, cout_pad)
    up = Lo.alloc_padded(b, h, w, cout_pad, dev)
    st = L.lib.ryolo_zero_insert2x(L.ptr(dzb), cout_pad, b, h // 2, w // 2, cout_pad, L.ptr(up), cout_pad, h, w, L.stream_ptr())
    assert st == 0, L.last_error()
    plan = wgrad_plan(3, cin_pad, cout_pad, b, h, w, gemm_sms())
    assert plan["tg"] == 3 and plan["ksplit"] > 1
    dw = torch.zeros(9, cout_pad, cin_pad, device=dev)
    wgrad(up, cout_pad, cout_pad, xb, cin_pad, cin_pad, b, h, w, 3, dw)
    torch.cuda.synchronize()
    want, mag = ref_wgrad(x, dz, 3, stride=2)
    r = worst_ratio(unpacked(dw, 3, cout_pad, cin_pad, cout, cin), want, mag, plan["n_add"])
    print("[wgrad] zero-insert stride 2: ksplit %d worst ratio %.4f" % (plan["ksplit"], r))
    assert r <= 1.0, r


def test_wgrad_plan_mirror_is_self_consistent():
    """the mirror's split arithmetic: every split non-empty, the splits cover the k-steps exactly"""
    for ks, cin_pad, cout_pad, b, h, w in [(3, 64, 64, 4, 76, 76), (2, 256, 128, 2, 38, 38), (1, 768, 256, 2, 38, 38),
                                           (3, 512, 1024, 1, 19, 19), (3, 64, 64, 1, 8, 8)]:
        for sms in (132, 114, 72, 16):
            p = wgrad_plan(ks, cin_pad, cout_pad, b, h, w, sms)
            assert 1 <= p["last"] <= p["per_split"]
            assert (p["ksplit"] - 1) * p["per_split"] + p["last"] == p["ksteps"]
            # max_split = ceil(k-steps / 16) rounds up: a split gets at least 8 k-steps (13 in the 50-k-step cases)
            assert p["ksplit"] == 1 or p["per_split"] >= 8
