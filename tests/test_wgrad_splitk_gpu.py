"""Split-K reduction kernel and 64-filter (thin) tiles of the wgmma weight gradient (csrc/wgrad.cu).

With several splits every CTA of conv_wgrad_kernel stores its fp32 fragment and wgrad_splitk_reduce_kernel adds the
splits of each dW entry in split order; a layer with cout_pad == 64 runs thin tiles, whose two MMA warp groups split the
(tap, channel box) pairs of a stage instead of owning 64 filters each.  Checked here:
  * the float64 bound of test_wgrad_gpu.py (KAPPA * sqrt(n_add) * 2^-24 * A) on a one-tile launch with >= 100 splits, a
    two-tile launch, every thin (bn, tg) combination of the bf16 training step and of the parity-precision path
    (ryolo_px_wgrad), and the one-split direct store;
  * thin tiles against the 128-filter tiles bit for bit: the same dz / x with cout_pad 64 and cout_pad 128 (dz's
    channel stride stays 64, TMA zero-fills filters 64-127) have the same launch plan, so filters [0, 64) of dW must be
    the same bits;
  * repeated launches, and launches on two streams at once, bitwise equal."""
import ctypes

import pytest
import torch

from builders import ryolo_lib
from f64_refs import Case, gemm_sms, worst_ratio
from helpers import wgrad_plan

pytestmark = pytest.mark.gpu


def run(c, cout_pad, segmented=False, stream=None, dw=None):
    """c's launch with an explicit cout_pad (>= c.cout_pad; dz keeps its channel stride)"""
    L = ryolo_lib()
    if dw is None:
        dw = torch.zeros(c.k * c.k, cout_pad, c.cin_pad, dtype=torch.float32, device="cuda")
    fn = L.lib.ryolo_px_wgrad if segmented else L.lib.ryolo_conv_wgrad
    sp = ctypes.c_void_p(stream.cuda_stream) if stream is not None else L.stream_ptr(dw.device)
    st = fn(L.ptr(c.dzb), c.zcs, cout_pad, L.ptr(c.xb), c.xcs, c.cin_pad, c.b, c.h, c.w, c.k, L.ptr(dw), sp)
    assert st == 0, L.last_error()
    return dw


def plan(c, cout_pad=None, segmented=False):
    return wgrad_plan(c.k, c.cin_pad, cout_pad or c.cout_pad, c.b, c.h, c.w, gemm_sms(), segmented=segmented)


def check_bound(c, dw, p, tag):
    want, mag = c.ref()
    got = dw.view(c.k * c.k, -1, c.cin_pad)[:, :c.cout_pad]
    r = worst_ratio(c.got(got), want, mag, p["n_add"])
    print("[wgrad splitk] %s: bn %d tg %d tiles %d ksplit %d n_add %d worst |got-want|/bound %.4f"
          % (tag, p["bn"], p["tg"], p["tiles"], p["ksplit"], p["n_add"], r))
    assert r <= 1.0, (tag, r)


# name -> (Case kwargs, expected bn, tg, tiles)
WIDE = {
    "k1_256_128_one_tile": (dict(batch=24, h=76, w=76, cin=256, cout=128, ksize=1), (256, 1, 1)),
    "k1_384_128_two_tiles": (dict(batch=8, h=76, w=76, cin=384, cout=128, ksize=1), (256, 1, 2)),
}


@pytest.mark.parametrize("name", list(WIDE))
def test_wide_splitk_vs_float64(name):
    kw, (bn, tg, tiles) = WIDE[name]
    c = Case(**kw, seed=21)
    p = c.plan()
    assert (p["bn"], p["tg"], p["tiles"]) == (bn, tg, tiles), p
    if tiles == 1:
        assert p["ksplit"] >= min(100, gemm_sms()), p
    else:
        assert p["ksplit"] > 1, p
    check_bound(c, run(c, c.cout_pad), p, name)


# thin (cout_pad 64) launches: name -> (Case kwargs, segmented, expected bn, tg).  bf16 path: the training step's 608^2
# s2d 32 -> 64 (128, 2), 304^2 3x3 32 -> 64 (64, 3), 152^2 1x1 128 -> 64 (128, 1), 304^2 1x1 64 -> 32 (64, 1).
# Parity path: (128, 1), (64, 2) and (64, 1), the last with one (tap, box) pair, so warp group 2 idles.
THIN = {
    "bf16_s2d_c32": (dict(batch=4, h=38, w=38, s2d_c=32, cout=64, ksize=2), False, (128, 2)),
    "bf16_k3_c32": (dict(batch=4, h=76, w=76, cin=32, cout=64, ksize=3, narrow=True), False, (64, 3)),
    "bf16_k1_c128": (dict(batch=8, h=76, w=76, cin=128, cout=64, ksize=1), False, (128, 1)),
    "bf16_k1_c64_cout32": (dict(batch=8, h=76, w=76, cin=64, cout=32, ksize=1, narrow=True), False, (64, 1)),
    "seg_k1_c128": (dict(batch=4, h=76, w=76, cin=128, cout=64, ksize=1), True, (128, 1)),
    "seg_s2d_c16": (dict(batch=4, h=38, w=38, s2d_c=16, cout=64, ksize=2), True, (64, 2)),
    "seg_k3_c64": (dict(batch=2, h=76, w=76, cin=64, cout=48, ksize=3), True, (64, 1)),
}


@pytest.mark.parametrize("name", list(THIN))
def test_thin_vs_float64_and_full_tile(name):
    kw, seg, (bn, tg) = THIN[name]
    c = Case(**kw, seed=len(name))
    assert c.cout_pad == 64
    p = plan(c, segmented=seg)
    assert (p["bn"], p["tg"]) == (bn, tg) and p["ksplit"] > 1, p
    assert plan(c, 128, segmented=seg) == p          # m_tiles = 1 either way: the same launch plan
    thin = run(c, 64, seg)
    full = run(c, 128, seg)
    torch.cuda.synchronize()
    check_bound(c, thin, p, name)
    assert torch.equal(thin, full[:, :64]), name
    assert float(full[:, 64:].abs().max()) == 0.0     # zero-filled filters add nothing


@pytest.mark.parametrize("seg", [False, True])
@pytest.mark.parametrize("cout", [64, 128])
def test_single_split_direct_store(cout, seg):
    """ksplit == 1: the CTA adds its fragment to dW itself (no partials, no reduce launch)"""
    c = Case(batch=1, h=8, w=8, cin=64, cout=cout, ksize=3, seed=cout + seg)
    p = plan(c, segmented=seg)
    assert p["ksplit"] == 1, p
    dw = run(c, c.cout_pad, seg)
    torch.cuda.synchronize()
    check_bound(c, dw, p, "ksplit1 cout %d seg %d" % (cout, seg))
    if cout == 64:
        assert torch.equal(dw, run(c, 128, seg)[:, :64])


def test_repeated_and_concurrent_launches_bitwise():
    """the same launches repeated, then on two streams at once (each with its own scratch): the same bits.  A wide
    launch with 100+ splits and a thin one, so both reduce instantiations run while the other stream writes partials."""
    cases = [Case(**WIDE["k1_256_128_one_tile"][0], seed=31), Case(**THIN["bf16_s2d_c32"][0], seed=32)]
    ref = [run(c, c.cout_pad) for c in cases]
    again = [run(c, c.cout_pad) for c in cases]
    torch.cuda.synchronize()
    for a, b in zip(ref, again):
        assert torch.equal(a, b)
    cur = torch.cuda.current_stream()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs1 = [torch.zeros_like(r) for r in ref]
    outs2 = [torch.zeros_like(r) for r in ref]
    s1.wait_stream(cur)
    s2.wait_stream(cur)
    for _ in range(3):
        for c, o1, o2 in zip(cases, outs1, outs2):
            o1.zero_(), o2.zero_()
            s1.wait_stream(cur), s2.wait_stream(cur)
            run(c, c.cout_pad, stream=s1, dw=o1)
            run(c, c.cout_pad, stream=s2, dw=o2)
        torch.cuda.synchronize()
        for r, o1, o2 in zip(ref, outs1, outs2):
            assert torch.equal(r, o1) and torch.equal(r, o2)
    check_bound(cases[0], ref[0], cases[0].plan(), "wide, repeated")
