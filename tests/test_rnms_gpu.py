"""GPU parity of ryolo_rnms (through the Python boundary -> C-ABI) with the reference.

Tiers: (1) the reference kernel itself, compiled by nvcc with its default flags and run on an H100 on the seeded inputs
below (tests/golden/rnms_kernel_golden.npz, written by tests/golden/make_golden_rnms_kernel.py) -- the suppression MASK
must match bit-for-bit on every word the reference scan reads, and the kept-index tensor must be identical; (2) the CPU
oracle (both arithmetic variants) and the committed golden keep lists; (3) properties at the full 20k size."""
import ctypes
import os

import numpy as np
import pytest
import torch

import helpers
from helpers import GOLDEN, P, adversarial_dets, gen_dets, orc_rnms

pytestmark = pytest.mark.gpu

_KERNEL_GOLDEN = {}


def _kernel_golden(key):
    """the reference kernel's answer for one seeded case"""
    if not _KERNEL_GOLDEN:
        _KERNEL_GOLDEN.update(np.load(os.path.join(GOLDEN, "rnms_kernel_golden.npz")))
    return _KERNEL_GOLDEN[key]


def _case(*a):
    return "_".join(str(x).replace(".", "p").replace("-", "m") for x in a)


def _ours(dets, thr):
    import rotate_yolov3_b200 as pkg
    return pkg.r_nms(dets.cuda(), thr)


def _upper_words(mask, n):
    """zero the words the reference scan never reads (column block < row block)"""
    cb = (n + 63) // 64
    rb = (torch.arange(n, device=mask.device) // 64)[:, None]
    col = torch.arange(cb, device=mask.device)[None, :]
    return torch.where(col >= rb, mask, torch.zeros_like(mask))


@pytest.mark.parametrize("n,canvas,thr", [(1, 100, 0.5), (63, 60, 0.3), (64, 60, 0.3), (65, 60, 0.3), (500, 120, 0.1),
                                          (3000, 300, 0.5), (5000, 608, 0.3)])
def test_mask_and_keep_bit_identical_to_reference_kernel(n, canvas, thr):
    import rotate_yolov3_b200 as pkg
    dets = gen_dets(n, 100 + n, float(canvas))
    keep, boxes, order, mask = pkg.nms.rnms_debug(dets.cuda(), thr)
    # our sort is the stable descending sort the oracle uses
    want_order = np.argsort(-dets[:, 5].numpy(), kind="stable")
    assert np.array_equal(order.cpu().numpy(), want_order)
    assert torch.equal(boxes.cpu(), dets[torch.from_numpy(want_order)])
    # reference kernel on the same sorted boxes
    ref_mask = torch.from_numpy(_kernel_golden("mask_" + _case(n, canvas, thr)))
    assert torch.equal(_upper_words(mask, n).cpu(), ref_mask)
    assert np.array_equal(keep.cpu().numpy(), _kernel_golden("keep_" + _case(n, canvas, thr)))


@pytest.mark.parametrize("thr", [0.0, 0.1, 0.3, 0.5, 0.7])
def test_adversarial_inputs_vs_reference_kernel(thr):
    """duplicates, collinear neighbours, touching edges, concentric, zero-area and NaN boxes.

    Contract boundary: the reference stores candidate points in int_pts[16] = 8 points with no bounds check
    (rotate_polygon_nms_kernel.cu:235, 162-194); a pair that yields MORE than 8 candidates makes the reference
    itself overflow its stack buffer (undefined behaviour), so such pairs are excluded from bit-parity and must be
    the ONLY mask bits that differ (here: a box against its own zero-width copy, 10 candidates)."""
    import rotate_yolov3_b200 as pkg
    from helpers import oracle
    dets = adversarial_dets()
    n = len(dets)
    keep, boxes, order, mask = pkg.nms.rnms_debug(dets.cuda(), thr)
    m1 = _upper_words(mask, n).cpu().numpy().view(np.uint64)
    m2 = _kernel_golden("adv_mask_" + _case(thr)).view(np.uint64)
    bx = boxes.cpu().numpy()
    orc = oracle()
    ndiff = 0
    for i, w in zip(*np.nonzero(m1 != m2)):
        x = int(m1[i, w] ^ m2[i, w])
        for bit in range(64):
            if (x >> bit) & 1:
                j = w * 64 + bit
                if j <= i:
                    continue                      # diagonal-tile bits at or below the diagonal are never read
                orc.orc_ref_iou_fma(P(np.ascontiguousarray(bx[i])), P(np.ascontiguousarray(bx[j])))
                npts = ctypes.c_int.in_dll(orc, "orc_last_npts_fma").value
                assert npts > 8, ("mask bit (%d,%d) differs on a pair inside the contract" % (i, j), bx[i], bx[j])
                ndiff += 1
    assert ndiff <= 2


def test_negative_threshold_matches_reference():
    """thr < 0: even disjoint pairs satisfy IoU(=0) > thr; the pre-filter must switch itself off."""
    dets = gen_dets(300, 9, 2000.0)
    assert np.array_equal(_ours(dets, -0.5).cpu().numpy(), _kernel_golden("neg_keep"))
    assert len(_ours(dets, -0.5)) == 1


@pytest.mark.parametrize("thr", [0.1, 0.3, 0.5])
def test_golden_keep_lists(thr):
    g = np.load(os.path.join(GOLDEN, "rnms_ref_golden.npz"))
    got = _ours(torch.from_numpy(g["dets"]), thr).cpu().numpy()
    assert np.array_equal(got, g["keep_%02d" % int(thr * 10)])


def test_wrapper_fixture():
    g = np.load(os.path.join(GOLDEN, "rnms_ref_golden.npz"))
    out = _ours(torch.from_numpy(g["fixture"]), 0.1)
    assert out.dtype == torch.int64 and out.is_cuda
    assert out.cpu().tolist() == [0, 3]   # utils/nms/nms_wrapper_test.py:35-43, analytic answer


@pytest.mark.parametrize("n,canvas", [(2000, 250.0), (4000, 608.0), (3000, 60.0)])
def test_vs_cpu_oracle(n, canvas):
    """r_nms (lazy chunked mask) vs the CPU oracle; the 60-px canvas is a dense set where most boxes are suppressed early"""
    dets = gen_dets(n, 77 + n, canvas)
    got = _ours(dets, 0.5).cpu().numpy()
    assert np.array_equal(got, orc_rnms(dets.numpy(), 0.5, variant=1))
    assert np.array_equal(got, orc_rnms(dets.numpy(), 0.5, variant=0))


@pytest.mark.parametrize("n,canvas,thr", [(5000, 100.0, 0.3), (20000, 300.0, 0.5), (2500, 608.0, 0.1)])
def test_lazy_chunked_equals_full_mask_and_reference(n, canvas, thr):
    """the production path skips rows/columns suppressed by earlier 1024-box chunks; the kept list must not change"""
    import rotate_yolov3_b200 as pkg
    dets = gen_dets(n, 31 + n, canvas)
    lazy = _ours(dets, thr).cpu().numpy()
    full = pkg.nms.rnms_debug(dets.cuda(), thr)[0].cpu().numpy()
    assert np.array_equal(lazy, full)
    assert np.array_equal(lazy, _kernel_golden("lazy_keep_" + _case(n, canvas, thr)))


def test_reference_boundary_behaviour():
    import rotate_yolov3_b200 as pkg
    empty = pkg.r_nms(torch.zeros((0, 6), device="cuda"), 0.5)
    assert empty.device.type == "cpu" and empty.dtype == torch.int64 and empty.numel() == 0  # rotate_polygon_nms.cpp:9-10
    with pytest.raises(RuntimeError):
        pkg.r_nms(torch.zeros((3, 6)), 0.5)
    one = pkg.r_nms(torch.tensor([[5.0, 5, 4, 2, 0.1, 0.9]], device="cuda"), 0.5)
    assert one.tolist() == [0]
    # non-contiguous / wider input is accepted like dc[:, :6] in nms.py:64
    wide = torch.cat([gen_dets(200, 5, 80.0), torch.rand(200, 2)], 1).cuda()
    assert torch.equal(pkg.r_nms(wide[:, :6], 0.3), pkg.r_nms(wide[:, :6].contiguous(), 0.3))


def test_full_size_config3_properties():
    """BASELINE config 3: 20k boxes, thr 0.5.  Parity with the reference kernel, and properties."""
    import rotate_yolov3_b200 as pkg
    n, thr = 20000, 0.5
    dets = gen_dets(n, 2, 608.0)
    keep = _ours(dets, thr)
    k = keep.cpu().numpy()
    assert np.all(np.diff(k) > 0) and k.min() >= 0 and k.max() < n           # ascending original indices
    assert k[0] <= int(torch.argmax(dets[:, 5])) <= k[-1] and int(torch.argmax(dets[:, 5])) in set(k.tolist())
    # idempotence: NMS of the kept set keeps everything
    again = _ours(dets[keep.cpu()], thr)
    assert len(again) == len(k)
    # every kept pair has IoU <= thr under the fp64 oracle semantics is NOT implied (different algorithm), so use
    # the reference kernel for exactness
    assert np.array_equal(k, _kernel_golden("full_keep"))
    assert 7000 < len(k) < 10000  # SURVEY.md 6: K = 8666 for this distribution


def test_batched_segments_equal_single_problem_nms():
    """ryolo_rnms_batched: S independent problems with device-side counts in one set of launches -> per segment the kept
    list equals r_nms on that segment's rows (which is bit-identical to the reference kernel, tests above); includes empty,
    single-box, ragged and full segments, and `limit` < count (only the best-scored boxes enter the NMS)."""
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200.nms import r_nms_batched
    dev = torch.device("cuda")
    cap = 3000
    counts = [0, 1, 100, 1777, 3000, 2500]
    dets = torch.zeros((len(counts), cap, 6))
    for s, n in enumerate(counts):
        if n:
            dets[s, :n] = helpers.gen_dets(n, 50 + s, 300.0)
        dets[s, n:] = float("nan")                      # rows beyond the count must never be read
    dets = dets.to(dev)
    cnt = torch.tensor(counts, dtype=torch.int32, device=dev)
    for thr in (0.1, 0.5):
        keep, num = r_nms_batched(dets, cnt, thr)
        for s, n in enumerate(counts):
            got = keep[s, :int(num[s])].cpu()
            want = pkg.r_nms(dets[s, :n], thr).cpu() if n else torch.empty(0, dtype=torch.long)
            assert torch.equal(got, want), (thr, s, n, len(got), len(want))
    # limit: the top-`limit` boxes by score (stable) enter the NMS; kept indices still refer to the segment's rows
    limit = 1000
    keep, num = r_nms_batched(dets, cnt, 0.3, limit=limit)
    for s, n in enumerate(counts):
        got = keep[s, :int(num[s])].cpu()
        if n == 0:
            assert len(got) == 0
            continue
        sub = dets[s, :n]
        top = torch.argsort(sub[:, 5], descending=True, stable=True)[:limit]
        top_sorted = torch.sort(top).values
        want = top_sorted[pkg.r_nms(sub[top_sorted], 0.3)].cpu()
        assert torch.equal(got, want), (s, n, len(got), len(want))


def test_detect_select_and_batched_postprocess_equal_per_image_pipeline():
    """device-side candidate selection (exact top-cap) + segmented NMS == the per-image pipeline (nms_filter -> stable
    top-cap by confidence -> r_nms), image by image: one image with more candidates than the cap, one with fewer, one
    with none.  The bench's own detect shape runs the same comparison in test_detect_gpu.py."""
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(5)
    B, P, cap = 3, 40000, 1500
    io = torch.zeros(B, P, 7)
    for b in range(B):
        io[b, :, :5] = helpers.gen_boxes(P, 70 + b, 608.0)
    io[..., 5] = torch.rand(B, P, generator=g)
    io[..., 6] = 1.0
    io[1, :, 5] *= 0.02                         # image with fewer candidates than the cap
    io[1, :300, 5] = 0.6 + 0.3 * torch.rand(300, generator=g)
    io[0, :50, 2] = 1.0                         # too small -> filtered
    io[0, 50:60, 0] = float("nan")              # non-finite -> filtered
    io[2, :, 5] = 0.001                         # nothing above the threshold
    confs = helpers.check_postprocess_equals_per_image(io.to(dev), 0.5, 0.4, cap)
    assert [len(c) > cap for c in confs] == [True, False, False] and len(confs[2]) == 0
