"""Detection post-processing after the forward pass: ryolo_yolo_decode -> ryolo_detect_select -> ryolo_rnms_batched,
joined by nms.detect_postprocess.

* detect_select against an exact top-k restatement of utils/nms/nms.py:34-40 on the CPU, bit for bit, on the inputs
  where a confidence histogram goes wrong: thousands of rows in one bin ahead of more confident rows, all rows tied,
  confidences on bin edges, the filter's strict comparisons, non-finite values, and the CTA / block edges of P.
* detect_postprocess against the per-image pipeline (nms_filter -> stable top-k -> r_nms), including the bench's own
  detect shape: 32 images of 608x608 through a random-init yolov3.
* ryolo_yolo_decode against a float64 restatement of model/models.py:198-227 at the three 608x608 heads, batch 32."""
import pytest
import torch

import helpers
from f64_refs import decode_ref, yolov3_heads

pytestmark = pytest.mark.gpu

MIN_WH = 2.0


def _bits(t):
    return t.contiguous().view(torch.int32)


def ref_select(io_b, conf_thres, limit, min_wh=MIN_WH):
    """utils/nms/nms.py:34-40 on one image [P, 6+nc] (CPU): conf = obj * max(cls) as one fp32 multiply, the strict
    filter, then the `limit` largest conf by a stable sort (ties: lowest row index), back in input order.
    Returns the rows (x, y, w, h, theta, conf) [k, 6] and the number of rows passing the filter."""
    conf = io_b[:, 5] * io_b[:, 6:].max(1).values
    keep = (conf > conf_thres) & (io_b[:, 2] > min_wh) & (io_b[:, 3] > min_wh) & torch.isfinite(io_b).all(1) \
        & torch.isfinite(conf)
    idx = torch.nonzero(keep).flatten()
    top = idx[torch.argsort(-conf[idx], stable=True)[:limit]]
    sel = torch.sort(top).values
    return torch.cat([io_b[sel, :5], conf[sel, None]], 1), len(idx)


def check_select(io, conf_thres, limit, tag):
    from rotate_yolov3_b200.nms import detect_select
    dets, counts = detect_select(io.cuda(), conf_thres, limit)
    dets, counts = dets.cpu(), counts.cpu()
    for b in range(io.shape[0]):
        want, n_pass = ref_select(io[b], conf_thres, limit)
        n = int(counts[b])
        got = dets[b, :min(n, dets.shape[1])]
        if not (n == len(want) and torch.equal(_bits(got), _bits(want))):
            have = set(map(tuple, _bits(got).tolist()))
            missing = sum(1 for r in _bits(want).tolist() if tuple(r) not in have)
            pytest.fail("%s, image %d, limit %d: %d of the reference's %d rows missing; count %d, want %d "
                        "(%d rows pass the filter)" % (tag, b, limit, missing, len(want), n, len(want), n_pass))
        assert n == min(limit, n_pass)
    assert dets.shape == (io.shape[0], limit, 6)


def _image(conf, nc=1, seed=0):
    """one decoded image [P, 6+nc] with the given confidences (obj = conf, class score 1.0) and valid boxes"""
    p = len(conf)
    g = torch.Generator().manual_seed(seed)
    io = torch.zeros(p, 6 + nc)
    io[:, :5] = helpers.gen_boxes(p, 40 + seed, 608.0)
    io[:, 2:4] = 3.0 + 60.0 * torch.rand(p, 2, generator=g)
    io[:, 5] = conf
    io[:, 6:] = 0.999 * torch.rand(p, nc, generator=g)
    io[:, 6] = 1.0
    return io


def _dense_bin_late_high():
    """3500 rows in one 1/4096-wide bin (0.70001 / 0.70002) ahead, in input order, of 500 rows at 0.9"""
    conf = torch.full((40000,), 0.1)
    conf[:3000] = 0.70001
    conf[30000:30500] = 0.70002
    conf[39000:39500] = 0.9
    return conf


def _stack(*imgs):
    return torch.stack(imgs).contiguous()


def case_dense_bin():
    a = _image(_dense_bin_late_high(), seed=1)
    b = a[torch.randperm(len(a), generator=torch.Generator().manual_seed(2))]   # shuffled variant
    return _stack(a, b), [1000, 1]


def case_all_tied():
    g = torch.Generator().manual_seed(3)
    imgs = []
    for v in (0.75, 1.0, float(torch.nextafter(torch.tensor(0.5), torch.tensor(1.0)))):
        conf = torch.full((40000,), v)
        conf[torch.rand(40000, generator=g) < 0.3] = 0.2
        imgs.append(_image(conf, seed=len(imgs) + 4))
    return _stack(*imgs), [1, 1000, 20000, 27999, 28000, 28001]


def case_edges(nc):
    a = helpers.filter_edge_rows(nc, 0.5, MIN_WH, seed=11)
    b = helpers.filter_edge_rows(nc, 0.5, MIN_WH, seed=12)
    n = min(len(a), len(b))
    return _stack(a[:n], b[:n].flip(0)), [1, 700, 701, 2000, 5000, n]


def case_quantised():
    """scores on a 1/64 grid above the threshold, more rows at 1.0 than the limit in one image"""
    g = torch.Generator().manual_seed(21)
    c0 = torch.randint(0, 65, (40000,), generator=g).float() / 64
    c1 = c0.clone()
    c1[torch.rand(40000, generator=g) < 0.2] = 1.0
    return _stack(_image(c0, seed=22), _image(c1, seed=23)), [1, 3000, 9000]


def case_nothing_passes():
    a = _image(torch.full((9000,), 0.5), seed=30)                 # conf == conf_thres everywhere
    b = _image(torch.rand(9000, generator=torch.Generator().manual_seed(31)), seed=32)
    b[:, 3] = MIN_WH                                              # h == min_wh everywhere
    return _stack(a, b), [1, 5000]


CASES = {
    "dense_bin_late_high": case_dense_bin,
    "all_tied": case_all_tied,
    "bin_edges_strict_nonfinite_nc1": lambda: case_edges(1),
    "bin_edges_strict_nonfinite_nc3": lambda: case_edges(3),
    "quantised": case_quantised,
    "nothing_passes": case_nothing_passes,
}


@pytest.mark.parametrize("case", list(CASES))
def test_detect_select_exact_top_limit(case):
    io, limits = CASES[case]()
    for limit in limits:
        check_select(io, 0.5, limit, case)


@pytest.mark.parametrize("p", [1, 255, 256, 257, 8191, 8192, 8193, 40000])
def test_detect_select_exact_at_block_edges(p):
    """P at the 256-row block and 8192-rows-per-CTA edges; limit in {1, n_pass - 1, n_pass, n_pass + 1, > P} for the
    pass counts of two differently drawn images (uniform and 1/8-quantised confidences), plus one image with none"""
    g = torch.Generator().manual_seed(p)
    a = _image(torch.rand(p, generator=g), seed=50)
    b = _image(torch.randint(0, 9, (p,), generator=g).float() / 8, seed=51)
    c = _image(torch.full((p,), 0.25), seed=52)
    io = _stack(a, b, c)
    limits = {1, p + 7}
    for img in (a, b):
        n = ref_select(img, 0.5, p + 1)[1]
        limits |= {n - 1, n, n + 1}
    for limit in sorted(x for x in limits if x >= 1):
        check_select(io, 0.5, limit, "P=%d" % p)


def test_detect_select_rejects_negative_or_nan_threshold():
    from rotate_yolov3_b200.nms import detect_select
    io = _image(torch.rand(300, generator=torch.Generator().manual_seed(9)), seed=9)[None].cuda()
    for bad in (-0.25, -1e-30, float("nan")):
        with pytest.raises(RuntimeError, match="status -1"):
            detect_select(io, bad, 10)
    check_select(io.cpu(), 0.0, 10, "conf_thres=0")
    check_select(io.cpu(), -0.0, 10, "conf_thres=-0")


def test_detect_postprocess_rejects_multi_class():
    from rotate_yolov3_b200.nms import detect_postprocess
    io = torch.rand(2, 100, 9, device="cuda")
    with pytest.raises(ValueError, match="non_max_suppression"):
        detect_postprocess(io, 0.5, 0.5, 50)


# ---------------------------------------------------------------------------------------------------------------------
# detect_postprocess == the per-image pipeline
# ---------------------------------------------------------------------------------------------------------------------
def _dense_ties_io():
    """3 images of 40 000 rows whose candidates share few confidence values: the dense bin ahead of late high rows,
    scores on a 1/64 grid, and one image where every candidate ties -- the NMS order then rests on the row index"""
    g = torch.Generator().manual_seed(6)
    c1 = torch.randint(0, 65, (40000,), generator=g).float() / 64
    c2 = torch.where(torch.rand(40000, generator=g) < 0.4, torch.tensor(0.75), torch.tensor(0.25))
    io = _stack(_image(_dense_bin_late_high(), seed=60), _image(c1, seed=61), _image(c2, seed=62))
    return io.cuda(), 0.5, 0.4, 3000


def _bench_detect_io():
    """bench.py's detect workload (BASELINE configs[4]): random-init yolov3 in eval mode on 32 images of 608x608"""
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import cfgs
    model = pkg.Darknet(cfgs.yolov3_cfg(), {"context_factor": 1.0}, arc="default")
    helpers.init_darknet_weights(model, seed=1)
    model = model.cuda().eval()
    x = torch.rand(32, 3, 608, 608, generator=torch.Generator().manual_seed(0)).cuda()
    with torch.no_grad():
        io, _ = model(x)
    del model
    return io, 0.5, 0.5, 20000


def _parent_threshold_bin(conf, cap):
    """the 4096-bin linear histogram the selection used before it was exact: (threshold bin, its population, rows at
    or above it)"""
    h = torch.bincount((conf * 4096).long().clamp(max=4095), minlength=4096)
    suffix = h.flip(0).cumsum(0).flip(0)
    reach = torch.nonzero(suffix >= cap).flatten()
    t = int(reach[-1]) if len(reach) else 0
    return t, int(h[t]), int(suffix[t])


@pytest.mark.parametrize("inputs", ["dense_ties", "bench_detect"])
def test_detect_postprocess_equals_per_image_pipeline(inputs):
    """detect_postprocess == the per-image pipeline (nms_filter -> stable top-cap -> rows back in input order -> r_nms),
    bit for bit.  At the bench's detect shape, also print each image's population of the threshold bin of the
    4096-bin histogram the selection used before it was exact (it kept up to 2048 surplus rows)."""
    io, conf_thres, nms_thres, cap = _dense_ties_io() if inputs == "dense_ties" else _bench_detect_io()
    confs = helpers.check_postprocess_equals_per_image(io, conf_thres, nms_thres, cap, MIN_WH)
    if inputs == "bench_detect":
        worst = 0
        for b, conf in enumerate(confs):
            t, pop, at_or_above = _parent_threshold_bin(conf, cap)
            worst = max(worst, pop)
            print("image %2d: %6d candidates, threshold bin %4d holds %5d rows, %6d rows at or above it"
                  % (b, len(conf), t, pop, at_or_above))
        print("largest threshold-bin population of the 4096-bin histogram: %d (slack was 2048)" % worst)


# ---------------------------------------------------------------------------------------------------------------------
# ryolo_yolo_decode against float64
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nc", [1, 3])
@pytest.mark.parametrize("ctx", [1.0, 1.25])
def test_yolo_decode_vs_float64_at_608_heads(nc, ctx):
    """all three heads of a 608x608 yolov3 (72 anchors, grids 19/38/76) decoded into one [32, 545 832 + sentinels,
    6+nc] buffer through row_offset; nc = 1 runs the shared-memory staged kernel, nc = 3 the direct one.
    |got - want| <= 2^-20 * M per component, M = the sum of the magnitudes of the terms; p_out bit-exact."""
    import rotate_yolov3_b200 as pkg
    heads = yolov3_heads(nc)
    bs, no, pad = 32, nc + 6, 37
    rows = sum(a.shape[0] * ng * ng for a, ng, _ in heads)
    assert rows == 545832
    io = torch.full((bs, pad + rows + pad, no), 0x7FC0DEAD, dtype=torch.int32, device="cuda").view(torch.float32)
    g = torch.Generator(device="cuda").manual_seed(nc * 10 + int(ctx * 4))
    off = pad
    worst = 0.0
    for anchors, ng, stride in heads:
        na = anchors.shape[0]
        p = (torch.rand(bs, na * no, ng, ng, generator=g, device="cuda") * 2 - 1) * 15
        pp = torch.empty(bs, na, ng, ng, no, device="cuda")
        anc = anchors.cuda()
        st = pkg._lib.lib.ryolo_yolo_decode(pkg._lib.ptr(p), bs, na, nc, ng, ng, pkg._lib.ptr(anc), float(stride),
                                            float(ctx), 1, pkg._lib.ptr(io), pad + rows + pad, off, pkg._lib.ptr(pp),
                                            pkg._lib.stream_ptr())
        assert st == 0
        assert torch.equal(pp, p.view(bs, na, no, ng, ng).permute(0, 1, 3, 4, 2)), (ng, "p_out")
        want, mag = decode_ref(p, anchors, stride, ctx, nc)
        got = io[:, off:off + na * ng * ng].double()
        ratio = (got - want).abs() / (mag * 2.0 ** -20)
        ratio = torch.where(got == want, torch.zeros_like(ratio), ratio)   # M == 0 only where want == 0 exactly
        r = float(ratio.max())
        assert r <= 1.0, (ng, r, [float(ratio[..., k].max()) for k in range(no)])
        if nc == 1:
            assert bool((io[:, off:off + na * ng * ng, 6] == 1.0).all())
        worst = max(worst, r)
        off += na * ng * ng
        del p, pp, want, mag, got, ratio
    assert off == pad + rows
    assert torch.equal(_bits(io[:, :pad]), torch.full((bs, pad, no), 0x7FC0DEAD, dtype=torch.int32, device="cuda"))
    assert torch.equal(_bits(io[:, pad + rows:]),
                       torch.full((bs, pad, no), 0x7FC0DEAD, dtype=torch.int32, device="cuda"))
    print("nc %d ctx %.2f: worst |got - want| / (2^-20 M) = %.3f" % (nc, ctx, worst))
