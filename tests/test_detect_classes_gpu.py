"""Class-aware batched post-processing: nms.detect_postprocess_classes (ryolo_detect_select_classes ->
ryolo_rnms_batched_classes) and nms.detections_per_image.

* Against the reference's own non_max_suppression output (tests/golden/nms_driver_golden.npz), bit for bit.
* Against the per-image per-class pipeline (nms_filter -> stable top-cap by confidence -> rows back in input order ->
  r_nms on each class's rows), bit for bit, on inputs built to break a class-sorted segment: identical boxes in
  different classes, class runs straddling the 64-box blocks, empty classes, tied confidences and class scores,
  non-finite class scores, a cap that cuts across classes, images where nothing passes -- and at the bench's detect
  shape (32 images of 608x608 through a random-init yolov3 with 3 classes).
* Repeatability, and each image's result equals its batch-of-one result."""
import os

import numpy as np
import pytest
import torch

import helpers
from builders import check_equals_per_class_pipeline, postprocess_classes

pytestmark = pytest.mark.gpu


def _image(nc, cls, conf, seed, canvas=200.0):
    """one decoded image [P, 6+nc]: boxes of the bench generator on a small canvas (dense overlaps), objectness `conf`,
    class scores below 0.9 except 0.95 at the class `cls` of each row"""
    p = len(cls)
    g = torch.Generator().manual_seed(seed)
    io = torch.zeros(p, 6 + nc)
    io[:, :5] = helpers.gen_boxes(p, 100 + seed, canvas)
    io[:, 5] = conf
    io[:, 6:] = 0.9 * torch.rand(p, nc, generator=g)
    io[torch.arange(p), 6 + cls] = 0.95
    return io


def _rand_conf(p, seed):
    return 0.3 + 0.7 * torch.rand(p, generator=torch.Generator().manual_seed(seed))


def _shuffle(io, seed):
    return io[torch.randperm(len(io), generator=torch.Generator().manual_seed(seed))]


def case_identical_across_classes(nc):
    """every box appears once per class with the same confidence: within a class the boxes lie on a 500-pixel grid
    (longest side < 400), so all are kept; a class-agnostic NMS would keep one copy per box"""
    boxes = helpers.gen_boxes(40, 5, 4000.0)
    boxes[:, 0] = 250.0 + 500.0 * (torch.arange(40) % 8)
    boxes[:, 1] = 250.0 + 500.0 * (torch.arange(40) // 8)
    rows = []
    for c in range(nc):
        r = _image(nc, torch.full((40,), c), 0.8, seed=c)
        r[:, :5] = boxes
        rows.append(r)
    return torch.cat(rows)


def case_runs(nc):
    """class runs of 1, 63, 64, 65, 127, 129 candidates (the classes spread over all nc), each straddling 64-box
    blocks of the class-sorted segment"""
    runs = [1, 63, 64, 65, 127, 129]
    cls = torch.cat([torch.full((k,), (i * 5) % nc) for i, k in enumerate(runs)])
    return _shuffle(_image(nc, cls, _rand_conf(len(cls), 7), seed=8), 9)


def case_single_class(nc):
    """every candidate in class nc - 1 (all other classes empty)"""
    return _image(nc, torch.full((700,), nc - 1), _rand_conf(700, 10), seed=11)


def case_all_tied(nc):
    """every confidence equal, within a class and across classes: the order rests on (class, row)"""
    g = torch.Generator().manual_seed(12)
    return _image(nc, torch.randint(0, nc, (900,), generator=g), 0.75, seed=13)


def case_tied_class_scores(nc):
    """the maximum class score shared by two classes (the first wins), plus NaN / +-inf class scores (the row fails
    the filter)"""
    g = torch.Generator().manual_seed(14)
    io = _image(nc, torch.randint(0, nc, (800,), generator=g), _rand_conf(800, 15), seed=16)
    io[:300, 6 + nc - 1] = io[:300, 6:].max(1).values
    io[100:200, 6] = io[100:200, 6:].max(1).values
    for k, bad in enumerate((float("nan"), float("inf"), -float("inf"))):
        io[300 + 20 * k:320 + 20 * k, 6 + (k % nc)] = bad
    return io


def case_mixed(nc, p=1500, seed=20, canvas=300.0):
    g = torch.Generator().manual_seed(seed)
    return _image(nc, torch.randint(0, nc, (p,), generator=g), _rand_conf(p, seed + 1), seed=seed + 2, canvas=canvas)


def case_nothing_passes(nc):
    io = case_mixed(nc, 500, 30)
    io[:, 5] = 0.25
    return io


CASES = {
    "identical_across_classes": case_identical_across_classes,
    "runs_across_blocks": case_runs,
    "single_class": case_single_class,
    "all_tied": case_all_tied,
    "tied_and_nonfinite_class_scores": case_tied_class_scores,
}


def _batch(*imgs):
    p = max(len(x) for x in imgs)
    out = []
    for x in imgs:   # pad with rows that fail the filter (objectness 0)
        pad = torch.zeros(p - len(x), x.shape[1])
        out.append(torch.cat([x, pad]))
    return torch.stack(out).contiguous().cuda()


@pytest.mark.parametrize("nc", [2, 3, 15])
@pytest.mark.parametrize("case", list(CASES))
def test_equals_per_class_pipeline(case, nc):
    """each case next to an image where nothing passes and a mixed image; a cap above every count and caps that cut
    across classes"""
    io = _batch(CASES[case](nc), case_nothing_passes(nc), case_mixed(nc))
    for cap in (2000, 130, 64, 1):
        res, kept = check_equals_per_class_pipeline(io, 0.5, 0.4, cap)
        assert int(res["num_keep"][1]) == 0 and int(res["counts"][1]) == 0
        if case == "identical_across_classes" and cap == 2000:
            assert int(res["num_keep"][0]) == 40 * nc


def test_reference_driver_golden():
    """detections_per_image(detect_postprocess_classes(...)) == the reference's non_max_suppression, bit for bit"""
    from rotate_yolov3_b200.nms import detections_per_image
    g = np.load(os.path.join(helpers.GOLDEN, "nms_driver_golden.npz"))
    pred = torch.from_numpy(g["pred"]).cuda()
    before = pred.clone()
    out = detections_per_image(postprocess_classes(pred, float(g["conf_thres"]), float(g["nms_thres"]), 600))
    assert len(out) == 3
    for i in range(3):
        if bool(g["none_%d" % i]):
            assert out[i] is None
        else:
            assert np.array_equal(out[i].cpu().numpy(), g["out_%d" % i]), i
    assert torch.equal(pred.view(torch.int32), before.view(torch.int32))     # io is not modified
    pred1 = torch.from_numpy(g["pred1"]).cuda()
    out1 = detections_per_image(postprocess_classes(pred1, 0.5, 0.5, 600))
    for i in range(2):
        assert np.array_equal(out1[i].cpu().numpy(), g["out1_%d" % i]), i


def test_detections_per_image_order():
    """confidence descending, ties by class ascending, then by input row; None for an image with nothing kept"""
    from rotate_yolov3_b200.nms import detections_per_image
    io = _batch(case_all_tied(3), case_nothing_passes(3), case_mixed(3))
    res = postprocess_classes(io, 0.5, 0.4, 2000)
    out = detections_per_image(res)
    assert out[1] is None
    for b in (0, 2):
        k = int(res["num_keep"][b])
        rows = res["dets"][b][res["keep"][b, :k]].cpu()
        key = sorted(range(k), key=lambda i: (-float(rows[i, 5]), float(rows[i, 7]), i))
        assert torch.equal(out[b].cpu(), rows[key])


def _bench_io(nc):
    """bench.py's detect shape through a random-init yolov3 with nc classes: 32 images of 608x608, eval mode"""
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import cfgs
    model = pkg.Darknet(cfgs.yolov3_cfg(classes=nc), {"context_factor": 1.0}, arc="default")
    helpers.init_darknet_weights(model, seed=1)
    model = model.cuda().eval()
    x = torch.rand(32, 3, 608, 608, generator=torch.Generator().manual_seed(0)).cuda()
    with torch.no_grad():
        io, _ = model(x)
    del model
    return io


def test_bench_shape_three_classes():
    io = _bench_io(3)
    before = io.clone()
    res, kept = check_equals_per_class_pipeline(io, 0.5, 0.5, 20000)
    assert torch.equal(io.view(torch.int32), before.view(torch.int32))
    print("yolov3 nc=3, 32 x 608^2: %d candidates selected, %d kept"
          % (int(res["counts"].sum()), kept))


def test_bench_shape_single_class_equals_detect_postprocess():
    from rotate_yolov3_b200.nms import detect_postprocess
    io = _bench_io(1)
    res = postprocess_classes(io, 0.5, 0.5, 20000)
    ref = detect_postprocess(io, 0.5, 0.5, 20000)
    assert torch.equal(res["counts"], ref["counts"])
    for b in range(io.shape[0]):
        n = int(ref["counts"][b])
        assert torch.equal(res["dets"][b, :n, :6], ref["dets"][b, :n]), b
        assert torch.equal(res["dets"][b, :n, 7], torch.zeros(n, device=io.device)), b
    assert torch.equal(res["num_keep"], ref["num_keep"])
    for b in range(io.shape[0]):
        k = int(ref["num_keep"][b])
        assert torch.equal(res["keep"][b, :k], ref["keep"][b, :k]), b


def test_repeatable_and_independent_of_batch():
    io = _batch(case_runs(15), case_mixed(15, 3000, 40, 608.0), case_nothing_passes(15), case_all_tied(15))
    for cap in (2000, 100):
        a = postprocess_classes(io, 0.5, 0.4, cap)
        b = postprocess_classes(io, 0.5, 0.4, cap)
        for key in ("counts", "num_keep"):
            assert torch.equal(a[key], b[key]), key
        for i in range(io.shape[0]):
            n, k = int(a["counts"][i]), int(a["num_keep"][i])
            assert torch.equal(a["dets"][i, :n].view(torch.int32), b["dets"][i, :n].view(torch.int32))
            assert torch.equal(a["keep"][i, :k], b["keep"][i, :k])
            one = postprocess_classes(io[i:i + 1].contiguous(), 0.5, 0.4, cap)
            assert int(one["counts"][0]) == n and int(one["num_keep"][0]) == k
            assert torch.equal(one["dets"][0, :n].view(torch.int32), a["dets"][i, :n].view(torch.int32))
            assert torch.equal(one["keep"][0, :k], a["keep"][i, :k])
