"""The mAP evaluation on the device: metrics.match_batch (ryolo_match_batched) and metrics.Evaluator (ryolo_match_batched +
ryolo_ap_per_class), against test.py's loop restated over the per-image path (nms.detections_per_image, per-image
metrics.match_detections) and the numpy ap_per_class that tests/test_ap_cpu.py checks against the reference.

Batches of 608x608 images with nc in {1, 3}: detections are built around the targets -- close copies (matches), looser
ones (near-misses, and second matches of a target another detection already claimed), copies in the wrong class,
duplicate targets, background boxes, images without targets and images without detections; the targets are shuffled
across images."""
import math

import numpy as np
import pytest
import torch

import helpers
from ap_numpy import ap_per_class

pytestmark = pytest.mark.gpu

HW = (608, 608)


def make_batch(seed, bsz, nc, conf_thres, cap, background=300):
    """(detect_postprocess_classes result, targets [nt, 7] on the device)"""
    from rotate_yolov3_b200.nms import detect_postprocess_classes
    g = torch.Generator().manual_seed(seed)
    rand = lambda *s: torch.rand(*s, generator=g)
    rows_io, tgts = [], []
    for b in range(bsz):
        nt = 0 if b % 4 == 1 else int(torch.randint(1, 7, (1,), generator=g))
        boxes = helpers.gen_boxes(nt, seed * 100 + b, 500.0)
        boxes[:, :2] += 54.0
        cls = torch.randint(0, nc, (nt,), generator=g).float()
        if nt >= 2 and b % 3 == 0:                        # a duplicate target, same class
            boxes[1], cls[1] = boxes[0], cls[0]
        for k in range(nt):
            x, y = boxes[k, 0] / HW[1], boxes[k, 1] / HW[0]
            w, h = boxes[k, 2] / HW[1], boxes[k, 3] / HW[0]
            tgts.append([b, float(cls[k]), x, y, w, h, float(boxes[k, 4])])
        dets = []
        if b % 4 != 2:                                    # images 2, 6, ...: no detections
            for k in range(nt):
                for jit in (0.02, 0.05, 0.12, 0.25):
                    d = boxes[k].clone()
                    d[:2] += jit * d[2:4].max() * (rand(2) - 0.5)
                    d[2:4] *= 1 + jit * (rand(2) - 0.5)
                    d[4] += jit * (rand(1)[0] - 0.5)
                    c = int(cls[k]) if rand(1)[0] < 0.85 else int(torch.randint(0, nc, (1,), generator=g))
                    dets.append((d, c))
            bg = helpers.gen_boxes(background, seed * 1000 + b, 608.0)
            dets += [(bg[k], int(torch.randint(0, nc, (1,), generator=g))) for k in range(background)]
        io = torch.zeros(max(len(dets), 1), 6 + nc)
        for k, (d, c) in enumerate(dets):
            io[k, :5] = d
            io[k, 5] = 0.002 + 0.99 * rand(1)[0]
            io[k, 6:] = 0.5 * rand(nc)
            io[k, 6 + c] = 0.6 + 0.4 * rand(1)[0]
        rows_io.append(io)
    p = max(len(x) for x in rows_io)
    io = torch.stack([torch.cat([x, torch.zeros(p - len(x), 6 + nc)]) for x in rows_io]).cuda()
    res = detect_postprocess_classes(io, conf_thres, 0.7, cap)
    t = torch.tensor(tgts, dtype=torch.float32).reshape(-1, 7)
    t = torch.cat([t, torch.tensor([[bsz + 3.0, 0, 0.5, 0.5, 0.1, 0.1, 0.0]])])   # an image index past the batch
    t = t[torch.randperm(len(t), generator=g)]
    return res, t.cuda()


def per_image(res, targets, hw, iou_thres=0.5):
    """test.py:95-151 over the per-image path: per image (correct, conf, cls, tcls, ious)"""
    from rotate_yolov3_b200.metrics import match_detections_device
    from rotate_yolov3_b200.nms import detections_per_image
    from rotate_yolov3_b200.iou import rotated_iou_matrix
    out = []
    for si, pred in enumerate(detections_per_image(res)):
        labels = targets[targets[:, 0] == si, 1:]
        tbox = labels[:, 1:6].clone()
        tbox[:, [0, 2]] *= hw[1]
        tbox[:, [1, 3]] *= hw[0]
        if pred is None:
            out.append((None, None, None, labels[:, 0].cpu().numpy(), None))
            continue
        correct = match_detections_device(pred, tbox, labels[:, 0], iou_thres)
        iou = rotated_iou_matrix(pred[:, :5].contiguous(), tbox) if len(labels) else None
        out.append((correct, pred[:, 5], pred[:, 7], labels[:, 0].cpu().numpy(), iou))
    return out


def bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("nc", [1, 3])
@pytest.mark.parametrize("conf_thres,cap", [(0.3, 2000), (0.001, 20000), (0.5, 3)])
def test_match_batch_equals_per_image_path(nc, conf_thres, cap):
    from rotate_yolov3_b200.metrics import match_batch
    res, targets = make_batch(7 + nc, 8, nc, conf_thres, cap)
    got = match_batch(res, targets, HW)
    ref = per_image(res, targets, HW)
    n = int(got["count"])
    assert n == int(res["num_keep"].sum())
    timg = targets[:, 0].cpu()
    off, tstart, n_correct, n_claim_lost = 0, 0, 0, 0
    for b, (correct, conf, cls, tcls, iou) in enumerate(ref):
        t_b = int((timg == b).sum())
        if correct is not None:
            k = len(correct)
            assert torch.equal(got["correct"][off:off + k], correct), b
            assert torch.equal(bits(got["conf"][off:off + k]), bits(conf)), b
            assert torch.equal(bits(got["cls"][off:off + k]), bits(cls)), b
            if iou is not None:
                blk = got["iou"][cap * tstart:cap * tstart + k * t_b].view(k, t_b)
                assert torch.equal(bits(blk), bits(iou)), b
                best = iou.max(1).values > 0.5
                n_claim_lost += int((best & (correct == 0)).sum())
            n_correct += int(correct.sum())
            off += k
        tstart += t_b
    assert off == n
    if cap > 3:
        assert n_correct > 0 and n_claim_lost > 0      # matches, and overlaps > iou_thres that found their target taken


def restated_test_loop(batches, nc, iou_thres=0.5):
    """test.py:80-157 with the per-image path: stats per image, then ap_per_class and the per-class target count"""
    stats, seen = [], 0
    for res, targets, hw in batches:
        for correct, conf, cls, tcls, _ in per_image(res, targets, hw, iou_thres):
            seen += 1
            if correct is None:
                if len(tcls):
                    stats.append((np.zeros(0), np.zeros(0, np.float32), np.zeros(0, np.float32), tcls))
                continue
            stats.append((correct.cpu().numpy().astype(np.float64), conf.cpu().numpy(), cls.cpu().numpy(), tcls))
    stats = [np.concatenate(x, 0) for x in zip(*stats)]
    p, r, ap, f1, ap_class = ap_per_class(*stats)
    return p, r, ap, f1, ap_class, np.bincount(stats[3].astype(np.int64), minlength=nc), seen


def run_evaluator(batches, nc):
    from rotate_yolov3_b200.metrics import Evaluator
    ev = Evaluator(nc, 0.5, device="cuda")
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for res, targets, hw in batches:
            ev.add(res, targets, hw)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    return ev.compute(), ev


def check_against_reference(got, want):
    p, r, ap, f1, cls, nt, seen = got
    wp, wr, wap, wf1, wcls, wnt, wseen = want
    assert np.array_equal(cls, wcls) and np.array_equal(nt, wnt) and seen == wseen
    for a, b in ((p, wp), (r, wr), (f1, wf1)):
        assert np.array_equal(a.view(np.int64), np.asarray(b, np.float64).view(np.int64)), (a, b)
    assert np.all(np.abs(ap - wap) <= 1e-12 * np.abs(wap)), (ap, wap)


@pytest.mark.parametrize("nc", [1, 3])
def test_evaluator_equals_test_loop(nc):
    batches = [(*make_batch(31 + nc, 8, nc, 0.3, 2000), HW),
               (*make_batch(41 + nc, 8, nc, 0.001, 20000), HW),
               (*make_batch(51 + nc, 5, nc, 0.5, 40), HW)]
    got, ev = run_evaluator(batches, nc)
    want = restated_test_loop(batches, nc)
    check_against_reference(got, want)
    assert got[6] == 21 and len(got[4]) >= 1 and got[2].max() > 0
    again, ev2 = run_evaluator(batches, nc)
    for a, b in zip(got[:6], again[:6]):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
    assert torch.equal(ev._count, ev2._count)
    n = int(ev._count)
    for name in ("_correct", "_conf", "_cls"):
        assert torch.equal(getattr(ev, name)[:n], getattr(ev2, name)[:n]), name


def test_evaluator_edge_cases():
    """no adds; a batch whose images have no targets; a target class outside [0, nc) is refused"""
    from rotate_yolov3_b200.metrics import Evaluator
    p, r, ap, f1, cls, nt, seen = Evaluator(2, device="cuda").compute()
    assert len(p) == len(cls) == 0 and seen == 0 and np.array_equal(nt, [0, 0])
    res, _ = make_batch(3, 4, 2, 0.3, 500)
    ev = Evaluator(2, device="cuda")
    ev.add(res, torch.zeros(0, 7, device="cuda"), HW)
    p, r, ap, f1, cls, nt, seen = ev.compute()
    assert len(cls) == 0 and seen == 4 and int(ev._count) == int(res["num_keep"].sum()) > 0
    res, targets = make_batch(4, 4, 2, 0.3, 500)
    ev = Evaluator(1, device="cuda")
    targets[:, 1] = 1.0
    ev.add(res, targets, HW)
    with pytest.raises(ValueError):
        ev.compute()


def test_end_to_end_small_darknet():
    """letterbox -> eval forward of a small Darknet -> detect_postprocess_classes -> Evaluator, against the loop"""
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200.nms import detect_postprocess_classes
    model = pkg.Darknet(helpers.mini_cfg(64, 64), {"context_factor": 1.0}, arc="default")
    helpers.init_darknet_weights(model, seed=5)
    model = model.cuda().eval()
    rng = np.random.default_rng(9)
    batches = []
    for bi in range(2):
        shapes = [(48, 80), (96, 64), (64, 64)]
        imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shapes]
        x, meta = pkg.letterbox(imgs, 64)
        labels = []
        for i in range(len(imgs)):
            for _ in range(int(rng.integers(0, 4))):
                labels.append([i, 0, *rng.uniform(0.2, 0.8, 2), *rng.uniform(0.1, 0.4, 2), rng.uniform(-1, 1)])
        labels = torch.tensor(labels, dtype=torch.float32).reshape(-1, 7)
        targets = pkg.letterbox_labels(labels, meta, shapes, x.shape[2:]).cuda()
        with torch.no_grad():
            io, _ = model(x)
        res = detect_postprocess_classes(io.float().contiguous(), 0.001, 0.5, 300)
        batches.append((res, targets, tuple(x.shape[2:])))
    got, _ = run_evaluator(batches, 1)
    check_against_reference(got, restated_test_loop(batches, 1))
    assert got[6] == 6
