"""detect_multiscale (the batched detect.py --multi-scale) against multi_detect's per-image loop (detect.py:76-101),
restated from the package's per-image pieces on the same batched io of every size:

  per image and size: detect_postprocess_classes(io[b:b+1], conf_thres, 0.95, cap), rows in ascending keep order,
  scale_coords(...) and .round() on columns 0-3; then torch.cat over the sizes in the caller's order and
  detect_postprocess_classes(merged[None], conf_thres, nms_thres, ...) -> detections_per_image.

The package's non_max_suppression equals the reference's per-class r_nms loop (test_detect_classes_gpu.py), so this is
the reference's loop on these inputs.  Detections are compared bit for bit on random-weight models (randomised BN and
PReLU, so confidences spread), single-class and nc = 3, mixed source shapes, host and CUDA images, one to three sizes
given out of order, images silenced at one size or at every size, a threshold nothing passes, CUDA graphs on and off
and a non-default stream.  Also: a second call on CUDA images makes no synchronising call, and calls repeat bitwise."""
import numpy as np
import pytest
import torch

import helpers
from helpers import SMALL_ANCHORS
from multiscale_cases import collect  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

NMS, CAP = 0.4, 400


def _darknet(nc, seed):
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import cfgs
    m = pkg.Darknet(cfgs.yolov3_cfg(classes=nc, anchors=SMALL_ANCHORS, n_anchors=6), {"context_factor": 1.0},
                    arc="default")
    helpers.init_darknet_weights(m, seed=seed)
    return m.cuda().eval()


class Silenced(torch.nn.Module):
    """a Darknet whose io has objectness 0 for the listed (image, size) pairs: nothing of that image passes at that
    size.  Both the call under test and the restated loop run through it."""

    def __init__(self, net, silent=()):
        super().__init__()
        self.net = net
        self.silent = set(silent)

    def forward(self, x):
        io, ps = self.net(x)
        drop = [b for b, s in self.silent if s == x.shape[-1]]
        if drop:
            io = io.clone()
            io[drop, :, 5] = 0.0
        return io, ps


def _threshold(model, images, q=0.7):
    """a confidence threshold that about 30 % of the rows pass at 192 x 192 (a random-weight model's confidences sit
    wherever its biases put them)"""
    from rotate_yolov3_b200 import letterbox
    with torch.no_grad():
        img, _ = letterbox([im if isinstance(im, torch.Tensor) else torch.from_numpy(im).cuda() for im in images], 192)
        io, _ = model(img)
        score = io[..., 5] * io[..., 6:].max(-1).values
    return float(torch.quantile(score.flatten().float().cpu(), q))


def _images(seed, cuda_every=2):
    """landscape, portrait, tiny, square and odd sources; every `cuda_every`-th one a CUDA tensor"""
    g = np.random.RandomState(seed)
    shapes = [(96, 160), (200, 120), (7, 5), (64, 64), (33, 71), (150, 149)]
    out = []
    for k, (h, w) in enumerate(shapes):
        im = g.randint(0, 256, (h, w, 3)).astype(np.uint8)
        out.append(torch.from_numpy(im).cuda() if cuda_every and k % cuda_every == 1 else im)
    return out


def restated_loop(model, images, sizes, conf_thres, nms_thres, cap):
    """multi_detect per image on the batched io of each size; returns (final detections per image, merged rows per
    image)"""
    from rotate_yolov3_b200 import letterbox, scale_coords
    from rotate_yolov3_b200.nms import detect_postprocess_classes, detections_per_image
    srcs = [im if isinstance(im, torch.Tensor) else torch.from_numpy(im).cuda() for im in images]
    per_size = []
    with torch.no_grad():
        for s in sizes:
            img, _ = letterbox(srcs, s)
            io, _ = model(img)
            io = io.clone()
            rows = []
            for b, src in enumerate(srcs):
                r = detect_postprocess_classes(io[b:b + 1], conf_thres, 0.95, cap)
                k = int(r["num_keep"][0])
                det = r["dets"][0][r["keep"][0, :k]]                      # ascending keep order
                if len(det):
                    det[:, :4] = scale_coords((s, s), det[:, :4], tuple(src.shape)).round()
                rows.append(det)
            per_size.append(rows)
    finals, merged = [], []
    for b in range(len(srcs)):
        m = torch.cat([per_size[k][b] for k in range(len(sizes))], 0)
        merged.append(m)
        if len(m) == 0:
            finals.append(None)
            continue
        finals.append(detections_per_image(detect_postprocess_classes(m[None].contiguous(), conf_thres, nms_thres,
                                                                      len(m)))[0])
    return finals, merged


def _run(model, images, sizes, conf_thres, nms_thres=NMS, cap=CAP):
    from rotate_yolov3_b200 import detect_multiscale
    from rotate_yolov3_b200.nms import detections_per_image
    res = detect_multiscale(model, images, sizes, conf_thres, nms_thres, cap)
    assert res["dets"].shape == (len(images), len(sizes) * cap, 8)
    return detections_per_image(res)


def assert_same(got, want):
    assert len(got) == len(want)
    for b, (g, w) in enumerate(zip(got, want)):
        if w is None:
            assert g is None, (b, g.shape)
            continue
        assert g is not None, b
        assert g.shape == w.shape and torch.equal(g, w), (b, g.shape, w.shape)


def check(model, images, sizes, conf_thres=None, nms_thres=NMS, cap=CAP):
    if conf_thres is None:
        conf_thres = _threshold(model, images)
    got = _run(model, images, sizes, conf_thres, nms_thres, cap)
    want, merged = restated_loop(model, images, sizes, conf_thres, nms_thres, cap)
    assert_same(got, want)
    return got, merged


@pytest.mark.parametrize("sizes", [[192], [224, 160], [160, 256, 192]])
@pytest.mark.parametrize("graph", [False, True])
def test_single_class_equals_restated_loop(sizes, graph):
    net = _darknet(1, 31)
    net.use_cuda_graph = graph
    images = _images(1)
    got, merged = check(net, images, sizes)
    assert sum(g is not None for g in got) >= 4                        # detections on most images
    assert sum(len(g) for g in got if g is not None) > 20
    for g in got:
        if g is not None:                                              # nc = 1: class (1, 0), conf kept, class 0
            assert torch.all(g[:, 6] == 1.0) and torch.all(g[:, 7] == 0.0)
            assert torch.equal(g[:, :4], g[:, :4].round())            # original-image pixels, rounded


def test_multi_class_index_quirk():
    """nc = 3: the second stage takes the maximum over (class_conf, class index); a class-2 row comes out as class 1
    with its conf multiplied by 2"""
    net = _darknet(3, 32)
    got, merged = check(net, _images(2), [160, 224])
    found = 0
    for g, m in zip(got, merged):
        if g is None:
            continue
        assert set(g[:, 7].tolist()) <= {0.0, 1.0}
        for row in g[g[:, 6] == 2.0]:
            src = m[(m[:, :5] == row[:5]).all(1) & (m[:, 7] == 2.0)]
            assert len(src) >= 1
            assert row[7] == 1.0 and bool((src[:, 5] * 2.0 == row[5]).any())
            found += 1
    assert found > 0, "no class-2 detection survived: the quirk is not exercised"


def test_silenced_images_and_empty_batch():
    """an image with no survivors at one size, one with none at any size, and a threshold no row passes"""
    net = _darknet(1, 33)
    sizes = [256, 160]
    model = Silenced(net, silent=[(0, 256), (2, 160), (3, 256), (3, 160)]).eval()
    images = _images(3)
    got, merged = check(model, images, sizes)
    assert got[3] is None and len(merged[3]) == 0
    assert got[0] is not None and got[2] is not None
    got, _ = check(model, images, sizes, conf_thres=1.0)
    assert all(g is None for g in got)


def test_host_only_cuda_only_and_side_stream():
    net = _darknet(1, 34)
    host = _images(4, cuda_every=0)
    check(net, host, [224, 192])
    cuda = [torch.from_numpy(im).cuda() for im in host]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    conf = _threshold(net, cuda)
    with torch.cuda.stream(side):
        got = _run(net, cuda, [192, 224], conf)
        want, _ = restated_loop(net, cuda, [192, 224], conf, NMS, CAP)
    torch.cuda.synchronize()
    assert_same(got, want)


def test_second_call_does_not_synchronise_and_repeats():
    from rotate_yolov3_b200 import detect_multiscale
    from rotate_yolov3_b200.nms import detections_per_image
    net = _darknet(1, 35)
    images = [torch.from_numpy(im).cuda() for im in _images(5, cuda_every=0)]
    conf = _threshold(net, images)
    first = detections_per_image(detect_multiscale(net, images, [160, 224], conf, NMS, CAP))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        res = detect_multiscale(net, images, [160, 224], conf, NMS, CAP)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert_same(detections_per_image(res), first)
    for _ in range(2):
        assert_same(detections_per_image(detect_multiscale(net, images, [160, 224], conf, NMS, CAP)), first)


def test_short_last_batch():
    """a smaller batch after a full one (the last batch of an image list): a new eval pool next to the plans of the
    full batch"""
    net = _darknet(1, 36)
    images = _images(6)
    check(net, images, [224, 160])
    check(net, images[:2], [160, 224])
    check(net, images[1:], [224, 160])
