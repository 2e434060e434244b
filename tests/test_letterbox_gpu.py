"""The device letterbox (ryolo_letterbox via rotate_yolov3_b200.letterbox) against the reference's own letterbox and
LoadImages normalisation (tests/golden/letterbox_golden.npz): the fp32 and fp16 network input is bit for bit the
reference's for every case; border pixels, mixed-size batches, CUDA sources, CUDA-graph replay, scale_coords,
letterbox_labels, malformed input, and a Darknet forward on the device input against one on the reference input."""
import os

import numpy as np
import pytest
import torch

from builders import tensor_sha
from helpers import GOLDEN
from letterbox_cases import letterbox_case, net_input, source

pytestmark = pytest.mark.gpu

GOLD = os.path.join(GOLDEN, "letterbox_golden.npz")
DEV = torch.device("cuda", 0)


def _gold():
    return np.load(GOLD)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_every_case_bitwise_equals_reference(dtype):
    from rotate_yolov3_b200 import letterbox
    g = _gold()
    key = "sha32" if dtype == torch.float32 else "sha16"
    for name in g["cases"]:
        img, new_shape, mode, k = letterbox_case(g, str(name))
        x, meta = letterbox([img], new_shape, mode=mode, dtype=dtype, device=DEV)
        torch.cuda.synchronize()
        assert x.dtype == dtype and tuple(x.shape[2:]) == tuple(int(v) for v in g[k + "out_hw"])
        assert meta.dtype == torch.float64 and meta[0].tolist() == g[k + "meta"].tolist(), name
        if k + "lb" in g:                          # where the reference image is stored: count differing pixels
            want = torch.from_numpy(net_input(g[k + "lb"], np.float32 if dtype == torch.float32 else np.float16))
            ndiff = int((x[0].cpu() != want).sum())
            assert ndiff == 0, "%s: %d of %d values differ from the reference input" % (name, ndiff, want.numel())
        assert tensor_sha(x[0]) == str(g[k + key]), name


def test_border_is_exactly_128_over_255():
    from rotate_yolov3_b200 import letterbox
    img = source(5, 767, 1024)                      # 455 rows: top 76, bottom 77
    x, _ = letterbox([img], 608)
    grey = np.float32(128) / np.float32(255)
    assert (x[0, :, :76] == float(grey)).all() and (x[0, :, 76 + 455:] == float(grey)).all()
    assert not (x[0, :, 76] == float(grey)).all() and not (x[0, :, 76 + 454] == float(grey)).all()
    x16, _ = letterbox([img], 608, dtype=torch.float16)
    assert (x16[0, :, :76] == torch.tensor(grey).half().item()).all()


def test_mixed_batch_equals_single_calls_and_cuda_sources():
    from rotate_yolov3_b200 import letterbox
    g = _gold()
    names = ["land_1024x768", "hd_1920x1080", "int2x2", "upscale", "no_resize", "one_px_wide", "half_pad", "portrait"]
    imgs = [letterbox_case(g, n)[0] for n in names]
    batch, meta = letterbox(imgs, 608)
    for b, img in enumerate(imgs):
        one, m1 = letterbox([img], 608)
        assert torch.equal(batch[b], one[0]) and torch.equal(meta[b], m1[0])
    dev_imgs = [torch.from_numpy(im).to(DEV) for im in imgs]
    on_dev, meta2 = letterbox(dev_imgs, 608)
    assert torch.equal(on_dev, batch) and torch.equal(meta2, meta)
    # a CUDA source with padded rows (a crop of a wider buffer) reads with its row stride
    wide = torch.from_numpy(source(9, 768, 1100)).to(DEV)
    crop, _ = letterbox([wide[:, :1024]], 608)
    ref, _ = letterbox([np.ascontiguousarray(wide[:, :1024].cpu().numpy())], 608)
    assert torch.equal(crop, ref)
    # host tensors are accepted like arrays
    t, _ = letterbox([torch.from_numpy(imgs[0])], 608)
    assert torch.equal(t[0], batch[0])


def test_cuda_graph_replay_with_out():
    from rotate_yolov3_b200 import letterbox
    imgs = [torch.from_numpy(source(s, h, w)).to(DEV) for s, (h, w) in enumerate([(768, 1024), (1080, 1920), (300, 400)])]
    want, _ = letterbox(imgs, 608)
    out = torch.empty_like(want)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        letterbox(imgs, 608, out=out)              # uploads the job table, kept with `out`
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        letterbox(imgs, 608, out=out)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    for im, s in zip(imgs, (11, 12, 13)):          # replay reads the sources where they are
        im.copy_(torch.from_numpy(source(s, *im.shape[:2])))
    graph.replay()
    want2, _ = letterbox([im.cpu().numpy() for im in imgs], 608)
    torch.cuda.synchronize()
    assert torch.equal(out, want2)
    with pytest.raises(RuntimeError):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            letterbox([imgs[0]], 608, out=torch.empty_like(want[:1]))   # no warm-up call: no job table to replay


def test_scale_coords_matches_reference():
    from rotate_yolov3_b200 import scale_coords
    g = _gold()
    batch_in, batch_shapes, batch_want = [], [], []
    for i in range(5):
        c = torch.from_numpy(g["sc_%d_in" % i]).to(DEV)
        img1, img0 = (tuple(int(v) for v in s) for s in g["sc_%d_shapes" % i])
        got = scale_coords(img1, c[:, :4], img0 + (3,))
        assert torch.equal(got.cpu(), torch.from_numpy(g["sc_%d_out" % i])), i
        assert torch.equal(c[:, 4].cpu(), torch.from_numpy(g["sc_%d_in" % i][:, 4]))
        if img1 == (608, 608):
            batch_in.append(g["sc_%d_in" % i])
            batch_shapes.append(img0)
            batch_want.append(g["sc_%d_out" % i])
    dets = torch.from_numpy(np.stack(batch_in)).to(DEV)
    scale_coords((608, 608), dets, batch_shapes)   # batched, in place on columns 0-3
    assert torch.equal(dets[..., :4].cpu(), torch.from_numpy(np.stack(batch_want)))


def test_letterbox_labels_matches_reference():
    from rotate_yolov3_b200 import letterbox_labels
    g = _gold()
    lab_in, lab_out, shapes, metas = g["lab_in"], g["lab_out"], g["lab_shapes"], g["lab_meta"]
    for out_hw in {tuple(int(v) for v in s[2:]) for s in shapes}:
        sel = [i for i, s in enumerate(shapes) if tuple(int(v) for v in s[2:]) == out_hw]
        rows = [np.concatenate([np.full((len(lab_in[i]), 1), b, np.float32), lab_in[i]], 1) for b, i in enumerate(sel)]
        labels = torch.from_numpy(np.concatenate(rows)).to(DEV)
        got = letterbox_labels(labels, torch.from_numpy(metas[sel]), [tuple(int(v) for v in shapes[i][:2]) for i in sel],
                               out_hw)
        assert torch.equal(got[:, 0], labels[:, 0])
        assert torch.equal(got[:, 1:].cpu(), torch.from_numpy(np.concatenate([lab_out[i] for i in sel])))


def test_malformed_input_raises():
    from rotate_yolov3_b200 import letterbox
    img = source(0, 40, 50)
    with pytest.raises(ValueError):
        letterbox([], 608)
    with pytest.raises(ValueError):
        letterbox([img.astype(np.float32)], 608)
    with pytest.raises(ValueError):
        letterbox([img[:, :, :2]], 608)
    with pytest.raises(ValueError):
        letterbox([np.zeros((40, 50, 4), np.uint8)], 608)
    with pytest.raises(ValueError):
        letterbox([torch.from_numpy(img).to(DEV).float()], 608)
    with pytest.raises(ValueError):
        letterbox([img], 608, mode="rect")
    with pytest.raises(ValueError):
        letterbox([img], 608, out=torch.empty(1, 3, 608, 600, device=DEV))
    with pytest.raises(RuntimeError):
        letterbox([img], 608, device="cpu")


def test_darknet_io_on_device_input_equals_reference_input():
    """the device input is the reference's input bit for bit, so Darknet's eval io on it is too"""
    import helpers
    import rotate_yolov3_b200 as pkg
    g = _gold()
    img, new_shape, mode, k = letterbox_case(g, "e2e")            # 97 x 133 -> 128 x 128
    x, _ = pkg.letterbox([img], new_shape)
    ref = torch.from_numpy(net_input(g[k + "lb"], np.float32)).unsqueeze(0).to(DEV)
    m = pkg.Darknet(helpers.mini_cfg(128, 128), {"context_factor": 1.0}, arc="default")
    helpers.init_darknet_weights(m, seed=77)
    m = m.to(DEV).eval()
    with torch.no_grad():
        io_dev = m(x)[0].clone()
        io_ref = m(ref)[0].clone()
    assert torch.equal(x, ref)
    assert torch.equal(io_dev.view(torch.int32), io_ref.view(torch.int32))
