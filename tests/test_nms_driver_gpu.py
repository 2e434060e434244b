"""non_max_suppression / nms_filter / yolo decode against fixtures produced by the reference's own Python code
(tests/golden/make_golden.py)."""
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN

pytestmark = pytest.mark.gpu


def test_non_max_suppression_vs_reference_driver():
    import rotate_yolov3_b200 as pkg
    g = np.load(os.path.join(GOLDEN, "nms_driver_golden.npz"))
    pred = torch.from_numpy(g["pred"]).cuda()
    out = pkg.non_max_suppression(pred, conf_thres=float(g["conf_thres"]), nms_thres=float(g["nms_thres"]))
    assert len(out) == 3
    for i in range(3):
        if bool(g["none_%d" % i]):
            assert out[i] is None
        else:
            assert out[i].shape == g["out_%d" % i].shape
            assert np.array_equal(out[i].cpu().numpy(), g["out_%d" % i])     # rows are copies: bit-exact
    # the in-place side effect pred[:, 5] *= class_conf (nms.py:35)
    assert np.array_equal(pred.cpu().numpy(), g["pred_after"], equal_nan=True)
    pred1 = torch.from_numpy(g["pred1"]).cuda()
    out1 = pkg.non_max_suppression(pred1, 0.5, 0.5)
    for i in range(2):
        assert np.array_equal(out1[i].cpu().numpy(), g["out1_%d" % i])


def _same_bits(a, b):
    """bit-identical, except that any NaN equals any NaN (payloads are not part of IEEE arithmetic's result)"""
    nan = torch.isnan(a)
    return torch.equal(nan, torch.isnan(b)) and torch.equal(a.view(torch.int32)[~nan], b.view(torch.int32)[~nan])


def test_filter_large_and_empty():
    import helpers
    import rotate_yolov3_b200 as pkg
    g = torch.Generator().manual_seed(0)
    p = torch.rand(100003, 7, generator=g)
    p[:, 2:4] *= 10
    p[::7, 5] = 0.0
    # the uniform rows above, then rows at the filter's edges: conf on and next to 4096-bin edges and the threshold,
    # w / h == min_wh, NaN / +-inf in every column in turn, tied class maxima
    inputs = [(p, 0.25)] + [(helpers.filter_edge_rows(nc, 0.5, 2.0, seed=11), 0.5) for nc in (1, 3)]
    for p, conf_thres in inputs:
        ref = p.clone()
        cc, ci = ref[:, 6:].max(1)
        ref[:, 5] *= cc
        keep = (ref[:, 5] > conf_thres) & (ref[:, 2:4] > 2).all(1) & torch.isfinite(ref).all(1)
        want = torch.cat([ref[keep][:, :6], cc[keep, None], ci[keep, None].float()], 1)
        pc = p.cuda()
        got = pkg.nms_filter(pc, conf_thres, 2.0)
        assert _same_bits(got.cpu(), want)
        assert _same_bits(pc.cpu(), ref)
    none = pkg.non_max_suppression(torch.zeros(2, 10, 7, device="cuda"), 0.5, 0.5)
    assert none == [None, None]


@pytest.mark.parametrize("tag", ["a", "b"])
def test_yolo_decode_vs_reference_layer(tag):
    import ctypes
    import rotate_yolov3_b200 as pkg
    g = np.load(os.path.join(GOLDEN, "decode_golden.npz"))
    p = torch.from_numpy(g["p_" + tag]).cuda()
    nc = int(g["nc_" + tag])
    anchors = torch.from_numpy(g["anchors"]).float().cuda()
    bs, _, ny, nx = p.shape
    na = anchors.shape[0]
    rows = na * ny * nx
    io = torch.full((bs, rows + 10, nc + 6), -7.0, device="cuda")
    pp = torch.empty((bs, na, ny, nx, nc + 6), device="cuda")
    st = pkg._lib.lib.ryolo_yolo_decode(pkg._lib.ptr(p), bs, na, nc, ny, nx, pkg._lib.ptr(anchors),
                                        float(g["stride_" + tag]), float(g["ctx_" + tag]), 1, pkg._lib.ptr(io),
                                        rows + 10, 4, pkg._lib.ptr(pp), pkg._lib.stream_ptr())
    assert st == 0
    got = io[:, 4:4 + rows].cpu().numpy()
    want = g["io_" + tag]
    assert np.allclose(got, want, rtol=1e-4, atol=1e-5), float(np.abs(got - want).max())
    assert np.array_equal(pp.cpu().numpy(), g["pp_" + tag])
    assert float(io[:, :4].min()) == -7.0 and float(io[:, 4 + rows:].max()) == -7.0   # row_offset respected
