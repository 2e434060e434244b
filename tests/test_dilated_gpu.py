"""The multi-branch dilated graph (cfg/yolov3-m.cfg) on the GPU, eval mode: the phase-layout kernels bit for bit, every
dilated launch of the eval forward against float64 of its own inputs, and the whole forward against the REFERENCE
model's output (tests/golden/darknet_m_golden.npz, make_golden_m.py).

A dilated 3x3 conv runs as ryolo_dilate_split -> ordinary pad-1 3x3 conv_bn_act_fwd on the B*dh*dw phase images ->
ryolo_dilate_merge (+ the shortcut that follows it).  Each launch is re-run on the tensors the forward left in the plan,
and checked on its own: the split and the merge bit for bit against the index map of phase_split, the conv with
the bound of test_detect_forward_f64_gpu.py (E = n 2^-23 A, n = taps * cin_pad / 16; |got - want| <= 2^-8 (|want| + E)
+ E; no bias, activation or residual terms: the branch convs have none)."""
import ctypes
import json

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from builders import DILATIONS, golden_text, m_golden, m_model, phase_merge, phase_split, ryolo_lib
from helpers import init_darknet_weights

pytestmark = pytest.mark.gpu


def _padded(t, cs):
    from rotate_yolov3_b200 import layout as L
    return L.to_padded_nhwc(t, cs)


def _nchw(buf, c):
    from rotate_yolov3_b200 import layout as L
    return L.from_padded_nhwc(buf, c)


def _split(x, xcs, b, h, w, c, dh, dw, xp):
    lib = ryolo_lib()
    st = lib.lib.ryolo_dilate_split(ctypes.c_void_p(x), xcs, b, h, w, c, dh, dw, lib.ptr(xp), xp.shape[-1],
                                    lib.stream_ptr(xp.device))
    lib.check(st, "ryolo_dilate_split")


def _merge(yp, b, h, w, c, dh, dw, r, rcs, acc, y, ycs):
    lib = ryolo_lib()
    st = lib.lib.ryolo_dilate_merge(lib.ptr(yp), yp.shape[-1], b, h, w, c, dh, dw, ctypes.c_void_p(r) if r else None, rcs,
                                    acc, ctypes.c_void_p(y), ycs, lib.stream_ptr(yp.device))
    lib.check(st, "ryolo_dilate_merge")


@pytest.mark.parametrize("dil", DILATIONS)
def test_split_and_merge_bit_exact(dil):
    from rotate_yolov3_b200 import layout as L
    dh, dw = dil
    g = torch.Generator(device="cuda").manual_seed(dh * 100 + dw)
    for b, h, w, c, xcs in ((2, 13, 13, 64, 64), (3, 19, 26, 40, 64), (1, 52, 38, 256, 264)):
        x = torch.randn(b, c, h, w, device="cuda", generator=g).bfloat16().float()
        xb = _padded(x, xcs)
        hp, wp = -(-h // dh), -(-w // dw)
        xp = torch.full((b * dh * dw, hp + 2, wp + 2, c + 8), float("nan"), dtype=torch.bfloat16, device="cuda")
        xp[:, 0], xp[:, -1], xp[:, :, 0], xp[:, :, -1] = 0, 0, 0, 0
        _split(xb.data_ptr(), xcs, b, h, w, c, dh, dw, xp)
        torch.cuda.synchronize()
        assert torch.equal(_nchw(xp, c), phase_split(x, dh, dw))          # zero fill included
        assert bool((xp[:, 0] == 0).all() and (xp[:, :, -1] == 0).all())   # halo untouched
        assert bool(xp[:, 1:-1, 1:-1, c:].float().isnan().all())          # channels beyond c untouched
        # merge: plain, + residual, + residual + accumulate; fp32 sums in that order, one bf16 rounding
        p = torch.randn(b * dh * dw, c, hp, wp, device="cuda", generator=g).bfloat16().float()
        r = torch.randn(b, c, h, w, device="cuda", generator=g).bfloat16().float()
        y0 = torch.randn(b, c, h, w, device="cuda", generator=g).bfloat16().float()
        pb, rb = _padded(p, c), _padded(r, xcs)
        gathered = phase_merge(p, b, h, w, dh, dw)
        for res, acc, want in ((False, 0, gathered), (True, 0, gathered + r), (True, 1, gathered + r + y0)):
            yb = _padded(y0, xcs)
            _merge(pb, b, h, w, c, dh, dw, rb.data_ptr() if res else None, xcs, acc, yb.data_ptr(), xcs)
            torch.cuda.synchronize()
            assert torch.equal(_nchw(yb, c), want.bfloat16().float()), (res, acc)
            assert bool((yb[:, 0] == 0).all() and (yb[:, :, 0] == 0).all())
            assert bool((yb[..., c:] == 0).all())


def _dilated_steps(plan):
    steps = plan["steps"]
    return [(steps[k][1], steps[k + 1][1], steps[k + 2][1]) for k in range(len(steps)) if steps[k][0] == "dsplit"]


def test_every_dilated_launch_vs_float64_at_416():
    from rotate_yolov3_b200 import layout as L
    m = init_darknet_weights(m_model(), seed=21).cuda().eval()
    b = 8
    x = torch.rand(b, 3, 416, 416, device="cuda", generator=torch.Generator(device="cuda").manual_seed(22))
    with torch.no_grad():
        m(x)
    torch.cuda.synchronize()
    launches = _dilated_steps(m._plan)
    assert len(launches) == 36
    owners = {i: int(d["weight_from"]) for i, d in enumerate(m.module_defs) if "weight_from" in d}
    dconvs = [i for i, d in enumerate(m.module_defs) if d["type"] == "d-convolutional"]
    worst = 0.0
    for i, (sp, cv, mg) in zip(dconvs, launches):
        dh, dw = sp["dh"], sp["dw"]
        h, w, c = sp["h"], sp["w"], sp["c"]
        src = sp["keep"]
        xin = _nchw(src.buf, src.ch_off + c)[:, src.ch_off:].double()
        _split(sp["x"], sp["xcs"], b, h, w, c, dh, dw, sp["xp"])
        L.conv_fwd(cv["desc"], cv["x"], cv["w"], cv["b"], cv["y"], None, x.device)
        torch.cuda.synchronize()
        yp = _nchw(mg["yp"], mg["c"])
        wt = m.module_list[owners[i]].Conv2d.weight.detach().bfloat16().double()
        want = F.conv2d(xin, wt, padding=(dh, dw), dilation=(dh, dw))
        a = F.conv2d(xin.abs(), wt.abs(), padding=(dh, dw), dilation=(dh, dw))
        got = phase_merge(yp, b, h, w, dh, dw).double()
        e = 9 * L.round_up(c, 64) / 16 * 2.0 ** -23 * a
        bound = 2.0 ** -8 * (want.abs() + e) + e
        ratio = float(((got - want).abs() / bound).max())
        worst = max(worst, ratio)
        assert ratio <= 1.0, (i, dh, dw, ratio)
        # the merge the forward ran: the gathered conv output (+ the shortcut source), one rounding
        out = mg["keep"][1]
        want_out = phase_merge(yp, b, h, w, dh, dw)
        if mg["r"]:
            res = mg["keep"][0]
            want_out = want_out + _nchw(res.buf, res.ch_off + mg["c"])[:, res.ch_off:]
        assert torch.equal(_nchw(out.buf, out.ch_off + mg["c"])[:, out.ch_off:], want_out.bfloat16().float()), i
    print("dilated convs at 416, batch %d: worst |err| / bound %.3f" % (b, worst))


def test_yolov3m_eval_vs_reference_model_output():
    g = m_golden()
    sd = json.loads(golden_text(g, "seeds"))
    m = init_darknet_weights(m_model(), seed=sd["eval_w"]).cuda().eval()
    x = torch.rand(1, 3, 416, 416, generator=torch.Generator().manual_seed(sd["eval_x"])).cuda()
    with torch.no_grad():
        io, ps = m(x)
    assert tuple(io.shape) == tuple(g["eval_io_shape"]) and len(ps) == 16
    for k, p in enumerate(ps):
        assert tuple(p.shape) == tuple(g["eval_p%d_shape" % k])
        want = g["eval_p%d" % k]
        idx = torch.Generator().manual_seed(100 + k)
        got = p.reshape(-1)[torch.randint(0, p.numel(), (len(want),), generator=idx).cuda()].cpu().numpy()
        err, scale = np.abs(got - want), float(g["eval_p%d_absmax" % k])
        # the bf16 whole-net tolerance of test_darknet_gpu.py::test_vs_reference_model_output
        assert err.max() <= 3e-2 * scale, (k, float(err.max()), scale)
        assert np.sqrt((err ** 2).mean()) <= 6e-3 * scale, k
    # decoded rows: each within what its head's raw bound allows through sigmoid (slope 1/4, times the stride) and
    # atan (slope 1); the linear branch heads of this graph reach |p| ~ 460 with these weights
    rows_idx = torch.randint(0, io.shape[1], (len(g["eval_io_rows"]),), generator=torch.Generator().manual_seed(110))
    rows, want = io[0, rows_idx.cuda()].cpu().numpy(), g["eval_io_rows"]
    shapes = [g["eval_p%d_shape" % k] for k in range(16)]
    ends = np.cumsum([s[1] * s[2] * s[3] for s in shapes])
    head = np.searchsorted(ends, rows_idx.numpy(), side="right")
    draw = np.array([3e-2 * float(g["eval_p%d_absmax" % k]) for k in range(16)])[head]
    stride = np.array([416.0 / s[3] for s in shapes])[head]
    assert (np.abs(rows[:, :2] - want[:, :2]) <= np.maximum(0.5, 0.25 * stride * draw)[:, None]).all()
    assert (np.abs(rows[:, 4] - want[:, 4]) <= np.maximum(3e-2, draw)).all()
    assert (np.abs(rows[:, 5] - want[:, 5]) <= np.maximum(3e-2, 0.25 * draw)).all()


def _bits(t):
    """bit pattern (the decoded wh of this graph's large heads overflow to inf / nan, as in the reference)"""
    return t.contiguous().view(torch.int32)


def test_yolov3m_eval_is_repeatable_and_graph_replay_equals_eager():
    m = init_darknet_weights(m_model(), seed=5).cuda().eval()
    x = torch.rand(2, 3, 416, 416, device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
    with torch.no_grad():
        io1, _ = m(x)
        io1 = io1.clone()
        io2, _ = m(x)
        assert torch.equal(_bits(io1), _bits(io2))
        m.use_cuda_graph = True
        io3, ps3 = m(x)
        assert torch.equal(_bits(io1), _bits(io3)) and len(ps3) == 16
        # each image equals its batch-1 forward (no accumulation order depends on the batch)
        m.use_cuda_graph = False
        io_b1, _ = m(x[1:2])
        assert torch.equal(_bits(io_b1[0]), _bits(io1[1]))


def test_dropin_builds_and_runs_yolov3m():
    import sys
    import rotate_yolov3_b200.dropin as dropin
    dropin.install()
    Darknet = sys.modules["model.models"].Darknet
    from builders import m_cfg_text
    m = Darknet(m_cfg_text("cfg/yolov3-m.cfg"), {"context_factor": 1.0}, arc="default")
    init_darknet_weights(m, seed=7)
    m = m.cuda().eval()
    with torch.no_grad():
        io, ps = m(torch.rand(1, 3, 256, 320, device="cuda"))
    assert len(ps) == 16 and io.shape[0] == 1 and all(bool(torch.isfinite(p).all()) for p in ps)
