"""Whole-network eval forward of ``Darknet`` (Darknet-53 graph of cfg/yolov3.cfg) on the GPU.

(1) vs the committed output of the REFERENCE model (tests/golden/make_golden.py section 6, CPU fp32): the conv
    operands are bf16 (fp32 accumulate), so the comparison is at bf16 tolerance through 75 layers -- stated below;
(2) vs a plain PyTorch fp32 emulation of the SAME quantisation points (operands rounded to bf16 at every layer
    boundary, fp32 math): isolates kernel correctness from precision, much tighter."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from f64_refs import bf
from helpers import GOLDEN, SMALL_ANCHORS, init_darknet_weights

pytestmark = pytest.mark.gpu


def _model(width=96, height=64):
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import cfgs
    text = cfgs.yolov3_cfg(width=width, height=height, classes=1, anchors=SMALL_ANCHORS, n_anchors=6)
    m = pkg.Darknet(text, {"context_factor": 1.0}, arc="default")
    init_darknet_weights(m, seed=123)
    return m.cuda().eval()


def _emulate_bf16(model, x):
    """torch fp32 reference of the same op chain with bf16 operand rounding at the kernel's quantisation points"""
    outs = []
    heads = []
    for i, (d, mod) in enumerate(zip(model.module_defs, model.module_list)):
        t = d["type"]
        if t == "convolutional":
            w, scale, bias, slope = model._folded(i, x.device)
            wq = bf(w * scale.view(-1, 1, 1, 1)) if scale is not None else bf(w)
            xin = x if i == 0 else bf(x)
            # first layer (first.cu): tensor pipe with the image as bf16 hi + lo halves (16 mantissa bits: fp32 up to
            # 2^-17) and bf16 weights like every other layer -- so only the weights are quantised here
            k = w.shape[-1]
            y = F.conv2d(xin, wq, bias, stride=int(d["stride"]), padding=(k - 1) // 2)
            if slope is not None:
                y = torch.where(y > 0, y, slope * y)
            x = y
            if model.module_defs[i + 1]["type"] == "yolo":
                heads.append(y)
        elif t == "shortcut":
            x = x + bf(outs[i + int(d["from"])])
        elif t == "upsample":
            x = F.interpolate(x, scale_factor=2, mode="nearest")
        elif t == "route":
            ls = [int(v) for v in d["layers"].split(",")]
            ls = [l if l > 0 else i + l for l in ls]
            x = torch.cat([outs[l] for l in ls], 1) if len(ls) > 1 else outs[ls[0]]
        outs.append(x)
    return heads


def test_vs_reference_model_output():
    g = np.load(os.path.join(GOLDEN, "darknet_golden.npz"))
    m = _model()
    assert sum(p.numel() for p in m.parameters()) == int(g["n_params"])
    with torch.no_grad():
        io, ps = m(torch.from_numpy(g["x"]).cuda())
    assert io.shape == g["io"].shape and len(ps) == 3
    for k, p in enumerate(ps):
        want = g["p%d" % k]
        assert p.shape == want.shape
        err = np.abs(p.cpu().numpy() - want)
        scale = np.abs(want).max()
        # bf16 operands (8-bit mantissa) through 75 layers vs the fp32 reference: 3e-2 of the output scale
        assert err.max() <= 3e-2 * scale, (k, float(err.max()), float(scale))
        assert np.sqrt((err ** 2).mean()) <= 6e-3 * scale
    # decoded boxes: compare where exp() has not amplified the raw difference
    io_want = g["io"]
    xy_err = np.abs(io.cpu().numpy()[..., :2] - io_want[..., :2]).max()
    assert xy_err <= 0.5, float(xy_err)        # pixels (stride 8..32 times a sigmoid difference)
    assert np.abs(io.cpu().numpy()[..., 4:6] - io_want[..., 4:6]).max() <= 3e-2


def test_vs_torch_emulation_of_the_same_quantisation():
    m = _model()
    g = torch.Generator().manual_seed(3)
    x = torch.rand(2, 3, 64, 96, generator=g).cuda()
    with torch.no_grad():
        io, ps = m(x)
        heads = _emulate_bf16(m, x)
    for p, hd, yi in zip(ps, heads, m.yolo_layers):
        layer = m.module_list[yi]
        want = hd.view(hd.shape[0], layer.na, layer.nc + 6, hd.shape[2], hd.shape[3]).permute(0, 1, 3, 4, 2)
        err = (p - want).abs()
        scale = float(want.abs().max())
        # identical quantisation points; remaining differences = fp32 summation order flipping a bf16 rounding
        # somewhere upstream (one bf16 ulp = 0.4 %), diluted by the following layers
        assert float(err.max()) <= 2.5e-2 * scale, (float(err.max()), scale)
        assert float(err.pow(2).mean().sqrt()) <= 4e-3 * scale


def test_boundary_and_state_dict_names():
    import rotate_yolov3_b200 as pkg
    m = _model()
    names = list(m.state_dict().keys())
    assert "module_list.0.Conv2d.weight" in names and "module_list.0.BatchNorm2d.running_var" in names
    assert "module_list.0.activation.weight" in names and "module_list.81.Conv2d.bias" in names
    assert m.yolo_layers == [82, 94, 106] and len(m.module_list) == 107
    assert set(m.routes) >= {79, 85, 61, 91, 97, 36}
    with pytest.raises(RuntimeError):
        m(torch.zeros(1, 3, 64, 64))          # CPU tensor: no fallback
    with torch.no_grad():
        io1, _ = m(torch.rand(1, 3, 64, 64, device="cuda"))
        io2, _ = m(torch.rand(3, 3, 96, 64, device="cuda"))   # new shape -> new plan
    assert io1.shape == (1, 2 * (4 + 16 + 64), 7) and io2.shape == (3, 2 * (6 + 24 + 96), 7)
    yl = m.module_list[106]
    assert (yl.nx, yl.ny) == (8, 12) and float(yl.stride) == 8.0 and yl.anchor_vec.shape == (2, 3)


def test_eval_plan_follows_in_place_weight_updates():
    """the eval plan caches packed, BN-folded weights; an in-place parameter update (optimizer step, manual edit) must
    invalidate it"""
    import rotate_yolov3_b200 as pkg
    from helpers import init_darknet_weights, mini_cfg
    dev = torch.device("cuda")
    m = pkg.Darknet(mini_cfg(), {"context_factor": 1.0})
    init_darknet_weights(m, seed=3)
    m = m.to(dev).eval()
    x = torch.rand(2, 3, 64, 96, device=dev)
    with torch.no_grad():
        io0 = m(x)[0].clone()
        io1 = m(x)[0].clone()
        assert torch.equal(io0, io1)
        m.module_list[0].Conv2d.weight.mul_(1.5)          # in place, still in eval mode
        io2 = m(x)[0].clone()
    assert not torch.allclose(io0, io2)


def test_se_block_kernel_and_graph_vs_torch():
    """[se] blocks (reference SELayer, model/models.py:16-31, cfg/ICDAR/yolov3_608_se.cfg): the in-place kernel against
    x * sigmoid(W2 relu(W1 mean(x))) on the same bf16 tensor (one bf16 ulp), and a graph with an [se] block after its
    down-sampling conv against a torch fp32 walk of the same modules (bf16 tolerance of the throughput mode)."""
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import layout as L
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(4)
    b, c, h, w, cr = 3, 64, 13, 17, 4
    x = torch.randn(b, c, h, w, generator=g).to(dev).to(torch.bfloat16).float()
    w1 = (torch.randn(cr, c, generator=g) / 8).to(dev)
    w2 = (torch.randn(c, cr, generator=g) / 2).to(dev)
    buf = L.to_padded_nhwc(x, 64)
    sums = torch.zeros(b * c, device=dev)
    scale = torch.zeros(b * c, device=dev)
    st = pkg._lib.lib.ryolo_se_block(pkg._lib.ptr(buf), 64, b, h, w, c, pkg._lib.ptr(w1), pkg._lib.ptr(w2), cr,
                                     pkg._lib.ptr(sums), pkg._lib.ptr(scale), pkg._lib.stream_ptr(dev))
    assert st == 0, pkg._lib.last_error()
    s_want = torch.sigmoid(torch.relu(x.mean((2, 3)) @ w1.t()) @ w2.t())
    assert torch.allclose(scale.view(b, c), s_want, rtol=1e-5, atol=1e-6)
    want = x * s_want[:, :, None, None]
    got = L.from_padded_nhwc(buf, c)
    assert bool(((got - want).abs() <= 2.0 ** -8 * want.abs() + 1e-6).all())
    assert float(buf[:, 0].abs().max()) == 0 and float(buf[:, :, 0].abs().max()) == 0          # halo untouched

    def conv(f, k, s=1):
        return "[convolutional]\nbatch_normalize=1\nfilters=%d\nsize=%d\nstride=%d\npad=1\nactivation=leaky\n\n" % (f, k, s)
    cfg = ("[net]\nwidth=64\nheight=48\nchannels=3\n\n" + conv(32, 3) + conv(64, 3, 2) + "[se]\nchannels=64\n\n" + conv(32, 1) +
           conv(64, 3) + "[shortcut]\nfrom=-3\nactivation=linear\n\n" +
           "[convolutional]\nfilters=14\nsize=1\nstride=1\npad=1\nactivation=linear\n\n"
           "[yolo]\nmask = 0-1\nanchors = ara 900 / 5.0 / -45, 45\nclasses=1\nnum=2\n\n")
    m = pkg.Darknet(cfg, {"context_factor": 1.0})
    init_darknet_weights(m, seed=5)
    assert "module_list.2.fc.0.weight" in m.state_dict() and "module_list.2.fc.2.weight" in m.state_dict()
    m = m.to(dev).eval()
    xin = torch.rand(2, 3, 48, 64, generator=g).to(dev)
    with torch.no_grad():
        io, ps = m(xin)
        # torch fp32 walk of the same modules
        outs, t = [], xin
        for i, (d, mod) in enumerate(zip(m.module_defs, m.module_list)):
            ty = d["type"]
            if ty == "convolutional":
                wt, sc, bias, slope = m._folded(i, dev)
                wt = wt * sc.view(-1, 1, 1, 1) if sc is not None else wt
                t = F.conv2d(t, wt, bias, stride=int(d["stride"]), padding=(wt.shape[-1] - 1) // 2)
                if slope is not None:
                    t = torch.where(t > 0, t, slope * t)
            elif ty == "se":
                s_ = torch.sigmoid(torch.relu(t.mean((2, 3)) @ mod.fc[0].weight.t()) @ mod.fc[2].weight.t())
                t = t * s_[:, :, None, None]
            elif ty == "shortcut":
                t = t + outs[i + int(d["from"])]
            elif ty == "yolo":
                head = t
            outs.append(t)
    layer = m.module_list[m.yolo_layers[0]]
    want = head.view(2, layer.na, 7, head.shape[2], head.shape[3]).permute(0, 1, 3, 4, 2)
    err = (ps[0] - want).abs()
    assert float(err.max()) <= 3e-2 * float(want.abs().max()), float(err.max())


def test_half_module_runs_the_eval_path():
    """detect.py --half does model.half(): parameters become fp16.  The packed operands are bf16 anyway, so the eval
    forward must accept it (fp32 outputs) and agree with the fp32-parameter model up to the fp16 rounding of the weights"""
    m = _model()
    x = torch.rand(2, 3, 64, 96, generator=torch.Generator().manual_seed(8)).cuda()
    with torch.no_grad():
        io0, ps0 = m(x)
        io0, ps0 = io0.clone(), [p.clone() for p in ps0]
        mh = m.half()
        io1, ps1 = mh(x.half())
    assert io1.dtype == torch.float32
    for a, b in zip(ps0, ps1):
        assert float((a - b).abs().max()) <= 2e-2 * float(a.abs().max())
    mh.train()
    with pytest.raises(RuntimeError):
        mh(x)                                               # the fused training step needs fp32 master parameters
