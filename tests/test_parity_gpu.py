"""Parity-precision mode (``Darknet(..., precision="parity")``): conv activations and gradients within 1e-4 of the
output scale of the REFERENCE's fp32 results (north_star tolerance; VERDICT r1 item 1).

  * px_conv (split-bf16 operands, six exact-product terms, segment sums) vs a float64 convolution of the SAME fp32
    operands -- arbitrary fp32 inputs, not bf16-representable ones;
  * mini graph (every structural feature), Darknet-53 graph at 96 x 64 and 160 x 128, and the BASELINE shape --
    cfg/yolov3.cfg graph with its 216-anchor line (504-channel heads) at 608 x 608 -- against goldens produced by the
    reference model itself (tests/golden/make_golden.py, make_golden_608.py): eval heads + decoded rows, training-mode
    heads, parameter gradients.
Tolerance written out: |ours - ref| <= 1e-4 * max|ref| per tensor (TOL below)."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from builders import PARITY_TOL as TOL, report_and_check_gradients
from helpers import GOLDEN, SMALL_ANCHORS, init_darknet_weights, mini_cfg

pytestmark = pytest.mark.gpu


def _split(x_nchw, plane):
    """fp32 NCHW -> split bf16 padded NHWC [B, H+2, W+2, NP*plane] through the library"""
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import parity_path as PP
    L = pkg._lib
    b, c, h, w = x_nchw.shape
    buf = torch.zeros((b, h + 2, w + 2, PP.NP * plane), dtype=torch.bfloat16, device=x_nchw.device)
    st = L.lib.ryolo_px_split_from_nchw(L.ptr(x_nchw.contiguous()), b, c, h, w, L.ptr(buf), PP.NP * plane, plane, PP.NP,
                                        L.stream_ptr(x_nchw.device))
    assert st == 0, L.last_error()
    return buf


def _px_conv(x, wt, k, accumulate_into=None, ch_off=0, extra=0):
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import parity_path as PP
    L = pkg._lib
    dev = x.device
    b, cin, h, w = x.shape
    cout = wt.shape[0]
    plane = (cin + ch_off + extra + 63) // 64 * 64
    xs = torch.zeros((b, cin + ch_off + extra, h, w), device=dev)
    xs[:, ch_off:ch_off + cin] = x
    if extra:
        xs[:, ch_off + cin:] = 3.0            # neighbouring channels of a wider buffer meet zero weights
    buf = _split(xs, plane)
    pw = torch.empty(L.lib.ryolo_px_packed_weight_bytes(cout, cin, k, PP.NTERMS), dtype=torch.uint8, device=dev)
    st = L.lib.ryolo_px_pack_weights(L.ptr(wt.contiguous()), cout, cin, k, PP.NTERMS, PP.W_CODE, 0, L.ptr(pw), L.stream_ptr(dev))
    assert st == 0, L.last_error()
    po = (cout + 63) // 64 * 64
    z = torch.zeros((b, h + 2, w + 2, po), device=dev) if accumulate_into is None else accumulate_into
    st = L.lib.ryolo_px_conv(L.ptr(buf), PP.NP * plane, ch_off, plane, cin, L.ptr(pw), PP.NTERMS, PP.A_CODE, b, h, w, k, cout,
                             L.ptr(z), po, po, 0 if accumulate_into is None else 1, L.stream_ptr(dev))
    assert st == 0, L.last_error()
    torch.cuda.synchronize()
    return z


@pytest.mark.parametrize("cin,cout,k,h,w", [(64, 64, 1, 9, 11), (27, 32, 1, 16, 12), (128, 256, 3, 19, 19),
                                            (1024, 512, 1, 19, 19), (1024, 128, 3, 19, 19), (96, 40, 3, 10, 14)])
def test_px_conv_vs_float64(cin, cout, k, h, w):
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(cin + k)
    x = torch.randn(2, cin, h, w, generator=g).to(dev)
    wt = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).to(dev)
    z = _px_conv(x, wt, k)
    want = F.conv2d(x.double(), wt.double(), padding=(k - 1) // 2)
    got = z[:, 1:-1, 1:-1, :cout].permute(0, 3, 1, 2).double()
    err = (got - want).abs()
    scale = float(want.abs().max())
    rms = float(want.pow(2).mean().sqrt())
    # three planes carry the fp32 operands exactly; what is left is fp32 accumulation (segment sums, round to nearest)
    print("px_conv cin=%d k=%d: max %.2e rms %.2e (of scale / rms)" % (cin, k, float(err.max()) / scale,
                                                                        float(err.pow(2).mean().sqrt()) / rms))
    assert float(err.max()) <= 5e-6 * scale, (float(err.max()), scale)
    assert float(err.pow(2).mean().sqrt()) <= 2e-6 * rms
    bias = float(((got - want) * want.sign()).mean()) / rms
    assert abs(bias) <= 1e-6, bias               # no truncation bias (the raw tensor pipe shows -6.6e-6 at K = 9216)
    # halo and channel padding stay zero
    assert float(z[:, 0].abs().max()) == 0 and float(z[:, :, 0].abs().max()) == 0
    if z.shape[-1] > cout:
        assert float(z[..., cout:].abs().max()) == 0


def test_px_conv_view_offset_and_accumulate():
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 64, 12, 10, generator=g).to(dev)
    wt = (torch.randn(96, 64, 3, 3, generator=g) / 24).to(dev)
    z0 = _px_conv(x, wt, 3)
    z1 = _px_conv(x, wt, 3, ch_off=64, extra=64)          # same conv reading a slice of a wider (concat) buffer
    assert torch.equal(z0, z1)
    acc = z0.clone()
    _px_conv(x, wt, 3, accumulate_into=acc)
    assert torch.allclose(acc, 2 * z0, rtol=1e-6, atol=0)


def _check(name, got, want, tol=TOL):
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    scale = np.abs(want).max()
    err = np.abs(got - want).max()
    assert err <= tol * scale + 1e-30, "%s: max err %.3e vs %.1e * scale %.3e (ratio %.2e)" % (name, err, tol, scale,
                                                                                               err / max(scale, 1e-30))
    return err / max(scale, 1e-30)


def _parity_model(text, seed, train=False):
    import rotate_yolov3_b200 as pkg
    m = pkg.Darknet(text, {"context_factor": 1.0}, arc="default", precision="parity")
    init_darknet_weights(m, seed=seed)
    m = m.cuda()
    return m.train() if train else m.eval()


def test_mini_graph_eval_and_all_gradients_vs_reference():
    g = np.load(os.path.join(GOLDEN, "mini_train_golden.npz"))
    m = _parity_model(mini_cfg(64, 48), 77)
    x = torch.from_numpy(g["x"]).cuda()
    with torch.no_grad():
        io, ps = m(x)
    _check("io_eval", io.cpu().numpy(), g["io_eval"])
    for k, p in enumerate(ps):
        _check("pe%d" % k, p.cpu().numpy(), g["pe%d" % k])
    m.train()
    ps = m(x)
    for k, p in enumerate(ps):
        _check("p%d" % k, p.detach().cpu().numpy(), g["p%d" % k])
    loss = sum((p * torch.from_numpy(g["g%d" % k]).cuda()).sum() for k, p in enumerate(ps)) / 10.0
    assert abs(float(loss) - float(g["loss"])) <= 1e-4 * max(1.0, abs(float(g["loss"])))
    loss.backward()
    worst = 0.0
    for name, prm in m.named_parameters():
        worst = max(worst, _check("grad " + name, prm.grad.cpu().numpy(), g["grad:" + name]))
    print("mini graph: worst gradient error / scale = %.2e" % worst)


def test_darknet53_small_eval_vs_reference():
    from rotate_yolov3_b200 import cfgs
    g = np.load(os.path.join(GOLDEN, "darknet_golden.npz"))
    m = _parity_model(cfgs.yolov3_cfg(width=96, height=64, classes=1, anchors=SMALL_ANCHORS, n_anchors=6), 123)
    with torch.no_grad():
        io, ps = m(torch.from_numpy(g["x"]).cuda())
    for k, p in enumerate(ps):
        _check("p%d" % k, p.cpu().numpy(), g["p%d" % k])
    ion, want = io.cpu().numpy(), g["io"]
    _check("io xy/theta/obj", ion[..., [0, 1, 4, 5]], want[..., [0, 1, 4, 5]])
    assert np.all(np.abs(ion[..., 2:4] - want[..., 2:4]) <= 2e-4 * np.abs(want[..., 2:4]) + 1e-6)   # exp() amplifies the raw error


def test_darknet53_small_training_vs_reference():
    from rotate_yolov3_b200 import cfgs
    g = np.load(os.path.join(GOLDEN, "darknet_train_golden.npz"), allow_pickle=True)
    m = _parity_model(cfgs.yolov3_cfg(width=160, height=128, classes=1, anchors=SMALL_ANCHORS, n_anchors=6), 321, train=True)
    ps = m(torch.from_numpy(g["x"]).cuda())
    for k, p in enumerate(ps):
        _check("p%d" % k, p.detach().cpu().numpy(), g["p%d" % k])
    loss = sum((p * torch.from_numpy(g["g%d" % k]).cuda()).sum() for k, p in enumerate(ps)) / 100.0
    loss.backward()
    grads = dict(m.named_parameters())
    rows = []
    for name, norm, idx, smp in zip(g["names"], g["norms"], g["sample_idx"], g["samples"]):
        name = str(name)
        gr = grads[name].grad.reshape(-1)
        got = gr[torch.from_numpy(np.asarray(idx, dtype=np.int64)).cuda()].cpu().numpy()
        # samples against the gradient's own scale (norm / sqrt(numel) ~ rms; max ~ a few rms)
        scale = max(float(np.abs(smp).max()), float(norm) / gr.numel() ** 0.5)
        if name.endswith("activation.weight"):      # one scalar: error against the largest slope gradient of the net
            sscale = max(float(nn_) for nm_, nn_ in zip(g["names"], g["norms"]) if str(nm_).endswith("activation.weight"))
            e = abs(float(gr[0]) - float(np.asarray(smp).reshape(-1)[0])) / sscale
            rows.append((int(name.split(".")[1]), name, e, e))
            continue
        rows.append((int(name.split(".")[1]), name, float(np.abs(got - smp).max()) / scale,
                     abs(float(gr.norm()) - float(norm)) / float(norm)))
    report_and_check_gradients("darknet-53 160x128 training", rows)
    bn0 = m.module_list[0].BatchNorm2d
    _check("running_mean0", bn0.running_mean.cpu().numpy(), g["rm0"])
    _check("running_var0", bn0.running_var.cpu().numpy(), g["rv0"])


def _idx(numel, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, numel, (min(n, numel),), generator=g)


def test_baseline_shape_608_eval_vs_reference():
    """cfg/yolov3.cfg graph, 216 anchors (504-channel heads), 608 x 608, batch 1 -- the BASELINE configuration"""
    from rotate_yolov3_b200 import cfgs
    g = np.load(os.path.join(GOLDEN, "darknet608_golden.npz"), allow_pickle=True)
    m = _parity_model(cfgs.yolov3_cfg(), 608)
    assert sum(p.numel() for p in m.parameters()) == int(g["n_params"])
    x = torch.rand(1, 3, 608, 608, generator=torch.Generator().manual_seed(6080))
    assert np.array_equal(x.reshape(-1)[:64].numpy(), g["x_probe"])
    with torch.no_grad():
        io, ps = m(x.cuda())
    assert io.shape == (1, 545832, 7) and [tuple(p.shape) for p in ps] == [(1, 72, 19, 19, 7), (1, 72, 38, 38, 7), (1, 72, 76, 76, 7)]
    for k, p in enumerate(ps):
        flat = p.reshape(-1)
        got = flat[_idx(flat.numel(), 100000, 100 + k).cuda()].cpu().numpy()
        want = g["eval_p%d" % k]
        err = np.abs(got - want).max()
        assert err <= TOL * float(g["eval_p%d_absmax" % k]), (k, err, float(g["eval_p%d_absmax" % k]))
        print("608 eval head %d: max err / scale = %.2e" % (k, err / float(g["eval_p%d_absmax" % k])))
    rows = io[0, _idx(io.shape[1], 20000, 110).cuda()].cpu().numpy()
    want = g["eval_io_rows"]
    _check("io xy/theta/obj", rows[:, [0, 1, 4, 5]], want[:, [0, 1, 4, 5]])
    assert np.all(np.abs(rows[:, 2:4] - want[:, 2:4]) <= 5e-4 * np.abs(want[:, 2:4]) + 1e-6)


def test_baseline_shape_608_training_vs_reference():
    from rotate_yolov3_b200 import cfgs
    g = np.load(os.path.join(GOLDEN, "darknet608_golden.npz"), allow_pickle=True)
    m = _parity_model(cfgs.yolov3_cfg(), 609, train=True)
    x = torch.rand(2, 3, 608, 608, generator=torch.Generator().manual_seed(6090))
    ps = m(x.cuda())
    gen = torch.Generator().manual_seed(6091)
    gs = [torch.randn(p.shape, generator=gen) for p in ps]
    for k, p in enumerate(ps):
        flat = p.detach().reshape(-1)
        got = flat[_idx(flat.numel(), 100000, 200 + k).cuda()].cpu().numpy()
        err = np.abs(got - g["train_p%d" % k]).max()
        assert err <= TOL * float(g["train_p%d_absmax" % k]), (k, err)
        print("608 train head %d: max err / scale = %.2e" % (k, err / float(g["train_p%d_absmax" % k])))
    loss = sum((p * gg.cuda()).sum() for p, gg in zip(ps, gs)) / 100.0
    assert abs(float(loss) - float(g["train_loss"])) <= 1e-4 * max(1.0, abs(float(g["train_loss"])))
    loss.backward()
    grads = dict(m.named_parameters())
    rows = []
    for j, (name, norm, amax, smp) in enumerate(zip(g["grad_names"], g["grad_norms"], g["grad_absmax"], g["grad_samples"])):
        name = str(name)
        gr = grads[name].grad.reshape(-1)
        n = 8192 if name.split(".")[1] in ("81", "93", "105") else 128
        got = gr[_idx(gr.numel(), n, 1000 + j).cuda()].cpu().numpy()
        if name.endswith("activation.weight"):      # one scalar: error against the largest slope gradient of the net
            sscale = max(float(nn_) for nm_, nn_ in zip(g["grad_names"], g["grad_norms"]) if str(nm_).endswith("activation.weight"))
            e = abs(float(gr[0]) - float(np.asarray(smp).reshape(-1)[0])) / sscale
            rows.append((int(name.split(".")[1]), name, e, e))
            continue
        rows.append((int(name.split(".")[1]), name, float(np.abs(got - np.asarray(smp, dtype=np.float32)).max()) / float(amax),
                     abs(float(gr.norm()) - float(norm)) / float(norm)))
    report_and_check_gradients("608x608 training", rows)
    bn0 = m.module_list[0].BatchNorm2d
    _check("running_mean0", bn0.running_mean.cpu().numpy(), g["rm0"])
    _check("running_var0", bn0.running_var.cpu().numpy(), g["rv0"])
    _check("running_mean104", m.module_list[104].BatchNorm2d.running_mean.cpu().numpy(), g["rm104"])


def test_parity_plan_rejects_stale_backward():
    """ADVICE r1: two forwards before a backward would silently use overwritten activations -> must raise"""
    m = _parity_model(mini_cfg(64, 48), 3, train=True)
    x = torch.rand(2, 3, 48, 64, device="cuda")
    a = m(x)
    b = m(x)
    with pytest.raises(RuntimeError):
        sum(t.sum() for t in a).backward()
    sum(t.sum() for t in b).backward()


def test_parity_plan_does_not_outlive_its_replacement():
    """a new parity plan is built only after the previous one is gone, even while the caller keeps the last training
    step's heads (whose grad_fn is the step's autograd node): at batch 16 x 608^2 the training plan and its successor do
    not fit one 80 GB card together"""
    import weakref

    from rotate_yolov3_b200 import parity_path as PP
    m = _parity_model(mini_cfg(64, 48), 5, train=True)
    plans, alive_at_init = [], []
    init = PP.ParityPlan.__init__

    def recording_init(self, *a, **k):
        alive_at_init.append([p() is not None for p in plans])
        init(self, *a, **k)
        plans.append(weakref.ref(self))

    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(PP.ParityPlan, "__init__", recording_init)
        pred = m(torch.rand(2, 3, 48, 64, device="cuda"))
        m.eval()
        with torch.no_grad():
            m(torch.rand(2, 3, 48, 64, device="cuda"))
            m(torch.rand(2, 3, 32, 96, device="cuda"))
        m.train()
        stale = pred
        pred = m(torch.rand(1, 3, 48, 64, device="cuda"))
    assert alive_at_init == [[], [False], [False, False], [False, False, False]], alive_at_init
    with pytest.raises(RuntimeError, match="dropped"):
        sum(t.sum() for t in stale).backward()
    sum(t.sum() for t in pred).backward()
