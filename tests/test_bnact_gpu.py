"""Training-mode BatchNorm + PReLU (+ shortcut, + upsample) forward / backward kernels and the dgrad path against
PyTorch autograd in fp32 on the same bf16-representable inputs."""
import ctypes

import pytest
import torch
import torch.nn.functional as F
from f64_refs import bf

pytestmark = pytest.mark.gpu


# up: False plain dy, True dy at 2x resolution (nearest-upsample adjoint), 2 dy in the space-to-depth layout of a following
# 3x3/stride-2 block.  c = 32 / 48-wide strides take the direct kernels, the others the TMA row pipes (csrc/bnpipe.cuh);
# the 200 x 200 cases span several pieces per row and wrap the shared-memory ring several times per CTA.
@pytest.mark.parametrize("c,h,w,b,res,up", [(64, 6, 5, 3, False, False), (128, 9, 7, 2, True, False),
                                            (256, 5, 4, 2, False, True), (32, 8, 8, 2, False, False),
                                            (64, 200, 200, 4, True, False), (128, 8, 6, 2, False, 2),
                                            (64, 200, 200, 3, False, 2), (32, 8, 8, 2, False, 2), (1024, 19, 19, 8, True, False),
                                            (64, 120, 200, 2, False, True)])
def test_bn_stats_finalize_prelu_fwd_bwd_vs_autograd(c, h, w, b, res, up):
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import layout as L
    lib = pkg._lib.lib
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(c + h)
    z = bf(torch.randn(b, c, h, w, generator=g) * 1.5 + 0.3).to(dev)
    gamma = (0.5 + torch.rand(c, generator=g)).to(dev)
    beta = (0.3 * torch.randn(c, generator=g)).to(dev)
    slope = 0.17
    r = bf(torch.randn(b, c, h, w, generator=g)).to(dev) if res else None
    s2d = up == 2
    up = up is True
    oh, ow = (2 * h, 2 * w) if up else (h, w)
    dy = bf(torch.randn(b, c, oh, ow, generator=g)).to(dev)
    # ---- torch reference ----
    zt = z.clone().requires_grad_(True)
    gt, bt = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    st = torch.tensor([slope], device=dev, requires_grad=True)
    rt = r.clone().requires_grad_(True) if res else None
    y = F.prelu(F.batch_norm(zt, None, None, gt, bt, training=True, eps=1e-5), st)
    if res:
        y = y + rt
    if up:
        y = F.interpolate(y, scale_factor=2, mode="nearest")
    y.backward(dy)
    # ---- kernels ----
    cs = L.round_up(c, 64)
    zb = L.to_padded_nhwc(z, cs)
    pt = pkg._lib.ptr
    stream = pkg._lib.stream_ptr(dev)
    # statistics + finalisation in ONE call (the reduction of the per-CTA partial rows finalises each channel) ==
    # nn.BatchNorm2d's bookkeeping
    sums = torch.full((2 * c + 1,), 3.0, device=dev)       # sums[0, 2c) are overwritten, whatever they held
    f_mean, f_inv, f_sc, f_sh = (torch.empty(c, device=dev) for _ in range(4))
    rm, rv = torch.full((c,), 0.25, device=dev), torch.full((c,), 2.0, device=dev)
    assert lib.ryolo_bn_stats_finalize(pt(zb), cs, b, h, w, c, pt(sums), 1e-5, 0.1, pt(gamma), pt(beta), pt(f_mean), pt(f_inv),
                                       pt(f_sc), pt(f_sh), pt(rm), pt(rv), stream) == 0
    n = b * h * w
    mean = sums[:c] / n
    var = (sums[c:2 * c] / n - mean * mean).clamp_(min=0)
    assert torch.allclose(mean, z.mean((0, 2, 3)), atol=1e-4) and torch.allclose(var, z.var((0, 2, 3), unbiased=False), rtol=1e-3, atol=1e-4)
    invstd = torch.rsqrt(var + 1e-5)
    scale = (gamma * invstd).contiguous()
    shift = (beta - mean * scale).contiguous()
    assert torch.allclose(f_mean, mean, atol=1e-5) and torch.allclose(f_inv, invstd, rtol=1e-4)
    assert torch.allclose(f_sc, scale, rtol=1e-4, atol=1e-6) and torch.allclose(f_sh, shift, rtol=1e-4, atol=1e-5)
    assert torch.allclose(rm, 0.9 * 0.25 + 0.1 * mean, atol=1e-5)
    assert torch.allclose(rv, 0.9 * 2.0 + 0.1 * var * (n / (n - 1)), rtol=1e-4, atol=1e-5)
    yb = L.alloc_padded(b, oh, ow, cs, dev)
    rb = L.to_padded_nhwc(r, cs) if res else None
    sd = torch.tensor([slope], device=dev)     # the slope as a device scalar (nn.PReLU.weight): overrides the host value
    assert lib.ryolo_bn_act_fwd(pt(zb), cs, b, h, w, c, pt(scale), pt(shift), 123.0, 1, pt(rb) if res else None, cs, pt(yb),
                                cs, int(up), pt(sd), stream) == 0
    got_y = L.from_padded_nhwc(yb, c)
    assert float((got_y - y.detach()).abs().max()) <= 2.0 ** -7 * float(y.abs().max())
    dyb, dcs, mode = L.to_padded_nhwc(dy, cs), cs, int(up)
    if s2d:     # [b, c, h, w] -> [b, 4c, h/2, w/2] with channel block (y & 1) * 2 + (x & 1), channel stride exactly 4c
        q = torch.cat([dy[:, :, ry::2, rx::2] for ry in range(2) for rx in range(2)], 1)
        dyb, dcs, mode = L.to_padded_nhwc(q, 4 * c), 4 * c, 2
    bs = torch.zeros(2 * c + 1, device=dev)
    grb = L.alloc_padded(b, h, w, cs, dev) if res else None
    assert lib.ryolo_bn_act_bwd(pt(dyb), dcs, mode, pt(zb), cs, b, h, w, c, pt(scale), pt(shift), pt(mean.contiguous()),
                                pt(invstd.contiguous()), slope if res else -7.0, 1, 1, pt(bs), pt(grb) if res else None, cs, 0,
                                None if res else pt(sd), stream) == 0
    torch.cuda.synchronize()
    dz = L.from_padded_nhwc(zb, c)
    sc = float(zt.grad.abs().max())
    assert float((dz - zt.grad).abs().max()) <= 1.5e-2 * sc, (float((dz - zt.grad).abs().max()), sc)
    assert torch.allclose(bs[:c], bt.grad, rtol=1e-3, atol=1e-3 * float(bt.grad.abs().max()))
    assert torch.allclose(bs[c:2 * c], gt.grad, rtol=1e-3, atol=1e-3 * float(gt.grad.abs().max()))
    assert abs(float(bs[2 * c]) - float(st.grad)) <= 2e-3 * abs(float(st.grad)) + 1e-3
    if res:
        assert float((L.from_padded_nhwc(grb, c) - rt.grad).abs().max()) <= 1e-6
    assert float(zb[:, 0].abs().max()) == 0 and float(zb[:, :, -1].abs().max()) == 0   # halo stays zero


@pytest.mark.parametrize("cin,cout,k,stride,h,w", [(64, 128, 3, 1, 10, 9), (128, 64, 1, 1, 7, 7), (64, 128, 3, 2, 12, 10),
                                                    (384, 128, 1, 1, 6, 6)])
def test_dgrad_via_forward_kernel_vs_autograd(cin, cout, k, stride, h, w):
    """dX = conv(dz [zero-inserted for stride 2], mirrored/transposed W) through ryolo_conv_bn_act_fwd, accumulate mode"""
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import layout as L
    lib = pkg._lib.lib
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(cin + k)
    b = 2
    x = bf(torch.randn(b, cin, h, w, generator=g)).to(dev).requires_grad_(True)
    wt = bf(torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).to(dev)
    oh, ow = (h + stride - 1) // stride, (w + stride - 1) // stride
    dz = bf(torch.randn(b, cout, oh, ow, generator=g)).to(dev)
    F.conv2d(x, wt, None, stride=stride, padding=(k - 1) // 2).backward(dz)
    bn = 256 if cout > 128 else (128 if cout > 64 else 64)
    cout_pad = L.round_up(cout, bn)
    dzb = L.to_padded_nhwc(dz, cout_pad)
    pt = pkg._lib.ptr
    stream = pkg._lib.stream_ptr(dev)
    if stride == 2:
        up = L.alloc_padded(b, h, w, cout_pad, dev)
        assert lib.ryolo_zero_insert2x(pt(dzb), cout_pad, b, oh, ow, cout_pad, pt(up), cout_pad, h, w, stream) == 0
        dzb = up
    gcs = L.round_up(cin, 64) if cin != 384 else 384
    prior = bf(torch.randn(b, cin, h, w, generator=g)).to(dev)
    gx = L.to_padded_nhwc(prior, gcs)                       # accumulate on top of an existing gradient
    desc = L.make_desc(b, h, w, cout, cout_pad, cin, gcs, k, 1, False, 0.0, True, gcs, False, False)
    wd = wt.flip(2, 3).permute(1, 0, 2, 3).contiguous()
    pw = L.pack_weights(desc, wd)
    zero_b = torch.zeros(2048, device=dev)
    L.conv_fwd(desc, dzb.data_ptr(), pw, zero_b, gx.data_ptr(), gx.data_ptr(), dev)
    torch.cuda.synchronize()
    got = L.from_padded_nhwc(gx, cin)
    want = x.grad + prior
    sc = float(want.abs().max())
    assert float((got - want).abs().max()) <= 2.0 ** -7 * sc, (float((got - want).abs().max()), sc)

