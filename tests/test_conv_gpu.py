"""wgmma implicit-GEMM conv blocks vs a plain PyTorch fp32 reference of the same op (conv2d + bias + PReLU
[+ residual] [+ nearest x2]).  Inputs/weights are rounded to bf16 first (the kernel's operand type), so the only
differences are fp32 accumulation order (fp32-NCHW outputs: 1e-4 relative to the layer's output scale, the
north_star tolerance) and the final bf16 rounding (bf16 outputs: 1 bf16 ulp = 2^-8 relative)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _ref(x, w, b, stride, slope, act, res=None, up=False):
    k = w.shape[-1]
    y = F.conv2d(x, w, b, stride=stride, padding=(k - 1) // 2)
    if act:
        y = torch.where(y > 0, y, slope * y)
    if res is not None:
        y = y + res
    if up:
        y = F.interpolate(y, scale_factor=2, mode="nearest")
    return y


def _run(batch, h, w, cin, cout, k, stride=1, act=True, residual=False, up=False, f32=False, seed=0, cin_extra=0,
         cout_extra=0, narrow=False):
    from rotate_yolov3_b200 import layout as L
    dev = torch.device("cuda")
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(batch, cin, h, w, generator=g).to(dev).to(torch.bfloat16).float()
    wt = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).to(dev).to(torch.bfloat16).float()
    bias = torch.randn(cout, generator=g).to(dev)
    slope = 0.1
    oh, ow = (h + stride - 1) // stride, (w + stride - 1) // stride
    cin_cs = L.round_up(cin, 64) + cin_extra
    if narrow:                                   # 32-channel-granular buffers: TMA zero-fills the rest of the K chunk
        cin_cs = L.round_up(cin, 32)
    xb = L.to_padded_nhwc(x, cin_cs)
    if cin_extra:
        xb[..., L.round_up(cin, 64):] = 7.0      # neighbouring channels of a concat buffer must not leak in
    desc = L.make_desc(batch, h, w, cin, cin_cs, cout, 0, k, stride, act, slope, residual, 0, up, f32)
    bn = 256 if cout > 128 else (128 if cout > 64 else 64)
    cout_pad = L.round_up(cout, bn)
    cout_cs = L.round_up(cout, 32) if narrow else cout_pad + cout_extra
    desc.cout_stride = cout_cs
    res_t, res_buf = None, None
    if residual:
        res_t = torch.randn(batch, cout, oh, ow, generator=g).to(dev).to(torch.bfloat16).float()
        res_buf = L.to_padded_nhwc(res_t, cout_pad + 64)
        desc.res_stride = cout_pad + 64
    pw = L.pack_weights(desc, wt)
    pb = L.padded_bias(desc, bias)
    assert pb.numel() == cout_pad
    if f32:
        y = torch.full((batch, cout, oh, ow), float("nan"), device=dev)
    else:
        y = L.alloc_padded(batch, oh * (2 if up else 1), ow * (2 if up else 1), cout_cs, dev)
        if cout_extra:
            y[:, 1:-1, 1:-1, (cout + 31) // 32 * 32:] = 3.0
    L.conv_fwd(desc, xb.data_ptr(), pw, pb, y.data_ptr(), res_buf.data_ptr() if residual else None, dev)
    torch.cuda.synchronize()
    want = _ref(x, wt, bias, stride, slope, act, res_t, up)
    scale = float(want.abs().max())
    if f32:
        got = y
        err = float((got - want).abs().max())
        assert err <= 1e-4 * scale, (err, scale)
    else:
        got = L.from_padded_nhwc(y, cout)
        err = (got - want).abs()
        tol = 2.0 ** -8 * want.abs() + 1e-3 * scale * 2.0 ** -8 + 1e-6
        assert bool((err <= tol).all()), (float(err.max()), scale)
        # halo untouched (zero), channel padding zero, neighbours of a wider buffer untouched
        assert float(y[:, 0].abs().max()) == 0 and float(y[:, -1].abs().max()) == 0
        assert float(y[:, :, 0].abs().max()) == 0 and float(y[:, :, -1].abs().max()) == 0
        if cout_cs > cout and not cout_extra:
            assert float(y[:, 1:-1, 1:-1, cout:cout_cs].abs().max()) == 0     # zero-initialised, chunk-padded or untouched
        if cout_extra:
            assert float((y[:, 1:-1, 1:-1, (cout + 31) // 32 * 32:] - 3.0).abs().max()) == 0
    return err


@pytest.mark.parametrize("cfg", [
    dict(batch=1, h=8, w=8, cin=64, cout=64, k=1),                                  # smallest GEMM, BN=64
    dict(batch=2, h=19, w=19, cin=64, cout=128, k=3),                               # 9 taps, BN=128
    dict(batch=2, h=19, w=19, cin=128, cout=256, k=3, residual=True),               # BN=256 + shortcut add
    dict(batch=3, h=38, w=38, cin=256, cout=128, k=1, up=True, cout_extra=256),     # upsample into a concat buffer
    dict(batch=2, h=16, w=20, cin=32, cout=64, k=3, stride=2),                      # stride 2, cin padded 32->64
    dict(batch=2, h=19, w=19, cin=128, cout=504, k=1, act=False, f32=True),         # linear head, fp32 NCHW, 504 = 2 n-tiles
    dict(batch=1, h=76, w=76, cin=128, cout=256, k=3),                              # many m-tiles (persistent loop)
    dict(batch=2, h=38, w=38, cin=768, cout=256, k=1, cin_extra=0),                 # long K (12 chunks)
    dict(batch=2, h=19, w=19, cin=64, cout=32, k=1, cin_extra=128),                 # cout padded 32->64, wide input buffer
    dict(batch=1, h=19, w=19, cin=512, cout=1024, k=3),                             # 4 n-tiles x 72 k-steps
    dict(batch=2, h=12, w=16, cin=64, cout=32, k=1, up=True, cout_extra=64),        # 32 filters at offset 0 of a wider (concat) buffer: neighbours intact
    dict(batch=2, h=20, w=16, cin=32, cout=64, k=3, narrow=True),                   # 32-channel input buffer (stride 32 < K chunk)
    dict(batch=2, h=20, w=16, cin=64, cout=32, k=1, narrow=True),                   # 32-channel output buffer
    dict(batch=1, h=10, w=12, cin=160, cout=96, k=3, narrow=True),                  # strides 160 / 96: partial last K chunk
])
def test_conv_block_vs_torch(cfg):
    _run(**cfg)


@pytest.mark.parametrize("cout,cs,shape", [(32, 64, (2, 40, 56)), (32, 32, (3, 38, 50)), (16, 32, (1, 26, 26))])
def test_first_layer_tensor_core_conv(cout, cs, shape):
    """3 -> cout first layer on the tensor pipe (register im2col, image as bf16 hi+lo) vs an fp32 conv with the same
    bf16-rounded weights: within one bf16 ulp of the output; padding channels and halo zero."""
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import layout as L
    dev = torch.device("cuda")
    b, h, wd = shape
    g = torch.Generator().manual_seed(1)
    x = torch.rand(b, 3, h, wd, generator=g).to(dev)
    w = (torch.randn(cout, 3, 3, 3, generator=g) / 5).to(dev)
    bias = torch.randn(cout, generator=g).to(dev)
    y = L.alloc_padded(b, h, wd, cs, dev)
    y[:, 1:-1, 1:-1, cout:] = 5.0
    st = pkg._lib.lib.ryolo_conv_first_fwd(pkg._lib.ptr(x), b, h, wd, pkg._lib.ptr(w), pkg._lib.ptr(bias), cout, 0.1,
                                           pkg._lib.ptr(y), cs, pkg._lib.stream_ptr(dev))
    assert st == 0, pkg._lib.last_error()
    want = _ref(x, w.to(torch.bfloat16).float(), bias, 1, 0.1, True)
    got = L.from_padded_nhwc(y, cout)
    assert bool(((got - want).abs() <= 2.0 ** -8 * want.abs() + 2e-5).all()), float((got - want).abs().max())
    if cs > cout:
        assert float(y[..., cout:].abs().max()) == 0      # channel padding zeroed for the next layer's 64-wide K chunk
    assert float(y[:, 0].abs().max()) == 0 and float(y[:, :, 0].abs().max()) == 0
    # the same values written straight into the space-to-depth layout of a following stride-2 layer
    xs = L.alloc_padded(b, h // 2, wd // 2, L.round_up(4 * cout, 64), dev)
    st = pkg._lib.lib.ryolo_conv_first_s2d_fwd(pkg._lib.ptr(x), b, h, wd, pkg._lib.ptr(w), pkg._lib.ptr(bias), cout, 0.1,
                                               pkg._lib.ptr(xs), xs.shape[-1], pkg._lib.stream_ptr(dev))
    assert st == 0, pkg._lib.last_error()
    xs_want = L.alloc_padded(b, h // 2, wd // 2, L.round_up(4 * cout, 64), dev)
    st = pkg._lib.lib.ryolo_space_to_depth(pkg._lib.ptr(y), cs, b, h, wd, cout, pkg._lib.ptr(xs_want), xs_want.shape[-1],
                                           pkg._lib.stream_ptr(dev))
    assert st == 0, pkg._lib.last_error()
    torch.cuda.synchronize()
    assert torch.equal(xs, xs_want)


@pytest.mark.parametrize("cfg", [
    dict(batch=2, h=19, w=19, cin=64, cout=64, k=3),
    dict(batch=2, h=19, w=19, cin=128, cout=256, k=3),
    dict(batch=3, h=38, w=38, cin=256, cout=128, k=1),
    dict(batch=1, h=20, w=16, cin=32, cout=64, k=3),        # channel padding on the K... N side (cin 32 -> 64)
    dict(batch=2, h=19, w=19, cin=768, cout=256, k=1),      # cin_pad 768 = 3 n-tiles of 256
    dict(batch=4, h=38, w=38, cin=128, cout=504, k=1),      # cout_pad 512
    dict(batch=2, h=20, w=16, cin=32, cout=32, k=3, narrow=True),    # both operands in 32-channel buffers
    dict(batch=2, h=10, w=12, cin=160, cout=96, k=1, narrow=True),   # strides 160 / 96 (not tile multiples)
])
def test_conv_wgrad_vs_torch(cfg):
    """wgmma wgrad (K = pixels, MN-major operands, split-K partials added in split order) vs
    torch.nn.grad.conv2d_weight in fp32 on the same bf16-representable operands; tolerance 2e-3 of the gradient scale
    (the fp32 reference adds in yet another order).  The element-wise float64 bounds, the ksize 2 (space-to-depth) path
    and uneven split counts are in tests/test_wgrad_gpu.py."""
    import ctypes
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import layout as L
    b, h, w, cin, cout, k = (cfg[n] for n in ("batch", "h", "w", "cin", "cout", "k"))
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(5)
    x = torch.randn(b, cin, h, w, generator=g).to(dev).to(torch.bfloat16).float()
    dz = torch.randn(b, cout, h, w, generator=g).to(dev).to(torch.bfloat16).float()
    cin_pad = L.round_up(cin, 64)
    bn = 256 if cout > 128 else (128 if cout > 64 else 64)
    cout_pad = L.round_up(cout, bn)
    xcs = L.round_up(cin, 32) if cfg.get("narrow") else cin_pad
    zcs = L.round_up(cout, 32) if cfg.get("narrow") else cout_pad
    xb = L.to_padded_nhwc(x, xcs)
    dzb = L.to_padded_nhwc(dz, zcs)
    dw = torch.zeros((k * k, cout_pad, cin_pad), dtype=torch.float32, device=dev)
    st = pkg._lib.lib.ryolo_conv_wgrad(pkg._lib.ptr(dzb), zcs, cout_pad, pkg._lib.ptr(xb), xcs, cin_pad, b, h, w, k,
                                       pkg._lib.ptr(dw), pkg._lib.stream_ptr(dev))
    assert st == 0, pkg._lib.last_error()
    torch.cuda.synchronize()
    want = torch.nn.grad.conv2d_weight(x, (cout, cin, k, k), dz, stride=1, padding=(k - 1) // 2)
    got = dw.view(k, k, cout_pad, cin_pad)[:, :, :cout, :cin].permute(2, 3, 0, 1)
    scale = float(want.abs().max())
    assert float((got - want).abs().max()) <= 2e-3 * scale, (float((got - want).abs().max()), scale)
    assert float(dw.view(k, k, cout_pad, cin_pad)[:, :, cout:].abs().max() if cout_pad > cout else 0.0) == 0.0


@pytest.mark.parametrize("cin,cout,h,w", [(32, 64, 16, 20), (64, 128, 38, 38), (256, 512, 12, 10)])
def test_stride2_via_space_to_depth_vs_torch(cin, cout, h, w):
    """3x3/stride-2/pad-1 conv = space-to-depth + 2x2-tap stride-1 implicit GEMM (ksize = 2) with remapped weights"""
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200 import layout as L
    lib = pkg._lib.lib
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(cin)
    b = 2
    x = torch.randn(b, cin, h, w, generator=g).to(dev).to(torch.bfloat16).float()
    wt = (torch.randn(cout, cin, 3, 3, generator=g) / (cin * 9) ** 0.5).to(dev).to(torch.bfloat16).float()
    bias = torch.randn(cout, generator=g).to(dev)
    xb = L.to_padded_nhwc(x, L.round_up(cin, 64))
    xs = L.alloc_padded(b, h // 2, w // 2, L.round_up(4 * cin, 64), dev)
    assert lib.ryolo_space_to_depth(pkg._lib.ptr(xb), xb.shape[-1], b, h, w, cin, pkg._lib.ptr(xs), xs.shape[-1],
                                    pkg._lib.stream_ptr(dev)) == 0
    bn = 256 if cout > 128 else (128 if cout > 64 else 64)
    cout_pad = L.round_up(cout, bn)
    desc = L.make_desc(b, h // 2, w // 2, 4 * cin, xs.shape[-1], cout, cout_pad, 2, 1, True, 0.1)
    pw = L.pack_weights(desc, L.s2d_weight(wt))
    pb = L.padded_bias(desc, bias)
    y = L.alloc_padded(b, h // 2, w // 2, cout_pad, dev)
    L.conv_fwd(desc, xs.data_ptr(), pw, pb, y.data_ptr(), None, dev)
    torch.cuda.synchronize()
    want = _ref(x, wt, bias, 2, 0.1, True)
    got = L.from_padded_nhwc(y, cout)
    err = (got - want).abs()
    assert bool((err <= 2.0 ** -8 * want.abs() + 1e-3 * float(want.abs().max()) * 2.0 ** -8 + 1e-6).all()), float(err.max())
    # adjoint pair: depth_to_space(space_to_depth(x)) == x, accumulate doubles it
    back = L.alloc_padded(b, h, w, xb.shape[-1], dev)
    assert lib.ryolo_depth_to_space(pkg._lib.ptr(xs), xs.shape[-1], b, h, w, cin, pkg._lib.ptr(back), back.shape[-1], 0,
                                    pkg._lib.stream_ptr(dev)) == 0
    assert torch.equal(L.from_padded_nhwc(back, cin), x)
    assert lib.ryolo_depth_to_space(pkg._lib.ptr(xs), xs.shape[-1], b, h, w, cin, pkg._lib.ptr(back), back.shape[-1], 1,
                                    pkg._lib.stream_ptr(dev)) == 0
    assert torch.allclose(L.from_padded_nhwc(back, cin), 2 * x, rtol=1e-2, atol=1e-2)
