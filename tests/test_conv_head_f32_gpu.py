"""The fp32 NCHW head epilogue of conv_igemm_kernel (stride 1, no up-sampling): the fragment is transposed through the
staging area and each channel's pixels are stored as contiguous runs.  Checked against the fp32 PyTorch reference of the
same bf16-rounded op (1e-4 of the output scale, as in test_conv_gpu.py), at the head shapes of the 608 network with small
batches whose 128-pixel tiles cross image rows, halo pixels and image boundaries, and whose last tile is partial.  The
output lives inside a larger buffer whose sentinel regions before and after it must stay intact."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SENTINEL = 12345.5
PAD = 4096          # floats of sentinel on each side (a multiple of 4: the output stays 16-byte aligned)


@pytest.mark.parametrize("batch,hw,cin,cout,act", [
    (2, 76, 256, 504, False),     # 76^2 head: 2 * 78^2 = 12168 padded pixels, 95 full tiles + a partial one
    (3, 38, 512, 504, False),     # 38^2 head: 3 * 40^2 = 4800 padded pixels, partial last tile
    (2, 19, 1024, 504, False),    # 19^2 head
    (3, 13, 64, 100, True),       # BN = 128, 100 filters: the second 64-filter sub-tile is partly padding
    (2, 21, 64, 21, True),        # BN = 64, 21 filters
])
def test_head_f32_nchw_epilogue(batch, hw, cin, cout, act):
    from rotate_yolov3_b200 import layout as L
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(batch * 1000 + hw + cout)
    x = torch.randn(batch, cin, hw, hw, generator=g).to(dev).to(torch.bfloat16).float()
    wt = (torch.randn(cout, cin, 1, 1, generator=g) / cin ** 0.5).to(dev).to(torch.bfloat16).float()
    bias = torch.randn(cout, generator=g).to(dev)
    slope = 0.1
    xb = L.to_padded_nhwc(x, L.round_up(cin, 64))
    desc = L.make_desc(batch, hw, hw, cin, L.round_up(cin, 64), cout, 0, 1, 1, act, slope, False, 0, False, True)
    bn = 256 if cout > 128 else (128 if cout > 64 else 64)
    desc.cout_stride = L.round_up(cout, bn)
    pw = L.pack_weights(desc, wt)
    pb = L.padded_bias(desc, bias)
    n = batch * cout * hw * hw
    buf = torch.full((PAD + n + PAD,), SENTINEL, device=dev)
    y = buf[PAD:PAD + n].view(batch, cout, hw, hw)
    L.conv_fwd(desc, xb.data_ptr(), pw, pb, y.data_ptr(), None, dev)
    torch.cuda.synchronize()
    want = F.conv2d(x, wt, bias)
    if act:
        want = torch.where(want > 0, want, slope * want)
    scale = float(want.abs().max())
    err = float((y - want).abs().max())
    assert err <= 1e-4 * scale, (err, scale)
    assert bool((buf[:PAD] == SENTINEL).all()) and bool((buf[PAD + n:] == SENTINEL).all())
