"""The TMA-store epilogue of conv_igemm_kernel (same-grid bf16 outputs: training forward z, every dgrad, eval stride-1
blocks): the output map clips the stores to `store_cols` channels and `np` rows, so channels beyond the view, the halo
and the neighbours in a wider (concat) buffer must come out exactly as the layout requires.  Every case is compared with
F.conv2d at the tolerances of test_conv_gpu.py, and every byte outside the view's interior is checked."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SENTINEL = 5.0    # neighbouring channels of the buffer: must never be written
GARBAGE = 9.0     # halo of the view's channels before the call: the kernel stores zeros there


def _run(batch, h, w, cin, cout, k, width, off=0, acc=False, res_sep=False, seed=0):
    from rotate_yolov3_b200 import layout as L
    dev = torch.device("cuda")
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(batch, cin, h, w, generator=g).to(torch.bfloat16).float().to(dev)
    wt = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).to(torch.bfloat16).float().to(dev)
    act = not acc                       # a dgrad accumulate is linear with zero bias
    bias = torch.zeros(cout, device=dev) if acc else torch.randn(cout, generator=g).to(dev)
    store_cols = L.round_up(cout, 32)
    xb = L.to_padded_nhwc(x)
    buf = L.alloc_padded(batch, h, w, width, dev)
    buf.fill_(SENTINEL)
    buf[..., off:off + store_cols] = GARBAGE
    buf[:, 1:-1, 1:-1, off:off + store_cols] = 0.0
    res_t, res_ptr, res_stride = None, None, 0
    if acc:                             # the residual IS the output view (dgrad into an already written gradient)
        res_t = torch.randn(batch, cout, h, w, generator=g).to(torch.bfloat16).float().to(dev)
        buf[:, 1:-1, 1:-1, off:off + cout] = res_t.permute(0, 2, 3, 1).to(torch.bfloat16)
        res_ptr, res_stride = buf.data_ptr() + 2 * off, width
    elif res_sep:                       # shortcut from a separate buffer
        res_t = torch.randn(batch, cout, h, w, generator=g).to(torch.bfloat16).float().to(dev)
        rb = L.to_padded_nhwc(res_t, L.round_up(cout, 64) + 64)
        res_ptr, res_stride = rb.data_ptr(), rb.shape[-1]
    desc = L.make_desc(batch, h, w, cin, xb.shape[-1], cout, width, k, 1, act, 0.1, res_t is not None, res_stride)
    pw = L.pack_weights(desc, wt)
    pb = L.padded_bias(desc, bias)
    L.conv_fwd(desc, xb.data_ptr(), pw, pb, buf.data_ptr() + 2 * off, res_ptr, dev)
    torch.cuda.synchronize()

    y = F.conv2d(x, wt, bias, padding=(k - 1) // 2)
    if act:
        y = torch.where(y > 0, y, 0.1 * y)
    want = y + res_t if res_t is not None else y
    scale = float(want.abs().max())
    got = L.from_padded_nhwc(buf, cout, off)
    err = (got - want).abs()
    tol = 2.0 ** -8 * want.abs() + 1e-3 * scale * 2.0 ** -8 + 1e-6
    assert bool((err <= tol).all()), (float(err.max()), scale)
    view = buf[..., off:off + store_cols]
    assert float(view[:, 0].abs().max()) == 0 and float(view[:, -1].abs().max()) == 0
    assert float(view[:, :, 0].abs().max()) == 0 and float(view[:, :, -1].abs().max()) == 0
    if store_cols > cout:
        assert float(view[:, 1:-1, 1:-1, cout:].abs().max()) == 0
    for lo, hi in ((0, off), (off + store_cols, width)):
        if hi > lo:
            assert bool((buf[..., lo:hi] == SENTINEL).all()), (lo, hi)


@pytest.mark.parametrize("cfg", [
    # dgrad accumulating into a channel-offset view of a wider concat gradient buffer, halo garbage zeroed
    dict(batch=2, h=19, w=19, cin=128, cout=96, k=3, width=256, off=32, acc=True),
    dict(batch=2, h=38, w=38, cin=128, cout=256, k=1, width=768, off=256, acc=True),
    # np = 8 * 47 * 47 = 17672 = 138 * 128 + 8: partial last tile, 278 tiles (several per persistent CTA) + shortcut
    dict(batch=8, h=45, w=45, cin=64, cout=512, k=3, width=512, res_sep=True),
    # store_cols < BN in a wider buffer: 160 of 256 (the fourth 64-filter box lies wholly beyond), 96 of 128
    dict(batch=2, h=20, w=16, cin=64, cout=160, k=3, width=320),
    dict(batch=3, h=13, w=11, cin=192, cout=96, k=1, width=224),
])
def test_tma_store_epilogue_vs_torch(cfg):
    _run(**cfg)
