"""The residual of the same-grid conv epilogue (dgrad accumulate, eval shortcut) is loaded into the staging tile by TMA
and added there.  Exact oracle built from the kernel itself: the same launch with an fp32 output and no residual gives
act(acc + bias) in fp32 for the same tile width (the per-element wgmma result does not depend on how the output
leaves), so the bf16 output with the residual must equal (y32 + residual) rounded to bf16 bit for bit, and the bf16
output without it must equal y32 rounded to bf16.  The layout of every case (halo garbage stored as zeros, filters at
and above cout, the neighbours in a wider buffer) is checked by the TMA-store epilogue test's runner."""
import pytest
import torch

from builders import TMA_GARBAGE, TMA_SENTINEL, tma_epilogue_run

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.contiguous().view(torch.int16)


def _interior(buf, c, off):
    """bf16 [B, c, H, W] of the channels [off, off + c) of a padded-NHWC buffer"""
    return buf[:, 1:-1, 1:-1, off:off + c].permute(0, 3, 1, 2).contiguous()


def _exact(batch, h, w, cin, cout, k, width, off=0, acc=False, res_sep=False, seed=0):
    from rotate_yolov3_b200 import layout as L
    dev = torch.device("cuda")
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(batch, cin, h, w, generator=g).to(dev)
    wt = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).to(dev)
    act = not acc                       # a dgrad accumulate is linear with zero bias
    bias = torch.zeros(cout, device=dev) if acc else torch.randn(cout, generator=g).to(dev)
    res = torch.randn(batch, cout, h, w, generator=g).to(torch.bfloat16).to(dev)
    xb = L.to_padded_nhwc(x)
    store_cols = L.round_up(cout, 32)

    def launch(out_ptr, res_ptr=None, res_stride=0, out_f32=False, cout_stride=width):
        desc = L.make_desc(batch, h, w, cin, xb.shape[-1], cout, cout_stride, k, 1, act, 0.1, res_ptr is not None,
                           res_stride, out_f32=out_f32)
        L.conv_fwd(desc, xb.data_ptr(), L.pack_weights(desc, wt), L.padded_bias(desc, bias), out_ptr, res_ptr, dev)

    y32 = torch.empty(batch, cout, h, w, device=dev)
    launch(y32.data_ptr(), out_f32=True, cout_stride=cout)

    def buffer():
        buf = L.alloc_padded(batch, h, w, width, dev)
        buf.fill_(TMA_SENTINEL)
        buf[..., off:off + store_cols] = TMA_GARBAGE
        buf[:, 1:-1, 1:-1, off:off + store_cols] = 0.0
        return buf

    plain = buffer()
    launch(plain.data_ptr() + 2 * off)
    torch.cuda.synchronize()
    assert torch.equal(_bits(_interior(plain, cout, off)), _bits(y32.to(torch.bfloat16)))

    # garbage in the residual's halo and in its channels at and above cout: neither may reach the output
    out = buffer()
    if acc:                             # in place: the residual IS the output view
        out[:, 1:-1, 1:-1, off:off + cout] = res.permute(0, 2, 3, 1)
        out[:, 1:-1, 1:-1, off + cout:off + store_cols] = TMA_GARBAGE
        res_ptr, res_stride = out.data_ptr() + 2 * off, width
    else:                               # a separate buffer with a wider channel stride than the output
        rb = L.to_padded_nhwc(res, L.round_up(cout, 64) + 64)
        rb[:, 0] = TMA_GARBAGE
        rb[..., cout:] = TMA_GARBAGE
        res_ptr, res_stride = rb.data_ptr(), rb.shape[-1]
    launch(out.data_ptr() + 2 * off, res_ptr, res_stride)
    torch.cuda.synchronize()
    want = (y32 + res.float()).to(torch.bfloat16)
    got = _interior(out, cout, off)
    bad = _bits(got) != _bits(want)
    assert not bool(bad.any()), (int(bad.sum()), float((got.float() - want.float()).abs().max()))
    if store_cols > cout:
        assert float(out[:, 1:-1, 1:-1, off + cout:off + store_cols].abs().max()) == 0


CASES = [
    # the accumulating 1x1 dgrads of the training step at their grid and channel counts (as convolutions: the
    # forward's cout -> its cin), in place; 304^2 and 152^2 end in a partial tile and run several tiles per CTA
    dict(batch=1, h=304, w=304, cin=32, cout=64, k=1, width=64, acc=True),
    dict(batch=2, h=152, w=152, cin=64, cout=128, k=1, width=128, acc=True),
    dict(batch=2, h=76, w=76, cin=128, cout=256, k=1, width=256, acc=True),
    dict(batch=2, h=38, w=38, cin=256, cout=512, k=1, width=512, acc=True),
    dict(batch=4, h=19, w=19, cin=512, cout=1024, k=1, width=1024, acc=True),
    # in place into a channel-offset view of a wider concat gradient buffer, sentinel neighbours on both sides
    dict(batch=2, h=38, w=38, cin=256, cout=512, k=1, width=768, off=128, acc=True),
    # separate residual buffer with a wider stride, PReLU; np = 17672 = 138 * 128 + 8: partial last tile, 278 tiles
    dict(batch=8, h=45, w=45, cin=64, cout=512, k=3, width=512, res_sep=True),
    dict(batch=3, h=30, w=26, cin=64, cout=128, k=3, width=192, off=64, res_sep=True),
    # residual zero-filled at and above cout: 40 of BN 64, 160 of BN 256 (store_cols 160 < BN)
    dict(batch=2, h=20, w=16, cin=64, cout=40, k=1, width=128, off=64, acc=True),
    dict(batch=2, h=20, w=16, cin=64, cout=160, k=3, width=320, off=64, acc=True),
    dict(batch=2, h=20, w=16, cin=64, cout=160, k=3, width=160, res_sep=True),
]


def _case_id(c):
    return "%dx%d_%d-%d_k%d_w%d_o%d_%s" % (c["h"], c["w"], c["cin"], c["cout"], c["k"], c["width"], c.get("off", 0),
                                            "acc" if c.get("acc") else "sep")


@pytest.mark.parametrize("cfg", CASES, ids=_case_id)
def test_residual_epilogue_exact(cfg):
    _exact(**cfg)


@pytest.mark.parametrize("cfg", CASES, ids=_case_id)
def test_residual_epilogue_layout(cfg):
    r = tma_epilogue_run(**cfg)
    assert r["within"] and r["halo_zero"] and r["pad_zero"] and r["sentinels"], r
