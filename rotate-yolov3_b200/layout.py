"""Padded-NHWC bf16 activation layout helpers (see include/ryolo.h, conv section) and the thin Python binding of
the conv entry points.  Pure tensor plumbing: allocation and layout conversion for tests / model I/O."""
import ctypes

import torch

from . import _lib


def round_up(x, m):
    return (x + m - 1) // m * m


def alloc_padded(batch, h, w, cs, device):
    """[B, H+2, W+2, Cs] bf16, zero everywhere (the halo must stay zero; kernels never write it)."""
    return torch.zeros((batch, h + 2, w + 2, cs), dtype=torch.bfloat16, device=device)


def to_padded_nhwc(x_nchw, cs=None):
    b, c, h, w = x_nchw.shape
    cs = cs or round_up(c, 64)
    buf = alloc_padded(b, h, w, cs, x_nchw.device)
    buf[:, 1:h + 1, 1:w + 1, :c] = x_nchw.permute(0, 2, 3, 1).to(torch.bfloat16)
    return buf


def from_padded_nhwc(buf, c, ch_offset=0):
    h, w = buf.shape[1] - 2, buf.shape[2] - 2
    return buf[:, 1:h + 1, 1:w + 1, ch_offset:ch_offset + c].permute(0, 3, 1, 2).float().contiguous()


def make_desc(batch, in_h, in_w, cin, cin_stride, cout, cout_stride, ksize, stride=1, has_act=True, slope=0.1,
              has_residual=False, res_stride=0, upsample2x=False, out_f32=False):
    return _lib.ConvDesc(batch, in_h, in_w, cin, cin_stride, cout, cout_stride, ksize, stride, int(has_act),
                         float(slope), int(has_residual), res_stride, int(upsample2x),
                         _lib.DT_F32 if out_f32 else _lib.DT_BF16)


def pack_weights(desc, weight, scale=None, mode=0, out=None):
    """fp32 CUDA conv weight (+ optional per-filter scale) -> packed bf16 GEMM operand (uint8 tensor).  mode: see
    ryolo_conv_pack_weights_ex (0 plain, 1 dgrad of plain, 2 space-to-depth, 3 dgrad of space-to-depth); for modes
    1-3 `weight` is the ORIGINAL nn.Conv2d weight and the transform happens inside the packing kernel."""
    if out is None:
        nbytes = _lib.lib.ryolo_conv_packed_weight_bytes(ctypes.byref(desc))
        out = torch.empty(nbytes, dtype=torch.uint8, device=weight.device)
    w = weight.detach()
    if w.dtype != torch.float32 or not w.is_contiguous():
        w = w.float().contiguous()
    s = scale.detach().float().contiguous() if scale is not None else None
    st = _lib.lib.ryolo_conv_pack_weights_ex(ctypes.byref(desc), _lib.ptr(w), _lib.ptr(s) if s is not None else None,
                                             _lib.ptr(out), mode, _lib.stream_ptr(weight.device))
    _lib.check(st, "ryolo_conv_pack_weights_ex")
    return out


def padded_bias(desc, bias):
    cout_pad = _lib.lib.ryolo_conv_packed_weight_bytes(ctypes.byref(desc)) // (2 * desc.ksize * desc.ksize * round_up(desc.cin, 64))
    b = torch.zeros(cout_pad, dtype=torch.float32, device=bias.device)
    b[:desc.cout] = bias.detach().float()
    return b


_S2D_K = {(0, 1): 0, (1, 0): 1, (1, 1): 2}   # (tap q, phase p) -> original kernel index; (0, 0) has no contribution


def s2d_weight(w):
    """[cout, C, 3, 3] weights of a 3x3/stride-2/pad-1 conv -> [cout, 4C, 2, 2] weights of the equivalent 2x2-tap
    stride-1 conv on the space-to-depth input (channel = (py*2+px)*C + c, tap (qy, qx) at offset (qy-1, qx-1))."""
    cout, c = w.shape[0], w.shape[1]
    w2 = torch.zeros((cout, 4, c, 2, 2), dtype=w.dtype, device=w.device)
    for (qy, py), kh in _S2D_K.items():
        for (qx, px), kw in _S2D_K.items():
            w2[:, py * 2 + px, :, qy, qx] = w[:, :, kh, kw]
    return w2.reshape(cout, 4 * c, 2, 2)


def s2d_weight_grad(dw2, c):
    """inverse gather of s2d_weight for gradients: [cout, 4C, 2, 2] -> [cout, C, 3, 3]"""
    cout = dw2.shape[0]
    d = dw2.reshape(cout, 4, c, 2, 2)
    dw = torch.zeros((cout, c, 3, 3), dtype=dw2.dtype, device=dw2.device)
    for (qy, py), kh in _S2D_K.items():
        for (qx, px), kw in _S2D_K.items():
            dw[:, :, kh, kw] = d[:, py * 2 + px, :, qy, qx]
    return dw


def conv_fwd(desc, x_ptr, packed_w, bias, y_ptr, residual_ptr=None, device=None):
    st = _lib.lib.ryolo_conv_bn_act_fwd(ctypes.byref(desc), ctypes.c_void_p(x_ptr), _lib.ptr(packed_w), _lib.ptr(bias),
                                        ctypes.c_void_p(residual_ptr) if residual_ptr else None,
                                        ctypes.c_void_p(y_ptr), _lib.stream_ptr(device))
    _lib.check(st, "ryolo_conv_bn_act_fwd")
