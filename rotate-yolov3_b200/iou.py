"""Rotated-box IoU behind the reference's signature ``skew_bbox_iou(box1, box2, GIoU=False)``
(utils/utils.py:290-320), plus the batched all-pairs form the reference can only express as a Python loop
(test.py:134-151 calls it once per prediction)."""
import torch

from . import _lib


def _as_boxes(x, device):
    if isinstance(x, (list, tuple)):
        x = torch.tensor([float(v) for v in x], dtype=torch.float32, device=device)
    if not x.is_cuda:
        x = x.to(device)
    return x.to(torch.float32)


def skew_bbox_iou(box1, box2, GIoU=False):
    """box1: [5+] (list or tensor) or [N, 5+]; box2: [N, 5+] -> FloatTensor[N] on CUDA.
    Broadcast rules of the reference (utils/utils.py:294-297): a 1-D box1 is unsqueezed, and if the shapes
    still differ box1 is repeated len(box2) times."""
    dev = box2.device if isinstance(box2, torch.Tensor) and box2.is_cuda else (
        box1.device if isinstance(box1, torch.Tensor) and box1.is_cuda else torch.device("cuda", torch.cuda.current_device()))
    box1 = _as_boxes(box1, dev)
    box2 = _as_boxes(box2, dev)
    if box1.dim() < box2.dim():
        box1 = box1.unsqueeze(0)
    if box1.shape != box2.shape:
        box1 = box1.repeat(len(box2), 1)
    a = box1[:, :5].contiguous()
    b = box2[:, :5].contiguous()
    n = b.shape[0]
    out = torch.empty((n,), dtype=torch.float32, device=dev)
    if n == 0:
        return out
    with torch.cuda.device(dev):
        st = _lib.lib.ryolo_riou_paired(_lib.ptr(a), _lib.ptr(b), n, 5, 5,
                                        _lib.IOU_MODE_GIOU if GIoU else _lib.IOU_MODE_IOU, _lib.ptr(out),
                                        _lib.stream_ptr(dev))
    _lib.check(st, "ryolo_riou_paired")
    return out


def rotated_iou_matrix(a, b, GIoU=False, out=None):
    """All-pairs form: a [N, 5+], b [M, 5+] float32 CUDA -> [N, M] with out[i, j] = skew_bbox_iou(a[i], b[j:j+1])."""
    assert a.is_cuda and b.is_cuda
    a = a.to(torch.float32)
    b = b.to(torch.float32)
    if a.stride(-1) != 1 or (a.shape[0] > 1 and a.stride(0) < 5):
        a = a.contiguous()
    if b.stride(-1) != 1 or (b.shape[0] > 1 and b.stride(0) < 5):
        b = b.contiguous()
    n, m = a.shape[0], b.shape[0]
    if out is None:
        out = torch.empty((n, m), dtype=torch.float32, device=a.device)
    elif (out.dtype != torch.float32 or tuple(out.shape) != (n, m) or out.device != a.device
          or not out.is_contiguous()):
        # the kernel writes out as a dense row-major fp32 [n, m] block
        raise ValueError("rotated_iou_matrix: out must be a contiguous float32 [%d, %d] tensor on %s, got %s %s %s%s"
                         % (n, m, a.device, out.dtype, tuple(out.shape), out.device,
                            "" if out.is_contiguous() else " (not contiguous)"))
    if n == 0 or m == 0:
        return out
    sa = a.stride(0) if n > 1 else a.shape[1]
    sb = b.stride(0) if m > 1 else b.shape[1]
    with torch.cuda.device(a.device):
        st = _lib.lib.ryolo_riou_pairwise(_lib.ptr(a), n, sa, _lib.ptr(b), m, sb,
                                          _lib.IOU_MODE_GIOU if GIoU else _lib.IOU_MODE_IOU, _lib.ptr(out),
                                          _lib.stream_ptr(a.device))
    _lib.check(st, "ryolo_riou_pairwise")
    return out


class _RotatedIoU(torch.autograd.Function):
    """IoU of paired rotated boxes with analytic gradients w.r.t. both boxes (csrc/riou_grad.cu)."""

    @staticmethod
    def forward(ctx, a, b):
        ctx.in_meta = ((a.shape, a.dtype), (b.shape, b.dtype))
        a = a[:, :5].contiguous().float()
        b = b[:, :5].contiguous().float()
        n = a.shape[0]
        out = torch.empty(n, dtype=torch.float32, device=a.device)
        with torch.cuda.device(a.device):
            st = _lib.lib.ryolo_riou_paired_grad(_lib.ptr(a), _lib.ptr(b), n, 5, 5, None, _lib.ptr(out), None, None,
                                                 _lib.stream_ptr(a.device))
        _lib.check(st, "ryolo_riou_paired_grad")
        ctx.save_for_backward(a, b)
        return out

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        n = a.shape[0]
        g = g.contiguous().float()
        ga = torch.empty_like(a) if ctx.needs_input_grad[0] else None
        gb = torch.empty_like(b) if ctx.needs_input_grad[1] else None
        with torch.cuda.device(a.device):
            st = _lib.lib.ryolo_riou_paired_grad(_lib.ptr(a), _lib.ptr(b), n, 5, 5, _lib.ptr(g), None,
                                                 _lib.ptr(ga) if ga is not None else None,
                                                 _lib.ptr(gb) if gb is not None else None, _lib.stream_ptr(a.device))
        _lib.check(st, "ryolo_riou_paired_grad")
        return _widen(ga, *ctx.in_meta[0]), _widen(gb, *ctx.in_meta[1])


def _widen(g, shape, dtype):
    """[N, 5] fp32 gradient -> the input's shape and dtype; the columns beyond the box get zero"""
    if g is None or (g.shape == shape and g.dtype == dtype):
        return g
    full = torch.zeros(shape, dtype=dtype, device=g.device)
    full[:, :5] = g
    return full


def rotated_iou(box1, box2):
    """differentiable IoU of paired rotated boxes: box1, box2 [N, >=5] (cx, cy, w, h, theta, ...) CUDA -> [N]; the
    gradients have the inputs' shapes and dtypes (zero beyond column 5)"""
    if not (box1.is_cuda and box2.is_cuda):
        raise RuntimeError("rotated_iou needs CUDA tensors (sm_90a kernels, no CPU fallback)")
    return _RotatedIoU.apply(box1, box2)


def riou_loss(pred, target, reduction="mean"):
    """rotated-IoU regression loss 1 - IoU(pred, target) (the README's 'riou loss'; the reference's compute_loss uses
    SmoothL1 + a horizontal wh_iou instead, SURVEY.md D1).  pred, target [N, >=5] rows; gradients flow to both."""
    loss = 1.0 - rotated_iou(pred, target)
    if reduction == "mean":
        return loss.mean() if loss.numel() else loss.sum()
    if reduction == "sum":
        return loss.sum()
    return loss
