"""Batched device-side prediction <-> ground-truth matching for mAP (SURVEY.md 8f item 1).

The reference (test.py:134-151) walks the predictions of an image in Python and calls ``skew_bbox_iou(pbox, tbox[m])``
once per prediction -- one kernel-equivalent plus a GPU<->CPU sync per box.  Here ONE rotated-IoU matrix launch covers
the whole image and ONE small kernel does the greedy assignment (class-restricted argmax per prediction, first maximum
like torch.max, each target claimed once); the host reads the result once per image.

``match_batch`` and ``Evaluator`` do the whole evaluation of test.py:80-151 and ap_per_class (utils/utils.py:200-286)
on the device: one set of launches per batch straight from ``detect_postprocess_classes``, nothing read back until
``Evaluator.compute``, which reads its result once."""
import ctypes

import numpy as np
import torch

from . import _lib
from .iou import rotated_iou_matrix


def match_detections_device(pred, tbox, tcls, iou_thres=0.5):
    """pred [P, 8] = (x, y, w, h, theta, conf, cls_conf, cls) CUDA, confidence-sorted as non_max_suppression returns it;
    tbox [T, 5] pixel (x, y, w, h, theta); tcls [T].  Returns ``correct`` as a CUDA uint8 tensor [P] (no host sync)."""
    p, t = len(pred), len(tbox)
    dev = pred.device
    correct = torch.zeros(p, dtype=torch.uint8, device=dev)
    if p == 0 or t == 0:
        return correct
    with torch.cuda.device(dev):
        pred = pred.float().contiguous()
        tb = tbox[:, :5].float().contiguous().to(dev)
        tc = tcls.float().contiguous().to(dev)
        iou = rotated_iou_matrix(pred[:, :5].contiguous(), tb)
        claimed = torch.empty(t, dtype=torch.uint8, device=dev)
        st = _lib.lib.ryolo_match_detections(_lib.ptr(iou), p, t, t, _lib.ptr(pred[:, 7:]), pred.shape[1], _lib.ptr(tc),
                                             float(iou_thres), _lib.ptr(claimed), _lib.ptr(correct), _lib.stream_ptr(dev))
        _lib.check(st, "ryolo_match_detections")
    return correct


def match_detections(pred, tbox, tcls, iou_thres=0.5):
    """same, as the list of 0/1 the reference builds (test.py:131-151): one host read per image"""
    return match_detections_device(pred, tbox, tcls, iou_thres).tolist()


def _match_into(res, targets, hw, iou_thres, correct, conf, pcls, count, hist, nc):
    """ryolo_match_batched: this batch's rows appended to (correct, conf, pcls) at the device row count `count`"""
    dets, keep, num = res["dets"], res["keep"], res["num_keep"]
    if dets.dim() != 3 or dets.shape[2] != 8 or keep.shape != dets.shape[:2] or num.shape != dets.shape[:1]:
        raise ValueError("match_batch takes detect_postprocess_classes' dict (dets [B, cap, 8], keep [B, cap], "
                         "num_keep [B]), got dets %s" % (tuple(dets.shape),))
    bsz, cap = keep.shape
    dev = dets.device
    t = torch.as_tensor(targets).to(device=dev, dtype=torch.float32).reshape(-1, 7).contiguous()
    nt = t.shape[0]
    height, width = int(hw[0]), int(hw[1])
    iou = torch.empty(cap * nt, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        stream = _lib.stream_ptr(dev)
        need = ctypes.c_size_t(0)
        args = [bsz, cap, _lib.ptr(t) if nt else None, nt, height, width, float(iou_thres), _lib.ptr(correct),
                _lib.ptr(conf), _lib.ptr(pcls), _lib.ptr(count), _lib.ptr(hist) if hist is not None else None, int(nc),
                _lib.ptr(iou) if nt else None]
        _lib.check(_lib.lib.ryolo_match_batched(None, None, None, *args, None, ctypes.byref(need), stream),
                   "ryolo_match_batched")
        ws = torch.empty(need.value, dtype=torch.uint8, device=dev)
        _lib.check(_lib.lib.ryolo_match_batched(_lib.ptr(dets.contiguous()), _lib.ptr(keep), _lib.ptr(num), *args,
                                                _lib.ptr(ws), ctypes.byref(need), stream), "ryolo_match_batched")
    return iou


def match_batch(res, targets, hw, iou_thres=0.5):
    """test.py's per-image matching (test.py:119-151) for a whole batch, with no host read.

    res: the dict ``detect_postprocess_classes`` returns; targets [nt, 7] (image, class, x, y, w, h, theta) normalised
    to the letterboxed image as ``letterbox_labels`` gives them, in any order; hw: the letterboxed (height, width).
    Returns dict(correct uint8, conf, cls float32 [B * cap], count int32 [1], iou): rows [0, count) are every kept
    detection in test.py's order -- images in batch order, within an image confidence descending, ties by class
    ascending, then by input row (``detections_per_image``'s order).  ``iou`` is the IoU scratch (layout in
    include/ryolo.h, ryolo_match_batched)."""
    bsz, cap = res["keep"].shape
    dev = res["dets"].device
    correct = torch.empty(bsz * cap, dtype=torch.uint8, device=dev)
    conf = torch.empty(bsz * cap, dtype=torch.float32, device=dev)
    pcls = torch.empty(bsz * cap, dtype=torch.float32, device=dev)
    count = torch.zeros(1, dtype=torch.int32, device=dev)
    iou = _match_into(res, targets, hw, iou_thres, correct, conf, pcls, count, None, 1)
    return {"correct": correct, "conf": conf, "cls": pcls, "count": count, "iou": iou}


class Evaluator:
    """The statistics test.py gathers over an evaluation (test.py:80-151) and ap_per_class over them, on the device.

        ev = Evaluator(nc, iou_thres=0.5, device="cuda:0")
        for each batch:  ev.add(detect_postprocess_classes(io, conf_thres, nms_thres, cap), targets, (height, width))
        p, r, ap, f1, ap_class, nt, seen = ev.compute()

    ``add`` synchronises nothing with the host: the batch's rows are appended to a device arena sized by the bound
    batch * cap, its target classes are added to a device histogram and its images to ``seen``.  As in test.py, an
    image without detections still counts its targets, and one without targets adds its rows as incorrect.
    ``compute`` reads its result once: per class present in the targets (ascending, ``ap_class``) precision, recall,
    AP and F1 as numpy float64 arrays, ``nt`` the targets per class (int64 [nc]) and ``seen`` the images added.  Rows
    with equal confidence keep their order (images in the order added); the reference's argsort leaves it unspecified.
    Target classes must be integers in [0, nc)."""

    def __init__(self, nc, iou_thres=0.5, device=None):
        self.nc = int(nc)
        if self.nc < 1:
            raise ValueError("Evaluator: nc must be >= 1, got %d" % self.nc)
        self.iou_thres = float(iou_thres)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.seen = 0
        self._bound = 0                      # rows the arena may hold: the sum of batch * cap over the adds
        self._correct = torch.empty(0, dtype=torch.uint8, device=self.device)
        self._conf = torch.empty(0, dtype=torch.float32, device=self.device)
        self._cls = torch.empty(0, dtype=torch.float32, device=self.device)
        self._count = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._hist = torch.zeros(self.nc + 1, dtype=torch.int32, device=self.device)

    def add(self, res, targets, hw):
        """append one batch: res from detect_postprocess_classes, targets / hw as for match_batch"""
        bsz, cap = res["keep"].shape
        need = self._bound + bsz * cap
        if need >= 2 ** 31:
            raise ValueError("Evaluator: more than 2^31 - 1 detection rows (batch * cap summed over the adds)")
        if need > len(self._conf):
            rows = max(need, 2 * len(self._conf))
            for name in ("_correct", "_conf", "_cls"):
                old = getattr(self, name)
                new = torch.empty(rows, dtype=old.dtype, device=self.device)
                new[:self._bound] = old[:self._bound]
                setattr(self, name, new)
        _match_into(res, targets, hw, self.iou_thres, self._correct, self._conf, self._cls, self._count, self._hist,
                    self.nc)
        self._bound = need
        self.seen += bsz

    def compute(self):
        """(p, r, ap, f1, ap_class, nt, seen) as test.py computes them, with one host read"""
        nc = self.nc
        dev = self.device
        out = torch.empty(nc * 4, dtype=torch.float64, device=dev)
        with torch.cuda.device(dev):
            stream = _lib.stream_ptr(dev)
            args = [_lib.ptr(self._correct), _lib.ptr(self._conf), _lib.ptr(self._cls), _lib.ptr(self._count),
                    self._bound, _lib.ptr(self._hist), nc, _lib.ptr(out)]
            need = ctypes.c_size_t(0)
            _lib.check(_lib.lib.ryolo_ap_per_class(*args, None, ctypes.byref(need), stream), "ryolo_ap_per_class")
            ws = torch.empty(need.value, dtype=torch.uint8, device=dev)
            _lib.check(_lib.lib.ryolo_ap_per_class(*args, _lib.ptr(ws), ctypes.byref(need), stream),
                       "ryolo_ap_per_class")
            host = torch.cat([out, self._hist.to(torch.float64)]).cpu().numpy()
        stats = host[:nc * 4].reshape(nc, 4)
        hist = host[nc * 4:].astype(np.int64)
        if hist[nc]:
            raise ValueError("Evaluator: %d targets have a class that is not an integer in [0, %d)" % (hist[nc], nc))
        nt = hist[:nc]
        ap_class = np.nonzero(nt)[0].astype(np.int32)
        p, r, ap, f1 = (stats[ap_class, k].copy() for k in range(4))
        return p, r, ap, f1, ap_class, nt, self.seen
