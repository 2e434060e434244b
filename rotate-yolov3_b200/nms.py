"""Rotated NMS behind the reference's Python signatures.

* ``r_nms(dets, threshold)``            <- utils/nms/src/rotate_polygon_nms.cpp:7-16 (pybind module ``r_nms``)
* ``non_max_suppression(prediction, conf_thres, nms_thres)`` <- utils/nms/nms.py:4-69 (the ``use_cuda_nms`` branch)

Everything below the tensor plumbing happens in libryolo.so (ryolo_rnms / ryolo_nms_filter)."""
import ctypes

import numpy as np
import torch

from . import _lib

_vp = ctypes.c_void_p

def _workspace(nbytes, device):
    # torch's caching allocator is stream-aware; 256-B alignment is guaranteed (512-B blocks)
    return torch.empty(int(nbytes), dtype=torch.uint8, device=device)


def r_nms(dets, threshold):
    """dets: Tensor[N, 6] float32 CUDA (x, y, w, h, theta, score) -> Tensor[K] int64 of kept ORIGINAL indices,
    ascending (utils/nms/src/rotate_polygon_nms_kernel.cu:380-383).

    Reference behaviours kept: a non-CUDA input raises RuntimeError (CHECK_CUDA, rotate_polygon_nms.cpp:3,8);
    an empty input returns an empty CPU long tensor (:9-10); the call is synchronous."""
    if not isinstance(dets, torch.Tensor) or not dets.is_cuda:
        raise RuntimeError("dets must be a CUDAtensor ")
    if dets.numel() == 0:
        return torch.empty((0,), dtype=torch.long, device="cpu")
    if dets.dim() != 2 or dets.shape[1] < 6:
        raise RuntimeError("r_nms: dets must be [N, 6] (x, y, w, h, theta, score)")
    with torch.cuda.device(dets.device):
        d = dets[:, :6].to(torch.float32).contiguous()
        n = d.shape[0]
        ws_bytes = _lib.lib.ryolo_rnms_workspace_bytes(n)
        ws = _workspace(ws_bytes, d.device)
        keep = torch.empty((n,), dtype=torch.long, device=d.device)
        num = torch.empty((1,), dtype=torch.int32, device=d.device)
        st = _lib.lib.ryolo_rnms(_lib.ptr(d), n, float(threshold), _lib.ptr(keep), _lib.ptr(num), _lib.ptr(ws),
                                 ws_bytes, _lib.stream_ptr(d.device))
        _lib.check(st, "ryolo_rnms")
        k = int(num.item())  # the reference is synchronous too (blocking D2H of the whole mask)
        return keep[:k]


def rnms_debug(dets, threshold):
    """Test hook: run r_nms and also return (sorted_boxes [N,6], order [N] int32, mask [N, ceil(N/64)] int64 view)."""
    d = dets[:, :6].to(torch.float32).contiguous()
    n = d.shape[0]
    with torch.cuda.device(d.device):
        ws_bytes = _lib.lib.ryolo_rnms_workspace_bytes(n)
        ws = _workspace(ws_bytes, d.device)
        keep = torch.empty((n,), dtype=torch.long, device=d.device)
        num = torch.empty((1,), dtype=torch.int32, device=d.device)
        st = _lib.lib.ryolo_rnms_full_mask(_lib.ptr(d), n, float(threshold), _lib.ptr(keep), _lib.ptr(num), _lib.ptr(ws),
                                           ws_bytes, _lib.stream_ptr(d.device))
        _lib.check(st, "ryolo_rnms_full_mask")
        k = int(num.item())
        pb, po, pm = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
        _lib.check(_lib.lib.ryolo_rnms_debug_views(_lib.ptr(ws), n, ctypes.byref(pb), ctypes.byref(po),
                                                   ctypes.byref(pm)), "ryolo_rnms_debug_views")
        base = ws.data_ptr()
        cb = (n + 63) // 64

        def view(p, nbytes, dtype, shape):
            off = p.value - base
            return ws[off:off + nbytes].view(dtype).view(shape).clone()
        boxes = view(pb, n * 6 * 4, torch.float32, (n, 6))
        order = view(po, n * 4, torch.int32, (n,))
        mask = view(pm, n * cb * 8, torch.int64, (n, cb))
        return keep[:k].clone(), boxes, order, mask


def nms_filter(pred, conf_thres, min_wh=2.0):
    """Candidate filter of non_max_suppression for ONE image (utils/nms/nms.py:34-40,55).
    pred [P, 6+nc] float32 CUDA, modified in place (pred[:, 5] *= class_conf).  Returns Tensor[n, 8]
    (x, y, w, h, theta, conf, class_conf, class) in input order."""
    assert pred.is_cuda and pred.dtype == torch.float32 and pred.is_contiguous()
    p, no = pred.shape
    nc = no - 6
    with torch.cuda.device(pred.device):
        out = torch.empty((p, 8), dtype=torch.float32, device=pred.device)
        num = torch.empty((1,), dtype=torch.int32, device=pred.device)
        ws_bytes = _lib.lib.ryolo_nms_filter_workspace_bytes(p)
        ws = _workspace(ws_bytes, pred.device)
        st = _lib.lib.ryolo_nms_filter(_lib.ptr(pred), p, nc, float(conf_thres), float(min_wh), _lib.ptr(out), p,
                                       _lib.ptr(num), _lib.ptr(ws), ws_bytes, _lib.stream_ptr(pred.device))
        _lib.check(st, "ryolo_nms_filter")
        return out[:int(num.item())]


def non_max_suppression(prediction, conf_thres=0.5, nms_thres=0.5):
    """Drop-in for utils/nms/nms.py:4-69: per image, (x, y, w, h, a, object_conf*class_conf, class_conf, class)
    rows of the survivors sorted by confidence, or None.  Mutates prediction[..., 5] like the reference (:35)."""
    min_wh = 2
    output = [None] * len(prediction)
    for image_i, pred in enumerate(prediction):
        if prediction.numel() == 0:
            continue
        if not pred.is_contiguous():  # keep the in-place side effect on the caller's tensor
            raise RuntimeError("non_max_suppression: prediction must be contiguous")
        cand = nms_filter(pred, conf_thres, min_wh)
        if len(cand) == 0:
            continue
        cand = cand[(-cand[:, 5]).argsort()]
        if pred.shape[1] == 7:
            # single-class configs (every cfg the reference ships): class_pred is 0 for every row, so the per-class loop,
            # its unique() (a host sync), the boolean masks and both re-sorts are identities -- r_nms returns ascending
            # indices into the confidence-sorted rows, i.e. the result is already in the reference's final order
            inds = r_nms(cand[:, :6], nms_thres)
            output[image_i] = cand[inds]
            continue
        det_max = []
        for c in cand[:, -1].unique():
            dc = cand[cand[:, -1] == c]
            dc = dc[(-dc[:, 5]).argsort()]
            inds = r_nms(dc[:, :6], nms_thres)
            det_max.append(dc[inds])
        if len(det_max):
            det_max = torch.cat(det_max)
            output[image_i] = det_max[(-det_max[:, 5]).argsort()]
    return output


def r_nms_batched(dets, counts, threshold, limit=None):
    """S independent rotated-NMS problems in one set of launches, no host synchronisation.
    dets [S, cap, 6] float32 CUDA contiguous, counts [S] int32 CUDA (rows used per segment), limit: at most this many
    best-scored boxes per segment enter the NMS.  Returns (keep [S, cap] int64, num_keep [S] int32): segment s keeps rows
    keep[s, :num_keep[s]] (ascending row indices within the segment) -- per segment identical to r_nms(dets[s, :n])."""
    s_, cap = dets.shape[0], dets.shape[1]
    limit = cap if limit is None else int(limit)
    with torch.cuda.device(dets.device):
        ws_bytes = _lib.lib.ryolo_rnms_batched_workspace_bytes(s_, cap)
        ws = _workspace(ws_bytes, dets.device)
        keep = torch.empty((s_, cap), dtype=torch.long, device=dets.device)
        num = torch.empty((s_,), dtype=torch.int32, device=dets.device)
        st = _lib.lib.ryolo_rnms_batched(_lib.ptr(dets), s_, cap, _lib.ptr(counts), limit, float(threshold), _lib.ptr(keep),
                                         _lib.ptr(num), _lib.ptr(ws), ws_bytes, _lib.stream_ptr(dets.device))
        _lib.check(st, "ryolo_rnms_batched")
    return keep, num


def detect_select(io, conf_thres, limit, min_wh=2.0):
    """Candidate selection of a whole decoded batch on the device: per image the `limit` most confident rows that pass
    the reference's filter (utils/nms/nms.py:34-40), ties resolved by lowest row index, in input order.
    conf_thres must be >= 0.  Returns (dets [B, limit, 6], counts [B] int32 = min(limit, rows passing the filter))."""
    bsz, p, no = io.shape
    cap = int(limit)
    with torch.cuda.device(io.device):
        dets = torch.empty((bsz, cap, 6), dtype=torch.float32, device=io.device)
        counts = torch.empty((bsz,), dtype=torch.int32, device=io.device)
        ws_bytes = _lib.lib.ryolo_detect_select_workspace_bytes(bsz, p)
        ws = _workspace(ws_bytes, io.device)
        st = _lib.lib.ryolo_detect_select(_lib.ptr(io), bsz, p, no - 6, float(conf_thres), float(min_wh), int(limit),
                                          _lib.ptr(dets), cap, _lib.ptr(counts), _lib.ptr(ws), ws_bytes,
                                          _lib.stream_ptr(io.device))
        _lib.check(st, "ryolo_detect_select")
    return dets, counts


def detect_postprocess(io, conf_thres, nms_thres, cap, filter_done_event=None):
    """detect.py:204-213 after the forward, for a whole batch WITHOUT host round trips: device-side candidate selection
    (filter + top-`cap` by confidence; the reference has no cap and relies on trained weights, a random-init network puts
    ~half of the 545 832 proposals above any threshold) and ONE segmented rotated NMS over all images, one segment per
    image.  Single-class configs only: io [B, P, 7] float32 CUDA contiguous.
    Returns dict(dets [B, cap, 6], counts [B], keep [B, cap] int64, num_keep [B] int32): image b keeps rows
    dets[b, keep[b, :num_keep[b]]]."""
    if io.dim() != 3 or io.shape[-1] != 7:
        raise ValueError("detect_postprocess runs class-agnostic NMS and takes single-class io [B, P, 7], got %s; "
                         "use non_max_suppression for multi-class configs (NMS per class)" % (tuple(io.shape),))
    if not io.is_contiguous():
        io = io.contiguous()
    dets, counts = detect_select(io, conf_thres, cap)
    if filter_done_event is not None:
        filter_done_event.record()
    keep, num = r_nms_batched(dets, counts, nms_thres)
    return {"dets": dets, "counts": counts, "keep": keep, "num_keep": num}


def detect_postprocess_classes(io, conf_thres, nms_thres, cap, min_wh=2.0):
    """detect_postprocess for any number of classes, still without host round trips: the same device-side selection of
    the top-`cap` candidates per image (over all classes), written with the class columns, then one segmented rotated
    NMS with one segment per image that suppresses only within a class -- the reference's per-class loop
    (utils/nms/nms.py:47-56).  io [B, P, 6+nc] float32 CUDA, nc >= 1, not modified; conf_thres >= 0.
    Returns dict(dets [B, cap, 8] = (x, y, w, h, theta, conf, class_conf, class) in input order, counts [B] int32,
    keep [B, cap] int64, num_keep [B] int32): image b keeps rows dets[b, keep[b, :num_keep[b]]] (ascending rows)."""
    if io.dim() != 3 or io.shape[-1] < 7:
        raise ValueError("detect_postprocess_classes takes io [B, P, 6+nc] with nc >= 1, got %s" % (tuple(io.shape),))
    if not io.is_contiguous():
        io = io.contiguous()
    bsz, p, no = io.shape
    cap = int(cap)
    with torch.cuda.device(io.device):
        dets = torch.empty((bsz, cap, 8), dtype=torch.float32, device=io.device)
        counts = torch.empty((bsz,), dtype=torch.int32, device=io.device)
        ws_bytes = _lib.lib.ryolo_detect_select_workspace_bytes(bsz, p)
        ws = _workspace(ws_bytes, io.device)
        stream = _lib.stream_ptr(io.device)
        st = _lib.lib.ryolo_detect_select_classes(_lib.ptr(io), bsz, p, no - 6, float(conf_thres), float(min_wh), cap,
                                                  _lib.ptr(dets), cap, _lib.ptr(counts), _lib.ptr(ws), ws_bytes, stream)
        _lib.check(st, "ryolo_detect_select_classes")
        keep = torch.empty((bsz, cap), dtype=torch.long, device=io.device)
        num = torch.empty((bsz,), dtype=torch.int32, device=io.device)
        ws_bytes = _lib.lib.ryolo_rnms_batched_classes_workspace_bytes(bsz, cap)
        ws = _workspace(ws_bytes, io.device)
        st = _lib.lib.ryolo_rnms_batched_classes(_lib.ptr(dets), bsz, cap, _lib.ptr(counts), float(nms_thres),
                                                 _lib.ptr(keep), _lib.ptr(num), _lib.ptr(ws), ws_bytes, stream)
        _lib.check(st, "ryolo_rnms_batched_classes")
    return {"dets": dets, "counts": counts, "keep": keep, "num_keep": num}


def multiscale_sizes(img_size, rng=np.random):
    """The two sizes detect.py --multi-scale draws for base size img_size (detect.py:54-59): multiples of 32 between
    about img_size / 1.5 and img_size * 1.3, two distinct, from rng.choice (numpy's global RNG by default, so a seeded
    numpy draws the reference's sizes).  Returns a list of two ints in the drawn order."""
    img_sz_min = round(img_size / 32 / 1.5) + 1
    img_sz_max = round(img_size / 32 * 1.3) - 1
    return [int(x) for x in rng.choice(range(img_sz_min * 32, (img_sz_max + 1) * 32, 32), 2, False)]


STAGE1_NMS_THRES = 0.95      # multi_detect's per-scale NMS threshold (detect.py:90)


def detect_multiscale(model, images, sizes, conf_thres, nms_thres, cap):
    """detect.py --multi-scale (multi_detect, detect.py:16-119) for a whole batch, without host round trips.

    images: list of uint8 [H, W, 3] BGR images (cv2.imread / decode_images; host or CUDA), uploaded once.  For every
    size s of `sizes` (multiples of 32, square letterbox), largest first: letterbox(images, s), the eval forward of
    `model`, and the per-scale detection detect_postprocess_classes(io, conf_thres, 0.95, cap) before the next forward
    overwrites io.  Then, per image, the kept rows of every scale mapped to original-image pixels as
    scale_coords(...).round() maps them, concatenated in the order of `sizes` (kept rows ascending within a scale), and
    the second detection detect_postprocess_classes(merged, conf_thres, nms_thres, len(sizes) * cap) on those 8-column
    rows: as in the reference, its class maximum runs over (class_conf, class index), so a row of class c >= 1 has its
    conf multiplied by c and comes out as class 1 (INTEGRATION.md §4).  `cap` bounds the candidates per image and scale;
    the second stage never truncates.

    Returns detect_postprocess_classes' dict (dets, counts, keep, num_keep) in original-image pixels:
    detections_per_image of it is multi_detect's final_dets per image."""
    from . import preprocess
    if model.training:
        raise ValueError("detect_multiscale runs the eval forward: call model.eval() first")
    sizes = [int(s) for s in sizes]
    if not sizes:
        raise ValueError("detect_multiscale: sizes is empty")
    if len(sizes) > _lib.MERGE_MAX_SCALES:
        raise ValueError("detect_multiscale: at most %d sizes, got %d" % (_lib.MERGE_MAX_SCALES, len(sizes)))
    bad = [s for s in sizes if s <= 0 or s % 32]
    if bad:
        raise ValueError("detect_multiscale: every size must be a positive multiple of 32, got %s" % (bad,))
    if not conf_thres >= 0:
        raise ValueError("detect_multiscale: conf_thres must be >= 0, got %r" % (conf_thres,))
    cap = int(cap)
    if cap < 1:
        raise ValueError("detect_multiscale: cap must be >= 1, got %d" % cap)
    device = next(model.parameters()).device
    srcs = preprocess.upload_images(images, device)
    bsz, scales = len(srcs), len(sizes)
    shapes = [tuple(s.shape[:2]) for s in srcs]
    table = np.empty((scales, bsz, 3), np.float32)     # (padx, pady, gain), each rounded to float32 as scale_coords does
    for k, s in enumerate(sizes):
        table[k] = np.array(preprocess.scale_coords_terms((s, s), shapes), np.float64).T
    stage1 = [None] * scales
    with torch.cuda.device(device), torch.no_grad():
        table_dev = preprocess.upload_table(table, device)
        # largest first: the eval pool of this batch size grows at most once and keeps every size's plan
        for k in sorted(range(scales), key=lambda k: -sizes[k]):
            img, _ = preprocess.letterbox(srcs, sizes[k], device=device)
            io, _ = model(img)
            stage1[k] = detect_postprocess_classes(io, conf_thres, STAGE1_NMS_THRES, cap)
        merged = torch.empty((bsz, scales * cap, 8), dtype=torch.float32, device=device)
        arr = lambda key: (_vp * scales)(*[r[key].data_ptr() for r in stage1])
        st = _lib.lib.ryolo_merge_scales(arr("dets"), arr("keep"), arr("num_keep"), scales, bsz, cap, _lib.ptr(table_dev),
                                         _lib.ptr(merged), _lib.stream_ptr(device))
        _lib.check(st, "ryolo_merge_scales")
        return detect_postprocess_classes(merged, conf_thres, nms_thres, scales * cap)


def detections_per_image(res):
    """The result of detect_postprocess_classes as non_max_suppression's list: per image a Tensor[k, 8] of the kept rows
    ordered by confidence descending, ties by class ascending, then by input row -- or None when nothing is kept.
    One host read (the kept counts) for the whole batch."""
    nums = res["num_keep"].tolist()
    out = []
    for b, k in enumerate(nums):
        if k == 0:
            out.append(None)
            continue
        rows = res["dets"][b][res["keep"][b, :k]]                       # input order
        rows = rows[torch.argsort(rows[:, 7], stable=True)]             # class ascending, input order within a class
        out.append(rows[torch.argsort(rows[:, 5], descending=True, stable=True)])
    return out
