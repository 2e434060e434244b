"""Training batches on the device: the reference's ``LoadImagesAndLabels.__getitem__`` with ``augment=True`` and its
``collate_fn`` (``utils/datasets.py:423-509``), for the transforms whose arithmetic the reference defines with cv2 and
numpy (``utils/augment.py``): ``random_affine``, ``Gamma``, ``HSV``, ``HorizontalFlip`` and ``VerticalFlip``.

Per image, in the reference's order:

* pre-resize: when ``img_size / max(img.shape) < 1``, ``cv2.resize(INTER_LINEAR)`` to ``(int(w r), int(h r))``;
* letterbox (``preprocess.geometry``, cv2's ``INTER_AREA`` and a grey border) into a uint8 HWC image;
* Affine: ``cv2.warpAffine`` of the letterboxed image, border 128;
* Gamma, HSV, the flips, BGR->RGB and ``/255`` in one finishing pass.

The pixels are byte for byte the reference's and the target rows bit for bit ``collate_fn``'s.  ``Noise``, ``Blur``
and ``Grayscale`` are imgaug augmenters with no arithmetic to restate: their random draws are consumed (so every
other draw lines up with the reference) and reported in the draw record, but the image is not changed for them.

The Python ``random`` draws are replayed exactly (``draw``); the label rows are a few per image and are computed on
the host in the reference's dtypes (``transform_labels``) and uploaded with the pixels.  A batch is one pinned upload
and three or four kernel launches: the pre-resize (only when some image needs it), the letterbox, the warp with the
per-image maximum (only when some image is warped or gamma-corrected) and the finish."""
import ctypes
import math
import random as _random

import numpy as np
import torch

from . import _lib
from .preprocess import _JOB_BYTES, _check_image, _packed, _pinned, _staging, geometry

HYP_KEYS = ("degrees", "translate", "scale", "shear", "noise", "gamma", "blur", "hsv_s", "hsv_v", "grayscale")
DRAW_KEYS = ("gray_alpha", "affine", "noise", "gamma", "blur", "hsv", "hflip", "vflip", "grayscale")
_WARP_BYTES = ctypes.sizeof(_lib.WarpJob)
_FIN_BYTES = ctypes.sizeof(_lib.FinishJob)


def draw(hyp, rng=_random):
    """One image's random draws in the order the reference's ``__getitem__`` makes them, from ``rng`` (a
    ``random.Random`` or the ``random`` module).  Returns the record ``train_batch`` takes and returns:
    gray_alpha (``Grayscale.__init__``), affine (a, s, tx, ty) or None, gamma gm or None, hsv (a, b) or None, and
    noise / blur / hflip / vflip / grayscale booleans.  tx and ty are the uniform fractions: as in the reference,
    x is translated by tx times the image height and y by ty times its width.  A missing hyp key raises KeyError."""
    deg, tr, sc = hyp["degrees"], hyp["translate"], hyp["scale"]
    hyp["shear"], hyp["noise"]
    gam, sat, val = hyp["gamma"], hyp["hsv_s"], hyp["hsv_v"]
    hyp["blur"]
    rec = {"gray_alpha": rng.uniform(hyp["grayscale"], 1.0)}

    def fires(p):
        rng.random()                     # Transform's own `random() < 1` test
        return rng.random() < p

    rec["affine"] = ((rng.uniform(-deg, deg), rng.uniform(1 - sc, 1 + sc), rng.uniform(-tr, tr),
                      rng.uniform(-tr, tr)) if fires(0.5) else None)
    rec["noise"] = fires(0.2)
    rec["gamma"] = rng.uniform(1 - gam, 1 + gam) if fires(0.4) else None
    rec["blur"] = fires(0.5)
    rec["hsv"] = (rng.uniform(-1, 1) * sat + 1, rng.uniform(-1, 1) * val + 1) if fires(0.5) else None
    rec["hflip"] = fires(0.5)
    rec["vflip"] = fires(0.5)
    rec["grayscale"] = fires(0.5)
    return rec


def rotation_matrix(angle, center, scale):
    """cv2.getRotationMatrix2D in float64 (the centre is a float32 point, as cv2 takes it)"""
    a = angle * (math.pi / 180)
    alpha, beta = math.cos(a) * scale, math.sin(a) * scale
    cx, cy = float(np.float32(center[0])), float(np.float32(center[1]))
    return np.array([[alpha, beta, (1 - alpha) * cx - beta * cy], [-beta, alpha, beta * cx + (1 - alpha) * cy]])


def affine_matrix(rec_affine, hw):
    """random_affine's M = T @ R (3 x 3, float64) for an image of shape hw"""
    a, s, tx, ty = rec_affine
    h, w = hw
    R = np.eye(3)
    R[:2] = rotation_matrix(a, (w / 2, h / 2), s)
    T = np.eye(3)
    T[0, 2] = tx * h
    T[1, 2] = ty * w
    return T @ R


def invert_affine(M):
    """the dst -> src map cv2.warpAffine computes from M (float64, in cv2's order)"""
    m = [float(v) for v in np.asarray(M, np.float64)[:2].reshape(-1)]
    d = m[0] * m[4] - m[1] * m[3]
    d = 1.0 / d if d != 0 else 0.0
    a11, a22 = m[4] * d, m[0] * d
    m0, m1, m3, m4 = a11, m[1] * -d, m[3] * -d, a22
    return [m0, m1, -m0 * m[2] - m1 * m[5], m3, m4, -m3 * m[2] - m4 * m[5]]


def _corners_inside(t, hw):
    """the four rotated corners of each (x, y, w, h, a) row strictly inside the image, computed as
    get_rotated_coors computes them: float32 tensors and a float64 rotation matrix per row"""
    h, w = hw
    keep = np.zeros(len(t), bool)
    for k, row in enumerate(torch.from_numpy(np.ascontiguousarray(t[:, 1:]))):
        cx, cy, bw, bh, a = row
        x0, x1 = cx - bw * 0.5, cx + bw * 0.5
        y0, y1 = cy - bh * 0.5, cy + bh * 0.5
        R = rotation_matrix(float(-a * 180 / math.pi), (float(cx), float(cy)), 1.0)
        xs = [px * R[0, 0] + py * R[0, 1] + R[0, 2] for px, py in ((x0, y0), (x0, y1), (x1, y1), (x1, y0))]
        ys = [px * R[1, 0] + py * R[1, 1] + R[1, 2] for px, py in ((x0, y0), (x0, y1), (x1, y1), (x1, y0))]
        keep[k] = all(bool(v < w) and bool(v > 0) for v in xs) and all(bool(v < h) and bool(v > 0) for v in ys)
    return keep


def transform_labels(x, src_hw, meta, out_hw, rec):
    """One image's label rows through the letterbox (``datasets.py:453-467``), ``random_affine``'s update and
    filter, the flips and the normalisation (``:486-490``), in the reference's float32 / float64 arithmetic.
    x: float32 [n, 6] (cls, x, y, w, h, a; x..h in 0-1 units of the source); src_hw: the (pre-resized) source shape;
    meta: (ratiow, ratioh, padw, padh).  Returns float32 [m, 6]."""
    if x.size == 0:
        return np.zeros((0, 6), np.float32)
    h, w = src_hw
    ratiow, ratioh, padw, padh = meta
    lab = x.copy()
    lab[:, 1] = ratiow * w * lab[:, 1] + padw
    lab[:, 2] = ratioh * h * lab[:, 2] + padh
    lab[:, 3] = ratiow * w * lab[:, 3]
    lab[:, 4] = ratioh * h * lab[:, 4]
    H, W = out_hw
    if rec["affine"] is not None:
        a, s = rec["affine"][0], rec["affine"][1]
        M = affine_matrix(rec["affine"], out_hw)
        lab[:, 5] -= a / 180 * math.pi
        lab[:, 5][lab[:, 5] > 0.5 * math.pi] -= math.pi
        lab[:, 5][lab[:, 5] < -0.5 * math.pi] += math.pi
        cx = lab[:, 1] * M[0, 0] + lab[:, 2] * M[0, 1] + M[0, 2]
        cy = lab[:, 1] * M[1, 0] + lab[:, 2] * M[1, 1] + M[1, 2]
        lab[:, 1] = cx
        lab[:, 2] = cy
        lab[:, [3, 4]] *= s
        lab[:, 1] = lab[:, 1].clip(0, W)
        lab[:, 2] = lab[:, 2].clip(0, H)
        bw, bh = lab[:, 3], lab[:, 4]
        ar = np.maximum(bw / (bh + 1e-16), bh / (bw + 1e-16))
        lab = lab[(bw > 4) & (bh > 4) & (ar < 15) & _corners_inside(lab, out_hw)]
    if rec["hflip"] and len(lab):
        lab[:, 1] = W - lab[:, 1]
        lab[:, 5] = -lab[:, 5]
    if rec["vflip"] and len(lab):
        lab[:, 2] = H - lab[:, 2]
        lab[:, 5] = -lab[:, 5]
    if len(lab):
        lab[:, [2, 4]] /= H
        lab[:, [1, 3]] /= W
    return lab


def pre_resize_shape(hw, img_size):
    """the reference's training pre-resize: (int(h r), int(w r)) when r = img_size / max(img.shape) < 1, else None"""
    r = img_size / max(hw[0], hw[1], 3)
    return (int(hw[0] * r), int(hw[1] * r)) if r < 1 else None


def _check_record(rec, i):
    if not isinstance(rec, dict) or any(k not in rec for k in DRAW_KEYS):
        raise ValueError("train_batch: draws[%d] must be a record with keys %s" % (i, DRAW_KEYS))
    if rec["affine"] is not None and len(rec["affine"]) != 4:
        raise ValueError("train_batch: draws[%d]['affine'] must be (a, s, tx, ty) or None" % i)
    if rec["hsv"] is not None and (len(rec["hsv"]) != 2 or min(rec["hsv"]) < 0):
        raise ValueError("train_batch: draws[%d]['hsv'] must be two factors >= 0 or None, got %r" % (i, rec["hsv"]))


def _host_image(im, i):
    if isinstance(im, torch.Tensor):
        if im.dtype != torch.uint8:
            raise ValueError("train_batch: image %d must be uint8, got %s" % (i, im.dtype))
        _check_image(im, i)
        if not im.is_cuda:
            return np.ascontiguousarray(im.numpy())
        if im.stride(2) != 1 or im.stride(1) != 3:       # the kernels read pixel x, channel c at row + 3 x + c
            im = im.contiguous()
        return im
    im = np.asarray(im)
    if im.dtype != np.uint8:
        raise ValueError("train_batch: image %d must be uint8, got %s" % (i, im.dtype))
    _check_image(im, i)
    return np.ascontiguousarray(im)


def train_batch(images, labels, hyp, new_shape=608, mode="square", rng=_random, draws=None, dtype=torch.float32,
                device=None, out=None, img_size=None):
    """One augmented training batch on the device, as ``LoadImagesAndLabels(augment=True)`` and ``collate_fn`` give
    it (with Noise, Blur and Grayscale as identities).

    images: list of uint8 [H, W, 3] BGR images (numpy, CPU or CUDA tensors; sizes may differ), as ``cv2.imread``
    returns them; CUDA images with any strides (rows need not be contiguous, pixels and channels are made so).
    labels: list of float32 [n, 6] (cls, x, y, w, h, a; x..h in 0-1 units, as the label files hold
    them; n may be 0).  hyp: the training hyperparameters (``degrees``, ``translate``, ``scale``, ``shear``,
    ``noise``, ``gamma``, ``blur``, ``hsv_s``, ``hsv_v``, ``grayscale``).  new_shape: int for mode='square' (also the
    pre-resize size), (h, w) for mode='rect' (the batch shape, ``dataset.batch_shapes[bi]``).  img_size: the
    dataset's ``img_size``, which sets the pre-resize (``datasets.py:433-440``); in mode='rect' it defaults to
    max(h, w), which is the dataset's img_size when that is a multiple of 32 -- pass it when it is not.  In
    mode='square' it is new_shape.  rng: where the
    draws come from unless ``draws`` (a list of records from an earlier call or ``draw``) replays them.
    dtype: torch.float32 or torch.float16.  out: optional [B, 3, H, W] CUDA tensor of dtype.

    Returns (imgs [B, 3, H, W], targets [nt, 7] float32 on the device (image index, cls, x, y, w, h, a), draws)."""
    if dtype not in (torch.float32, torch.float16):
        raise ValueError("train_batch: dtype must be torch.float32 or torch.float16, got %s" % (dtype,))
    if not isinstance(images, (list, tuple)) or len(images) == 0 or len(images) > 65535:
        raise ValueError("train_batch: images must be a list of 1 to 65535 [H, W, 3] uint8 images")
    if not isinstance(labels, (list, tuple)) or len(labels) != len(images):
        raise ValueError("train_batch: labels must be a list of one [n, 6] array per image")
    if mode == "square" and isinstance(new_shape, int):
        out_hw = (new_shape, new_shape)
    elif mode == "rect" and not isinstance(new_shape, int) and len(new_shape) == 2:
        out_hw = (int(new_shape[0]), int(new_shape[1]))
    else:
        raise ValueError("train_batch: mode='square' takes an int new_shape, mode='rect' an (h, w); got %r, %r"
                         % (mode, new_shape))
    if img_size is None:
        img_size = max(out_hw)
    elif (not isinstance(img_size, int) or isinstance(img_size, bool) or img_size < 1
          or (mode == "square" and img_size != new_shape)):
        raise ValueError("train_batch: img_size must be a positive int (new_shape itself in mode='square'), got %r"
                         % (img_size,))
    missing = [k for k in HYP_KEYS if k not in hyp]
    if missing:
        raise KeyError(missing[0])
    if device is None:
        device = next((im.device for im in images if isinstance(im, torch.Tensor) and im.is_cuda),
                      out.device if out is not None else torch.device("cuda", torch.cuda.current_device()))
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("train_batch runs on a CUDA device only, got %s (there is no CPU path)" % (device,))
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    srcs = [_host_image(im, i) for i, im in enumerate(images)]
    for i, s in enumerate(srcs):
        if isinstance(s, torch.Tensor) and s.device != device:
            raise ValueError("train_batch: image %d is on %s, not %s" % (i, s.device, device))
    labs = []
    for i, x in enumerate(labels):
        x = np.asarray(x.cpu() if isinstance(x, torch.Tensor) else x, dtype=np.float32)
        if x.size == 0:
            x = np.zeros((0, 6), np.float32)
        if x.ndim != 2 or x.shape[1] != 6:
            raise ValueError("train_batch: labels[%d] must be [n, 6], got shape %s" % (i, x.shape))
        labs.append(x)
    if draws is None:
        draws = [draw(hyp, rng) for _ in srcs]
    elif not isinstance(draws, (list, tuple)) or len(draws) != len(srcs):
        raise ValueError("train_batch: draws must hold one record per image")
    for i, rec in enumerate(draws):
        _check_record(rec, i)
    bsz = len(srcs)
    if out is None:
        out = torch.empty((bsz, 3) + out_hw, dtype=dtype, device=device)
    elif (not out.is_cuda or out.device != device or out.dtype != dtype or tuple(out.shape) != (bsz, 3) + out_hw
          or not out.is_contiguous()):
        raise ValueError("train_batch: out must be a contiguous %s CUDA tensor %s on %s"
                         % (dtype, [bsz, 3, *out_hw], device))
    plan, targets = batch_plan([tuple(s.shape[:2]) for s in srcs], labs, draws, new_shape, mode, img_size)
    with torch.cuda.device(device):
        launch, tgt, _ = _stage(srcs, plan, targets, out_hw, out, dtype, device)
        launch()
    return out, tgt, list(draws)


def batch_plan(shapes, labels, draws, new_shape=608, mode="square", img_size=None):
    """The host half of ``train_batch``, from shapes, label rows and draws alone (img_size: the pre-resize size,
    max of the output shape by default): per image (source shape,
    pre-resized shape or None, letterboxed shape, top, left, draw record), and collate_fn's float32 target rows
    [nt, 7] (image index, cls, x, y, w, h, a)."""
    out_hw = (new_shape, new_shape) if mode == "square" else tuple(int(v) for v in new_shape)
    img_size = max(out_hw) if img_size is None else img_size
    plan, rows = [], []
    for b, (hw0, x, rec) in enumerate(zip(shapes, labels, draws)):
        pre = pre_resize_shape(hw0, img_size)
        hw = pre or hw0
        (nh, nw), (top, bottom, left, right), meta = geometry(hw, new_shape if mode == "square" else out_hw, mode)
        if nh < 1 or nw < 1 or top < 0 or left < 0 or top + nh + bottom != out_hw[0] or left + nw + right != out_hw[1]:
            raise ValueError("train_batch: image %d of shape %s does not letterbox into %s" % (b, hw0, out_hw))
        if mode == "rect":              # the reference's rect letterbox returns numpy float64 scalars (batch_shapes)
            meta = tuple(np.float64(v) for v in meta)
        lab = transform_labels(x, hw, meta, out_hw, rec)
        rows.append(np.concatenate([np.full((len(lab), 1), b, np.float32), lab], 1))
        plan.append((hw0, pre, (nh, nw), top, left, rec))
    return plan, (np.concatenate(rows, 0) if rows else np.zeros((0, 7), np.float32))


def _align(n):
    return (n + 15) // 16 * 16


def _stage(srcs, plan, targets, out_hw, out, dtype, device):
    """Upload a batch's job tables, targets and host images (one pinned copy) and return (launch, targets on the
    device, buffers): launch() issues the batch's kernels on the current stream, and may be replayed (or captured in
    a CUDA graph) for as long as the buffers are kept."""
    bsz = len(srcs)
    H, W = out_hw
    pre_idx = [b for b, p in enumerate(plan) if p[1] is not None]
    pre_hw = (max((plan[b][1][0] for b in pre_idx), default=0), max((plan[b][1][1] for b in pre_idx), default=0))
    warp_idx = [b for b, p in enumerate(plan) if p[5]["affine"] is not None or p[5]["gamma"] is not None]
    # device workspace: pre-resized images | letterboxed images | warped images | row maxima
    img_bytes = H * W * 3
    pre_bytes = _align(len(pre_idx) * pre_hw[0] * pre_hw[1] * 3)
    n_warped = sum(1 for b in warp_idx if plan[b][5]["affine"] is not None)
    ws = torch.empty(pre_bytes + _align(bsz * img_bytes) + _align(max(n_warped, 1) * img_bytes) + bsz * H,
                     dtype=torch.uint8, device=device)
    pre_base = ws.data_ptr()
    lb_base = pre_base + pre_bytes
    warp_base = lb_base + _align(bsz * img_bytes)
    rowmax = warp_base + _align(max(n_warped, 1) * img_bytes)
    # staged upload: pre jobs | lb jobs | warp jobs | finish jobs | targets | tables | host images
    pre_packs = [_packed(plan[b][0], plan[b][1], True) for b in pre_idx]
    lb_packs = [_packed(plan[b][1] or plan[b][0], plan[b][2]) for b in range(bsz)]
    o_pre = 0
    o_lb = _align(o_pre + len(pre_idx) * _JOB_BYTES)
    o_warp = _align(o_lb + bsz * _JOB_BYTES)
    o_fin = _align(o_warp + len(warp_idx) * _WARP_BYTES)
    o_tgt = _align(o_fin + bsz * _FIN_BYTES)
    o_tab = _align(o_tgt + targets.nbytes)
    tab_words = sum(p[3].size + p[4].size for p in pre_packs + lb_packs)
    o_img = _align(o_tab + 4 * tab_words)
    total = o_img + sum(s.nbytes for s in srcs if isinstance(s, np.ndarray))
    dev = torch.empty(total, dtype=torch.uint8, device=device)
    pinned = _pinned(device, total)
    stage = pinned[:total].numpy()
    base = dev.data_ptr()
    tabs = stage[o_tab:o_tab + 4 * tab_words].view(np.int32)
    word, pos = 0, o_img
    src_ptr = []
    for s in srcs:
        if isinstance(s, np.ndarray):
            stage[pos:pos + s.nbytes] = s.reshape(-1)
            src_ptr.append((base + pos, s.shape[1] * 3))
            pos += s.nbytes
        else:
            src_ptr.append((s.data_ptr(), s.stride(0)))

    def lb_job(src, stride, shw, dhw, top, left, pack):
        nonlocal word
        kind, kx, ky, xt, yt = pack
        tabs[word:word + xt.size] = xt
        tabs[word + xt.size:word + xt.size + yt.size] = yt
        j = _lib.LetterboxJob(src, stride, shw[0], shw[1], dhw[0], dhw[1], top, left, kind, kx, ky, word,
                              word + xt.size, 0)
        word += xt.size + yt.size
        return j

    pre_jobs = (_lib.LetterboxJob * max(len(pre_idx), 1))()
    lb_src = list(src_ptr)
    for k, b in enumerate(pre_idx):
        pre_jobs[k] = lb_job(*src_ptr[b], plan[b][0], plan[b][1], 0, 0, pre_packs[k])
        lb_src[b] = (pre_base + k * pre_hw[0] * pre_hw[1] * 3, pre_hw[1] * 3)
    lb_jobs = (_lib.LetterboxJob * bsz)()
    for b in range(bsz):
        hw0, pre, nhw, top, left, _ = plan[b]
        lb_jobs[b] = lb_job(*lb_src[b], pre or hw0, nhw, top, left, lb_packs[b])
    warp_jobs = (_lib.WarpJob * max(len(warp_idx), 1))()
    fin_src = [(lb_base + b * img_bytes, W * 3) for b in range(bsz)]
    k_w = 0
    for k, b in enumerate(warp_idx):
        rec = plan[b][5]
        m = (ctypes.c_double * 6)()
        if rec["affine"] is not None:
            m[:] = invert_affine(affine_matrix(rec["affine"], out_hw))
            dst = warp_base + k_w * img_bytes
            fin_src[b] = (dst, W * 3)
            k_w += 1
            warp_jobs[k] = _lib.WarpJob(lb_base + b * img_bytes, dst, W * 3, m, 1, b)
        else:
            warp_jobs[k] = _lib.WarpJob(lb_base + b * img_bytes, None, W * 3, m, 0, b)
    fin_jobs = (_lib.FinishJob * bsz)()
    for b in range(bsz):
        rec = plan[b][5]
        flags = ((1 if rec["gamma"] is not None else 0) | (2 if rec["hsv"] is not None else 0)
                 | (4 if rec["hflip"] else 0) | (8 if rec["vflip"] else 0))
        hs, hv = (np.float32(rec["hsv"][0]), np.float32(rec["hsv"][1])) if rec["hsv"] is not None else (1.0, 1.0)
        fin_jobs[b] = _lib.FinishJob(fin_src[b][0], fin_src[b][1], rec["gamma"] if rec["gamma"] is not None else 1.0,
                                     float(hs), float(hv), flags, 0)
    for off, arr, n in ((o_pre, pre_jobs, len(pre_idx) * _JOB_BYTES), (o_lb, lb_jobs, bsz * _JOB_BYTES),
                        (o_warp, warp_jobs, len(warp_idx) * _WARP_BYTES), (o_fin, fin_jobs, bsz * _FIN_BYTES)):
        stage[off:off + n] = np.frombuffer(bytes(arr), np.uint8)[:n]
    stage[o_tgt:o_tgt + targets.nbytes] = targets.reshape(-1).view(np.uint8)
    dev.copy_(pinned[:total], non_blocking=True)
    ev = torch.cuda.Event()
    ev.record()
    _staging[device.index] = (pinned, ev)
    tab_ptr = ctypes.c_void_p(base + o_tab)

    def launch():
        st = _lib.stream_ptr(device)
        if pre_idx:
            _lib.check(_lib.lib.ryolo_letterbox(ctypes.c_void_p(base + o_pre), len(pre_idx), tab_ptr,
                                                ctypes.c_void_p(pre_base), pre_hw[0], pre_hw[1], _lib.DT_U8, st),
                       "ryolo_letterbox (pre-resize)")
        _lib.check(_lib.lib.ryolo_letterbox(ctypes.c_void_p(base + o_lb), bsz, tab_ptr, ctypes.c_void_p(lb_base),
                                            H, W, _lib.DT_U8, st), "ryolo_letterbox")
        if warp_idx:
            _lib.check(_lib.lib.ryolo_augment_warp(ctypes.c_void_p(base + o_warp), len(warp_idx),
                                                   ctypes.c_void_p(rowmax), H, W, st), "ryolo_augment_warp")
        _lib.check(_lib.lib.ryolo_augment_finish(ctypes.c_void_p(base + o_fin), bsz, ctypes.c_void_p(rowmax),
                                                 _lib.ptr(out), H, W,
                                                 _lib.DT_F32 if dtype == torch.float32 else _lib.DT_F16, st),
                   "ryolo_augment_finish")

    tgt = dev[o_tgt:o_tgt + targets.nbytes].view(torch.float32).view(-1, 7)
    return launch, tgt, (dev, ws)
