"""Letterboxing of detection and evaluation images on the device: uint8 BGR images in, the reference's network input
out (``utils/datasets.py``: ``letterbox`` followed by the ``LoadImages`` / ``LoadImagesAndLabels`` normalisation).

The output is byte for byte what the reference computes on the host with ``cv2.resize(..., INTER_AREA)``,
``cv2.copyMakeBorder`` (grey 128), BGR->RGB, CHW and ``/255`` in float32 (or float16 for ``--half``).  cv2's area
resize takes one of three arithmetic paths, chosen from the shapes alone, and ``resample_tables`` restates each one:

* ``AREA``      both axes downscale by non-integer factors: float32 tap weights, row sums and weighted row
                accumulation in cv2's order;
* ``AREA_INT``  both axes downscale by integer factors: integer block sums, ``(s + 2) >> 2`` for 2x2 and
                ``rint(s * float(1/area))`` otherwise;
* ``LINEAR``    either axis upscales: two-tap linear resampling with area-derived 11-bit fixed-point weights and
                cv2's rounding shifts in the vertical pass.

No resize (source already at the target size) is an ``AREA`` job with one unit tap per pixel, which copies.
The tables depend on shapes only, so they are built on the host in float64 rounded to float32, as cv2 builds them.
Everything runs in one kernel launch per batch (``ryolo_letterbox``); there is no host fallback."""
import ctypes
import functools
import math

import numpy as np
import torch

from . import _lib

AREA, AREA_INT, LINEAR = 0, 1, 2
DBL_EPSILON = np.finfo(np.float64).eps
COEF_SCALE = 2048                     # cv2's INTER_RESIZE_COEF_SCALE (11 fractional bits)


def geometry(shape, new_shape=608, mode="square"):
    """The reference's letterbox geometry from shapes alone.  shape: (h, w) of the source.  Returns
    (new_unpad_hw, (top, bottom, left, right), (ratiow, ratioh, dw, dh)) exactly as ``letterbox`` computes them."""
    if mode == "square":
        if not isinstance(new_shape, int):
            raise ValueError("mode='square' takes an int new_shape, got %r" % (new_shape,))
        ratio = float(new_shape) / max(shape)
    elif mode == "rect":
        if isinstance(new_shape, int) or len(new_shape) != 2:
            raise ValueError("mode='rect' takes new_shape=(h, w), got %r" % (new_shape,))
        ratio = max(new_shape) / max(shape)
    else:
        raise ValueError("mode must be 'square' or 'rect', got %r" % (mode,))
    new_w, new_h = int(round(shape[1] * ratio)), int(round(shape[0] * ratio))
    if mode == "square":
        dw, dh = (new_shape - new_w) / 2, (new_shape - new_h) / 2
    else:
        dw, dh = (new_shape[1] - new_w) / 2, (new_shape[0] - new_h) / 2
    top, bottom = int(round(dh - 0.1)), int(round(dh + 0.1))
    left, right = int(round(dw - 0.1)), int(round(dw + 0.1))
    return (new_h, new_w), (top, bottom, left, right), (ratio, ratio, dw, dh)


def _area_axis(ssize, dsize, scale):
    """cv2's computeResizeAreaTab for one axis: per output index the first source index, the tap count and the
    float32 weights (a partial pixel, the whole pixels, a partial pixel; overlaps <= 1e-3 dropped)."""
    starts, counts, weights = [], [], []
    for d in range(dsize):
        fs1 = d * scale
        fs2 = fs1 + scale
        cell = min(scale, ssize - fs1)
        s2 = min(math.floor(fs2), ssize - 1)
        s1 = min(math.ceil(fs1), s2)
        w = []
        start = s1
        if s1 - fs1 > 1e-3:
            start = s1 - 1
            w.append((s1 - fs1) / cell)
        w.extend([1.0 / cell] * (s2 - s1))
        if fs2 - s2 > 1e-3:
            w.append(min(min(fs2 - s2, 1.0), cell) / cell)
        starts.append(start)
        counts.append(len(w))
        weights.append(np.array(w, np.float64).astype(np.float32))
    return starts, counts, weights


def _linear_axis(ssize, dsize, scale, inv_scale, clamp_last):
    """cv2's area-mode coefficients of the linear resampler for one axis: source index sy = floor(d * scale) and the
    two 11-bit weights rint((1 - f) * 2048), rint(f * 2048) of f = frac((d + 1) - (sy + 1) * inv_scale) in float32.
    Horizontally cv2 pins f = 0 at the last source pixel (clamp_last); vertically it keeps f and clips the second row."""
    starts, weights = [], []
    for d in range(dsize):
        s = math.floor(d * scale)
        f = np.float32((d + 1) - (s + 1) * inv_scale)
        f = np.float32(0) if f <= 0 else np.float32(f - np.float32(math.floor(f)))
        if clamp_last and s >= ssize - 1:
            f, s = np.float32(0), ssize - 1
        a0 = int(np.rint(np.float32(np.float32(1) - f) * np.float32(COEF_SCALE)))
        a1 = int(np.rint(f * np.float32(COEF_SCALE)))
        starts.append(s)
        weights.append((a0, a1))
    return starts, weights


def _linear_resize_axis(ssize, dsize, scale):
    """cv2.resize(INTER_LINEAR)'s coefficients for one axis: fx = float32((d + 0.5) * scale - 0.5), sx = floor(fx),
    clamped to the image at both ends (fx = 0 there), and the 11-bit weights rint((1 - f) * 2048), rint(f * 2048)"""
    starts, weights = [], []
    for d in range(dsize):
        fx = np.float32((d + 0.5) * scale - 0.5)
        s = math.floor(fx)
        f = np.float32(fx - np.float32(s))
        if s < 0:
            f, s = np.float32(0), 0
        if s >= ssize - 1:
            f, s = np.float32(0), ssize - 1
        a0 = int(np.rint(np.float32(np.float32(1) - f) * np.float32(COEF_SCALE)))
        a1 = int(np.rint(f * np.float32(COEF_SCALE)))
        starts.append(s)
        weights.append((a0, a1))
    return starts, weights


def linear_resize_tables(src_hw, dst_hw):
    """The arithmetic path cv2.resize(INTER_LINEAR) takes for this pair of shapes, in resample_tables' format: an
    exact 2x downscale on both axes runs as INTER_AREA's 2x2 block mean (AREA_INT), every other pair as LINEAR."""
    (sh, sw), (dh, dw) = src_hw, dst_hw
    sx, sy = 1.0 / (dw / sw), 1.0 / (dh / sh)
    if (sh, sw) == (dh, dw):
        return resample_tables(src_hw, dst_hw)
    ix, iy = int(np.rint(sx)), int(np.rint(sy))
    if ix == 2 and iy == 2 and abs(sx - ix) < DBL_EPSILON and abs(sy - iy) < DBL_EPSILON:
        xs = ([2 * d for d in range(dw)], [2] * dw, None)
        return AREA_INT, (2, 2), xs, ([2 * d for d in range(dh)], [2] * dh, None)
    xs0, xw = _linear_resize_axis(sw, dw, sx)
    ys0, yw = _linear_resize_axis(sh, dh, sy)
    return LINEAR, (0, 0), (xs0, [2] * dw, xw), (ys0, [2] * dh, yw)


def resample_tables(src_hw, dst_hw):
    """The arithmetic path cv2.resize(INTER_AREA) takes for this pair of shapes, and its per-axis tables.

    Returns (kind, (kx, ky), xtab, ytab).  Each tab is (starts [dsize] int, counts [dsize] int, weights): for AREA the
    weights are a list of float32 arrays (one per output index), for LINEAR a list of (w0, w1) int pairs (the second
    source index is start + 1 clipped to the image), for AREA_INT None (start = d * k, count = k)."""
    (sh, sw), (dh, dw) = src_hw, dst_hw
    inv_x, inv_y = dw / sw, dh / sh                 # cv2::resize with an explicit dsize
    sx, sy = 1.0 / inv_x, 1.0 / inv_y
    if (sh, sw) == (dh, dw):
        xs = (list(range(dw)), [1] * dw, [np.ones(1, np.float32)] * dw)
        ys = (list(range(dh)), [1] * dh, [np.ones(1, np.float32)] * dh)
        return AREA, (0, 0), xs, ys
    if sx >= 1 and sy >= 1:
        ix, iy = int(np.rint(sx)), int(np.rint(sy))
        if abs(sx - ix) < DBL_EPSILON and abs(sy - iy) < DBL_EPSILON:
            xs = ([d * ix for d in range(dw)], [ix] * dw, None)
            ys = ([d * iy for d in range(dh)], [iy] * dh, None)
            return AREA_INT, (ix, iy), xs, ys
        return AREA, (0, 0), _area_axis(sw, dw, sx), _area_axis(sh, dh, sy)
    xs0, xw = _linear_axis(sw, dw, sx, inv_x, True)
    ys0, yw = _linear_axis(sh, dh, sy, inv_y, False)
    return LINEAR, (0, 0), (xs0, [2] * dw, xw), (ys0, [2] * dh, yw)


def _pack_axis(tab, kind):
    """one axis table as int32 words: dsize entries {start, count, woff} followed by the weights (woff relative to
    the start of this block)"""
    starts, counts, weights = tab
    n = len(starts)
    ent = np.zeros((n, 3), np.int32)
    ent[:, 0], ent[:, 1] = starts, counts
    if kind == AREA_INT:
        return ent.reshape(-1)
    if kind == AREA:
        flat = np.concatenate(weights).astype(np.float32).view(np.int32)
        ent[:, 2] = 3 * n + np.concatenate([[0], np.cumsum(counts)[:-1]])
    else:
        flat = np.asarray(weights, np.int32).reshape(-1)
        ent[:, 2] = 3 * n + 2 * np.arange(n)
    return np.concatenate([ent.reshape(-1), flat])


@functools.lru_cache(maxsize=256)
def _packed(src_hw, dst_hw, linear=False):
    kind, (kx, ky), xt, yt = (linear_resize_tables if linear else resample_tables)(src_hw, dst_hw)
    return kind, kx, ky, _pack_axis(xt, kind), _pack_axis(yt, kind)


_JOB_BYTES = ctypes.sizeof(_lib.LetterboxJob)
_staging = {}          # device index -> (pinned uint8 buffer, event recorded after its last upload)


def _pinned(device, nbytes):
    """the device's pinned staging buffer, once the upload that last read it has finished"""
    buf, ev = _staging.get(device.index, (None, None))
    if ev is not None:
        ev.synchronize()
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, pin_memory=True)
    return buf


def _check_image(img, i):
    if img.ndim != 3 or img.shape[2] != 3:
        raise ValueError("letterbox: image %d must be [H, W, 3] BGR, got shape %s" % (i, tuple(img.shape)))
    if img.shape[0] < 1 or img.shape[1] < 1:
        raise ValueError("letterbox: image %d is empty (%s)" % (i, tuple(img.shape)))


def _sources(images, device):
    """the checked images: CUDA tensors on `device` with rows of packed pixels, host images as C-contiguous numpy"""
    srcs = []
    for i, im in enumerate(images):
        if isinstance(im, torch.Tensor):
            if im.dtype != torch.uint8:
                raise ValueError("letterbox: image %d must be uint8, got %s" % (i, im.dtype))
            _check_image(im, i)
            if im.is_cuda:
                if im.device != device:
                    raise ValueError("letterbox: image %d is on %s, not %s" % (i, im.device, device))
                if im.stride(2) != 1 or im.stride(1) != 3:
                    im = im.contiguous()
                srcs.append(im)
                continue
            im = im.numpy()
        im = np.asarray(im)
        if im.dtype != np.uint8:
            raise ValueError("letterbox: image %d must be uint8, got %s" % (i, im.dtype))
        _check_image(im, i)
        srcs.append(np.ascontiguousarray(im))
    return srcs


def upload_images(images, device):
    """The images as uint8 [H, W, 3] CUDA tensors on `device`, for callers that letterbox the same images at several
    sizes: host images are staged in the pinned buffer and uploaded with one copy on the current stream, CUDA images
    are returned as they are.  images: as ``letterbox`` takes them."""
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("upload_images needs a CUDA device, got %s" % (device,))
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    if not isinstance(images, (list, tuple)) or len(images) == 0:
        raise ValueError("letterbox: images must be a non-empty list of [H, W, 3] uint8 images")
    srcs = _sources(images, device)
    offs, total = [], 0
    for s in srcs:
        offs.append(total)
        total += s.nbytes if isinstance(s, np.ndarray) else 0
    if total == 0:
        return srcs
    with torch.cuda.device(device):
        pinned = _pinned(device, total)
        stage = pinned[:total].numpy()
        for s, o in zip(srcs, offs):
            if isinstance(s, np.ndarray):
                stage[o:o + s.nbytes] = s.reshape(-1)
        dev = _send(pinned, torch.empty(total, dtype=torch.uint8, device=device), device)
    return [dev[o:o + s.nbytes].view(s.shape) if isinstance(s, np.ndarray) else s for s, o in zip(srcs, offs)]


def upload_table(arr, device):
    """a small host array (a job or coefficient table) as a uint8 device buffer, through the pinned staging buffer"""
    raw = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
    pinned = _pinned(device, raw.size)
    pinned[:raw.size].numpy()[:] = raw
    return _send(pinned, torch.empty(raw.size, dtype=torch.uint8, device=device), device)


def _send(pinned, dev, device):
    """one H2D copy of the first dev.numel() staged bytes into dev on the current stream; the staging buffer is free
    again once the event recorded after the copy has completed (_pinned waits for it)"""
    dev.copy_(pinned[:dev.numel()], non_blocking=True)
    ev = torch.cuda.Event()
    ev.record()
    _staging[device.index] = (pinned, ev)
    return dev


def letterbox(images, new_shape=608, mode="square", dtype=torch.float32, device=None, out=None):
    """The reference's ``letterbox`` + network-input normalisation for a batch of images, on the device.

    images: list of uint8 [H, W, 3] BGR arrays (numpy or CPU tensors, as ``cv2.imread`` returns) or CUDA tensors;
    sizes may differ.  Host images are staged in one pinned buffer and uploaded with one copy on the current stream;
    CUDA images are read where they are (so a caller letterboxing the same images at several sizes uploads once).
    new_shape: int for mode='square', (h, w) for mode='rect' (ratio max(new_shape) / max(shape)).
    dtype: torch.float32, or torch.float16 as ``LoadImages(half=True)`` / ``detect.py --half``.
    out: optional [B, 3, H, W] CUDA tensor of `dtype` to write into.  A call with out= and CUDA images only can be
    captured in a CUDA graph once the same call has run outside the capture (the job table is kept with `out`).

    Returns (imgs [B, 3, H, W], meta): meta is a host float64 [B, 4] tensor of (ratiow, ratioh, padw, padh), what the
    reference's letterbox returns, computed from shapes alone."""
    if dtype not in (torch.float32, torch.float16):
        raise ValueError("letterbox: dtype must be torch.float32 or torch.float16, got %s" % (dtype,))
    if not isinstance(images, (list, tuple)) or len(images) == 0:
        raise ValueError("letterbox: images must be a non-empty list of [H, W, 3] uint8 images")
    if len(images) > 65535:
        raise ValueError("letterbox: at most 65535 images per call, got %d" % len(images))
    if device is None:
        device = next((im.device for im in images if isinstance(im, torch.Tensor) and im.is_cuda),
                      out.device if out is not None else torch.device("cuda", torch.cuda.current_device()))
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("letterbox runs on a CUDA device only, got %s (there is no CPU path)" % (device,))
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    if mode == "square":
        out_hw = (int(new_shape), int(new_shape)) if isinstance(new_shape, int) else None
    else:
        out_hw = tuple(int(v) for v in new_shape) if not isinstance(new_shape, int) and len(new_shape) == 2 else None
    if out_hw is None:
        geometry((1, 1), new_shape, mode)                   # raises the ValueError for the bad new_shape / mode
    srcs = _sources(images, device)
    bsz = len(srcs)
    meta = torch.empty((bsz, 4), dtype=torch.float64)
    geo = []
    for b, s in enumerate(srcs):
        (nh, nw), (top, bottom, left, right), m = geometry(tuple(s.shape[:2]), new_shape, mode)
        if nh < 1 or nw < 1 or top < 0 or left < 0 or top + nh + bottom != out_hw[0] or left + nw + right != out_hw[1]:
            raise ValueError("letterbox: image %d of shape %s does not letterbox into %s (resized %s, borders %s)"
                             % (b, tuple(s.shape[:2]), out_hw, (nh, nw), (top, bottom, left, right)))
        meta[b] = torch.tensor(m, dtype=torch.float64)
        geo.append(((nh, nw), top, left))
    if out is None:
        out = torch.empty((bsz, 3) + out_hw, dtype=dtype, device=device)
    elif (not out.is_cuda or out.device != device or out.dtype != dtype or tuple(out.shape) != (bsz, 3) + out_hw
          or not out.is_contiguous()):
        raise ValueError("letterbox: out must be a contiguous %s CUDA tensor %s on %s, got %s %s on %s"
                         % (dtype, [bsz, 3, *out_hw], device, out.dtype, list(out.shape), out.device))
    all_cuda = all(isinstance(s, torch.Tensor) for s in srcs)
    key = (tuple((s.data_ptr(), s.stride(0), tuple(s.shape)) for s in srcs), tuple(geo), mode) if all_cuda else None
    capturing = torch.cuda.is_current_stream_capturing()
    with torch.cuda.device(device):
        kept = getattr(out, "_ryolo_letterbox", None)
        if key is not None and kept is not None and kept[0] == key:
            dev = kept[1]
        elif capturing:
            raise RuntimeError("letterbox under CUDA-graph capture needs CUDA images, out=, and the same call run once "
                               "before the capture (it uploads the job table then)")
        else:
            dev = _upload(srcs, geo, device)
            if key is not None:
                out._ryolo_letterbox = (key, dev)
        st = _lib.lib.ryolo_letterbox(_lib.ptr(dev), bsz, ctypes.c_void_p(dev.data_ptr() + bsz * _JOB_BYTES),
                                      _lib.ptr(out), out_hw[0], out_hw[1],
                                      _lib.DT_F32 if dtype == torch.float32 else _lib.DT_F16, _lib.stream_ptr(device))
        _lib.check(st, "ryolo_letterbox")
    return out, meta


def _upload(srcs, geo, device):
    """one device buffer [jobs | tables | host images] filled by one H2D copy from the pinned staging buffer"""
    bsz = len(srcs)
    packs = [_packed(tuple(s.shape[:2]), g[0]) for s, g in zip(srcs, geo)]
    tab_words = sum(p[3].size + p[4].size for p in packs)
    img_off = bsz * _JOB_BYTES + 4 * tab_words
    img_off = (img_off + 15) // 16 * 16
    host_bytes = sum(s.nbytes for s in srcs if isinstance(s, np.ndarray))
    total = img_off + host_bytes
    dev = torch.empty(total, dtype=torch.uint8, device=device)
    pinned = _pinned(device, total)
    stage = pinned[:total].numpy()
    jobs = (_lib.LetterboxJob * bsz)()
    word, pos = 0, img_off
    tabs = stage[bsz * _JOB_BYTES:bsz * _JOB_BYTES + 4 * tab_words].view(np.int32)
    for b, (s, ((nh, nw), top, left), (kind, kx, ky, xt, yt)) in enumerate(zip(srcs, geo, packs)):
        if isinstance(s, np.ndarray):
            stage[pos:pos + s.nbytes] = s.reshape(-1)
            src, stride = dev.data_ptr() + pos, s.shape[1] * 3
            pos += s.nbytes
        else:
            src, stride = s.data_ptr(), s.stride(0)
        tabs[word:word + xt.size] = xt
        tabs[word + xt.size:word + xt.size + yt.size] = yt
        jobs[b] = _lib.LetterboxJob(src, stride, s.shape[0], s.shape[1], nh, nw, top, left, kind, kx, ky,
                                    word, word + xt.size, 0)
        word += xt.size + yt.size
    stage[:bsz * _JOB_BYTES] = np.frombuffer(bytes(jobs), np.uint8)
    return _send(pinned, dev, device)


def scale_coords_terms(img1_shape, shapes):
    """the reference's scale_coords terms per original shape, in Python floats: (padx, pady, gain) lists; the
    transform is x = (x - padx) / gain, y = (y - pady) / gain, w = w / gain, h = h / gain with each term in float32"""
    gains = [max(img1_shape) / max(s[:2]) for s in shapes]
    padx = [(img1_shape[1] - s[1] * g) / 2 for s, g in zip(shapes, gains)]
    pady = [(img1_shape[0] - s[0] * g) / 2 for s, g in zip(shapes, gains)]
    return padx, pady, gains


def scale_coords(img1_shape, coords, img0_shape):
    """Map boxes (x, y, w, h, ...) from the letterboxed image back to the original image, in place on columns 0-3,
    as the reference's ``scale_coords`` (utils/utils.py:181-189) does.  coords [n, >= 4] with img0_shape (h, w[, c]),
    or batched: coords [B, n, >= 4] with img0_shape a list of B shapes.  Every value is the reference's float32 result
    (the division is a true division on every device).  Returns coords."""
    batched = coords.dim() == 3
    shapes = list(img0_shape) if batched else [img0_shape]
    if (batched and len(shapes) != coords.shape[0]) or coords.dim() not in (2, 3) or coords.shape[-1] < 4:
        raise ValueError("scale_coords: coords [n, >=4] with one shape or [B, n, >=4] with B shapes, got %s and %d "
                         "shapes" % (tuple(coords.shape), len(shapes)))
    padx, pady, gains = scale_coords_terms(img1_shape, shapes)
    view = coords if batched else coords.unsqueeze(0)
    col = lambda v: torch.tensor(v, dtype=coords.dtype).view(-1, 1).to(coords.device, non_blocking=True)
    view[..., 0] -= col(padx)
    view[..., 1] -= col(pady)
    view[..., :4] /= col(gains).unsqueeze(-1)
    return coords


def letterbox_labels(labels, meta, shapes, out_hw):
    """``LoadImagesAndLabels``' label transform with augment=False (utils/datasets.py:453-467, :489-490) for a batch.

    labels: [N, 7] float32 in collate_fn's layout (image index, class, x, y, w, h, a) with x, y, w, h normalised to
    the source image as in the label files; meta: [B, 4] (ratiow, ratioh, padw, padh) from ``letterbox``; shapes:
    the B source shapes (h, w); out_hw: the letterboxed (h, w).  Returns a new [N, 7] tensor on labels' device:
    x, y, w, h normalised to the letterboxed image, the reference's float32 values bit for bit."""
    if labels.dim() != 2 or labels.shape[1] != 7 or labels.dtype != torch.float32:
        raise ValueError("letterbox_labels: labels must be float32 [N, 7], got %s %s" % (labels.dtype, tuple(labels.shape)))
    meta = torch.as_tensor(meta, dtype=torch.float64).cpu()
    if meta.dim() != 2 or meta.shape[1] != 4 or meta.shape[0] != len(shapes):
        raise ValueError("letterbox_labels: meta [B, 4] and B shapes, got %s and %d" % (tuple(meta.shape), len(shapes)))
    rows = [(float(m[0]) * s[1], float(m[1]) * s[0], float(m[2]), float(m[3])) for m, s in zip(meta.tolist(), shapes)]
    f = torch.tensor(rows, dtype=torch.float32).to(labels.device, non_blocking=True)     # [B, 4], each a float32
    idx = labels[:, 0].long()
    sw, sh, pw, ph = (f[idx, k] for k in range(4))
    out = labels.clone()
    out[:, 2] = sw * labels[:, 2] + pw
    out[:, 3] = sh * labels[:, 3] + ph
    out[:, 4] = sw * labels[:, 4]
    out[:, 5] = sh * labels[:, 5]
    hw = torch.tensor([float(out_hw[0]), float(out_hw[1])], dtype=torch.float32).to(labels.device, non_blocking=True)
    out[:, [3, 5]] /= hw[0]
    out[:, [2, 4]] /= hw[1]
    return out
