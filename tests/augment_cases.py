"""TEST INFRASTRUCTURE: the augmentation fixture's batches and the numpy restatements of the augmentation kernels'
arithmetic (warp, 8-bit HSV, gamma tables) that test_augment_cpu.py checks against cv2 / numpy and
test_augment_gpu.py checks the device against."""
import os

import numpy as np

from helpers import GOLDEN

GOLD = os.path.join(GOLDEN, "augment_golden.npz")
f32 = np.float32
# a draw record in which nothing fires
DRAW_KEYS_NONE = {"gray_alpha": 1.0, "affine": None, "noise": False, "gamma": None, "blur": False, "hsv": None,
                  "hflip": False, "vflip": False, "grayscale": False}


def aug_module():
    import rotate_yolov3_b200.augment as aug
    return aug


def augment_golden():
    return np.load(GOLD)


def _load_generator():
    """the fixture generator as a module: its seeded sources, label rows and draw recorder are the tests' own, so the
    two cannot drift apart (loading it imports neither the reference nor cv2)"""
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden_augment", os.path.join(GOLDEN, "make_golden_augment.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


GEN = _load_generator()
KINDS = ("random", "dim", "black")             # the fixture stores a source's kind as its index here
Recorder = GEN.Recorder
label_rows = GEN.label_rows


def source(seed, h, w, kind=0):
    return GEN.source(seed, h, w, KINDS[kind])


def batch_case(g, name):
    """a fixture batch: (seed, hyp, new_shape, mode, img_size, source images, label rows, key prefix)"""
    k = "batch_%s_" % name
    hyp = dict(zip([str(v) for v in g[k + "hyp_keys"]], [float(v) for v in g[k + "hyp"]]))
    ns = g[k + "new_shape"]
    mode = str(g[k + "mode"])
    new_shape = int(ns[0]) if mode == "square" else (int(ns[0]), int(ns[1]))
    seed = int(g[k + "seed"])
    specs = [tuple(int(v) for v in r) for r in g[k + "specs"]]
    imgs = [source(100 * seed + i, h, w, kind) for i, (h, w, kind, n) in enumerate(specs)]
    labs = [label_rows(100 * seed + i, n) for i, (h, w, kind, n) in enumerate(specs)]
    return seed, hyp, new_shape, mode, int(g[k + "img_size"]), imgs, labs, k


# ---- restatements ----------------------------------------------------------------------------------------------

def warp_np(img, minv, border=128):
    """ryolo_augment_warp restated: cv2's fixed-point bilinear remap of warpAffine"""
    h, w = img.shape[:2]
    x = np.arange(w, dtype=np.float64)
    y = np.arange(h, dtype=np.float64)
    adelta = np.rint(minv[0] * x * 1024.0).astype(np.int64)
    bdelta = np.rint(minv[3] * x * 1024.0).astype(np.int64)
    X0 = np.rint((minv[1] * y + minv[2]) * 1024.0).astype(np.int64) + 16
    Y0 = np.rint((minv[4] * y + minv[5]) * 1024.0).astype(np.int64) + 16
    X = (X0[:, None] + adelta[None, :]) >> 5
    Y = (Y0[:, None] + bdelta[None, :]) >> 5
    sx, sy, ax, ay = X >> 5, Y >> 5, X & 31, Y & 31
    acc = np.zeros((h, w, 3), np.int64)
    for dy in (0, 1):
        for dx in (0, 1):
            wt = ((32 - ay) if dy == 0 else ay) * ((32 - ax) if dx == 0 else ax) * 32
            xx, yy = sx + dx, sy + dy
            inside = (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
            v = np.where(inside[..., None], img[np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)].astype(np.int64), border)
            acc += v * wt[..., None]
    return ((acc + 16384) >> 15).astype(np.uint8)


def _hsv_tables():
    i = np.arange(1, 256, dtype=np.float64)
    sdiv, hdiv = np.zeros(256, np.int64), np.zeros(256, np.int64)
    sdiv[1:] = np.rint((255 << 12) / i)
    hdiv[1:] = np.rint((180 << 12) / (6.0 * i))
    return sdiv, hdiv


def bgr2hsv_np(img):
    sdiv, hdiv = _hsv_tables()
    b, g, r = (img[..., k].astype(np.int64) for k in range(3))
    v = np.maximum(np.maximum(b, g), r)
    diff = v - np.minimum(np.minimum(b, g), r)
    s = (diff * sdiv[v] + 2048) >> 12
    h = np.where(v == r, g - b, np.where(v == g, b - r + 2 * diff, r - g + 4 * diff))
    h = (h * hdiv[diff] + 2048) >> 12
    return np.stack([h + np.where(h < 0, 180, 0), s, v], -1).astype(np.uint8)


def _fma(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c).astype(np.float32)


SECTORS = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])


def hsv2bgr_np(hsv, vec_pixels=32):
    """cv2's 8-bit HSV2BGR: vector blocks of vec_pixels per row (fused 1 - s*h, truncation), scalar tail (rounding)"""
    h = hsv[..., 0].astype(f32)
    s = hsv[..., 1].astype(f32) * f32(1 / 255)
    v = hsv[..., 2].astype(f32) * f32(1 / 255)
    hh = h * f32(6 / 180)
    pre = np.trunc(hh)
    fr = hh - pre
    sec = (pre - np.trunc(pre * f32(1 / 6)) * f32(6)).astype(np.int64)
    one = f32(1)
    tab = np.stack([v, v * (one - s), v * _fma(-s, fr, 1.0), v * _fma(-s, one - fr, 1.0)], -1)
    out = np.stack([np.take_along_axis(tab, SECTORS[sec][..., k:k + 1], -1)[..., 0] for k in range(3)], -1) * f32(255)
    w = hsv.shape[1]
    vec = np.arange(w) < w // vec_pixels * vec_pixels
    q = np.where(vec[None, :, None], np.trunc(out), np.rint(out))
    return np.clip(q, 0, 255).astype(np.uint8)


def hsv_np(img, a, b):
    hsv = bgr2hsv_np(img)
    S = hsv[..., 1].astype(f32) * f32(a)
    V = hsv[..., 2].astype(f32) * f32(b)
    hsv[..., 1] = np.minimum(S, f32(255))
    hsv[..., 2] = np.minimum(V, f32(255))
    return hsv2bgr_np(hsv)


def gamma_table_np(m, gm):
    """what the finish kernel's per-image table holds: numpy's uint8(power(v / float(M), gm) * M) for v <= M"""
    v = np.arange(256)
    if m == 0:
        return np.zeros(256, np.uint8)
    t = np.uint8(np.power(v[: m + 1] / float(m), gm) * np.uint8(m))
    return np.concatenate([t, np.zeros(255 - m, np.uint8)])


def all_colours():
    c = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8)
