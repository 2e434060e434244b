#!/usr/bin/env python
"""Golden fixtures of the training augmentation: the REFERENCE's own ``LoadImagesAndLabels.__getitem__`` with
augment=True and its ``collate_fn`` (utils/datasets.py:423-509, utils/augment.py), run here on the CPU with cv2 and
numpy, with imgaug's Noise, Blur and Grayscale stubbed as identities (imgaug is not installed).

    augment_golden.npz
        batch_*     per batch case: seed, hyp, new_shape, mode, the dataset's img_size, source shapes, per-image
                    label rows; the raw Python
                    `random` values the reference drew, in order; SHA-256 of the fp32 and fp16 network input
                    ([B, 3, H, W] C order; fp16 is the fp32 input rounded once); the exact collate_fn target rows
        direct_*    random_affine, Gamma, HSV and the flips called directly with the transform forced on, on a small
                    square image: the uint8 input and output, the label rows in and out, and the draws

Sources are regenerated from seeds by the tests (``source(seed, h, w)``); the fixture stores no source pixels except
the small direct cases.  Not run by the test-suite.  Re-run: python tests/golden/make_golden_augment.py"""
import hashlib
import math
import os
import random
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

HYP5 = {"degrees": 5.0, "translate": 0.1, "scale": 0.1, "shear": 0.0, "noise": 0.01, "gamma": 0.2, "blur": 1.3,
        "hsv_s": 0.5, "hsv_v": 0.3, "grayscale": 0.3}
HYP50 = dict(HYP5, degrees=50.0, scale=0.2)


def source(seed, h, w, kind="random"):
    """the seeded uint8 BGR source image of a case (the tests regenerate it the same way)"""
    if kind == "black":
        return np.zeros((h, w, 3), np.uint8)
    img = np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)
    return img // 2 + 20 if kind == "dim" else img             # dim: maximum 147 < 255


def label_rows(seed, n):
    """seeded label rows (cls, x, y, w, h, a) in 0-1 units, with rows that leave the image after the affine, lie on
    an edge, are thinner than 4 pixels or longer than 15 x their width"""
    if n == 0:
        return np.zeros((0, 6), np.float32)
    g = np.random.default_rng(1000 + seed)
    x = np.stack([g.integers(0, 3, n), g.uniform(0.05, 0.95, n), g.uniform(0.05, 0.95, n), g.uniform(0.02, 0.4, n),
                  g.uniform(0.02, 0.3, n), g.uniform(-1.5, 1.5, n)], 1).astype(np.float32)
    x[0, 1:5] = (0.02, 0.5, 0.3, 0.1)            # leaves the image
    if n > 1:
        x[1, 1:6] = (0.5, 0.5, 1.0, 0.2, 0.0)   # spans the whole width: corners on the edges
    if n > 2:
        x[2, 3] = 0.004                          # w < 4 pixels
    if n > 3:
        x[3, 3:5] = (0.9, 0.03)                  # aspect ratio > 15
    return x


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


class Recorder:
    """the `random` module as the reference calls it, recording every value it hands out"""
    def __init__(self, seed):
        self.r = random.Random(seed)
        self.vals = []

    def random(self):
        v = self.r.random()
        self.vals.append(v)
        return v

    def uniform(self, a, b):
        v = self.r.uniform(a, b)
        self.vals.append(v)
        return v


def trunc607():
    """a long side L whose pre-resize int(L * (608 / L)) truncates to 607 (the letterbox then upscales)"""
    for L in range(609, 5000):
        if int(L * (608 / L)) == 607:
            return L
    raise RuntimeError("no truncating size")


# name, seed, hyp, new_shape, mode, [(h, w, kind, n_labels)], dataset img_size (None: new_shape, or max of it)
def batch_cases():
    L = trunc607()
    return [
        ("square_hyp5", 11, HYP5, 608, "square",
         [(768, 1024, "random", 6), (1080, 1920, "random", 5), (500, 400, "random", 0), (608, 608, "random", 4)]),
        ("square_hyp50", 12, HYP50, 608, "square",
         [(768, 1024, "random", 6), (1080, 1920, "random", 4), (300, 200, "random", 3), (608, 608, "random", 0)]),
        ("trunc607", 13, HYP50, 608, "square", [(L // 2, L, "random", 5), (L, L // 3, "random", 4)]),
        ("rect", 14, HYP5, (352, 608), "rect", [(1080, 1920, "random", 5), (300, 608, "random", 2),
                                                (700, 1400, "random", 4)]),
        # img_size 600 is no multiple of 32: batch shape ceil([0.5625, 1] * 600 / 32) * 32 = (352, 608), so the
        # pre-resize (to 600) and the batch shape (608) differ, and the letterbox upscales
        ("rect_img600", 17, HYP50, (352, 608), "rect", [(1080, 1920, "random", 5), (675, 1200, "random", 3),
                                                        (500, 1000, "random", 4)], 600),
        ("odd_width", 18, HYP50, 100, "square", [(64, 80, "random", 3), (300, 250, "random", 2),
                                                 (100, 100, "dim", 2), (90, 120, "random", 0)]),
        ("small", 15, HYP50, 96, "square", [(64, 80, "random", 3), (96, 96, "dim", 2), (40, 96, "black", 1),
                                            (100, 37, "random", 0), (200, 250, "random", 4)]),
        ("many", 16, HYP50, 128, "square", [(97 + 7 * i, 133 - 5 * i, "dim" if i % 5 == 0 else "random", i % 4 + 2)
                                            for i in range(16)]),
    ]


def import_refs():
    import make_golden as mg
    ia = types.ModuleType("imgaug")
    iaa = types.ModuleType("imgaug.augmenters")

    class _Identity:
        def __init__(self, *a, **k):
            pass

        def augment_image(self, img):
            return img

    iaa.AdditiveGaussianNoise = iaa.GaussianBlur = iaa.Grayscale = _Identity
    ia.augmenters = iaa
    sys.modules.update({"imgaug": ia, "imgaug.augmenters": iaa})
    mg.import_reference()
    import utils.augment as ra  # noqa
    import utils.datasets as rd  # noqa
    return rd, ra


def run_batch(rd, ra, seed, hyp, new_shape, mode, specs, tmp, img_size):
    ds = rd.LoadImagesAndLabels.__new__(rd.LoadImagesAndLabels)
    ds.image_weights, ds.augment, ds.hyp = False, True, hyp
    ds.img_size = img_size
    ds.rect = mode == "rect"
    ds.batch_shapes = np.array([list(new_shape)]) if ds.rect else None
    ds.batch = [0] * len(specs)
    ds.img_files, ds.label_files, ds.imgs, ds.labels = [], [], [], []
    import cv2
    for i, (h, w, kind, n) in enumerate(specs):
        p = os.path.join(tmp, "images", "%d_%d.png" % (seed, i))
        os.makedirs(os.path.dirname(p), exist_ok=True)
        cv2.imwrite(p, source(100 * seed + i, h, w, kind))
        lp = p.replace("images", "labels").replace(".png", ".txt")
        os.makedirs(os.path.dirname(lp), exist_ok=True)
        open(lp, "w").close()
        ds.img_files.append(p)
        ds.label_files.append(lp)
        ds.imgs.append(None)
        ds.labels.append(label_rows(100 * seed + i, n))
    rec = Recorder(seed)
    ra.random = rec
    batch = [ds[i] for i in range(len(specs))]
    imgs, targets, _, _ = rd.LoadImagesAndLabels.collate_fn(batch)
    return imgs.numpy(), targets.numpy(), np.array(rec.vals, np.float64)


def main():
    import cv2
    rd, ra = import_refs()
    sav = {"cv2_version": cv2.__version__}
    tmp = tempfile.mkdtemp()
    names = []
    for name, seed, hyp, ns, mode, specs, *img_size in batch_cases():
        img_size = img_size[0] if img_size else (ns if mode == "square" else max(ns))
        x32, tg, vals = run_batch(rd, ra, seed, hyp, ns, mode, specs, tmp, img_size)
        k = "batch_%s_" % name
        sav[k + "img_size"] = img_size
        sav[k + "seed"] = seed
        sav[k + "hyp"] = np.array([hyp[key] for key in sorted(hyp)], np.float64)
        sav[k + "hyp_keys"] = np.array(sorted(hyp))
        sav[k + "new_shape"] = np.array(ns).reshape(-1)
        sav[k + "mode"] = mode
        sav[k + "specs"] = np.array([(h, w, ["random", "dim", "black"].index(kd), n) for h, w, kd, n in specs])
        sav[k + "draws"] = vals
        sav[k + "sha32"] = sha(x32)
        sav[k + "sha16"] = sha(x32.astype(np.float16))
        sav[k + "targets"] = tg
        names.append(name)
        print(name, x32.shape, "targets", tg.shape, "draws", len(vals), flush=True)
    sav["batches"] = np.array(names)

    # the transforms called directly, each forced on, on a small square image
    dnames = []
    for i, (name, kind) in enumerate([("affine5", "random"), ("affine50", "random"), ("gamma", "random"),
                                      ("gamma_dim", "dim"), ("gamma_black", "black"), ("hsv_up", "random"),
                                      ("hsv_down", "random"), ("hflip", "random"), ("vflip", "random")]):
        img = source(500 + i, 96, 96, kind)
        lab = label_rows(500 + i, 5)
        lab[:, [1, 3]] *= 96
        lab[:, [2, 4]] *= 96
        rec = Recorder(500 + i)
        ra.random = rec
        if name.startswith("affine"):
            deg = 5.0 if name == "affine5" else 50.0
            out, lo = ra.random_affine(img.copy(), lab.copy(), degrees=deg, translate=0.1,
                                       scale=0.1 if deg == 5.0 else 0.2, shear=0.0)
        elif name.startswith("gamma"):
            out, lo = ra.Gamma(0.2, p=1.0)(img.copy(), lab.copy())
        elif name.startswith("hsv"):
            while True:                                    # a seed whose factors lie on the wanted side of 1
                rec = Recorder(rec.r.randrange(1 << 30))
                probe = random.Random()
                probe.setstate(rec.r.getstate())
                probe.random()
                a, b = probe.uniform(-1, 1) * 0.5 + 1, probe.uniform(-1, 1) * 0.3 + 1
                if (a > 1 and b > 1) if name == "hsv_up" else (a < 1 and b < 1):
                    break
            ra.random = rec
            out, lo = ra.HSV(0.5, 0.3, p=1.0)(img.copy(), lab.copy())
        elif name == "hflip":
            out, lo = ra.HorizontalFlip(p=1.0)(img.copy(), lab.copy())
        else:
            out, lo = ra.VerticalFlip(p=1.0)(img.copy(), lab.copy())
        k = "direct_%s_" % name
        sav[k + "seed"] = 500 + i
        sav[k + "kind"] = kind
        sav[k + "img"] = img
        sav[k + "out"] = np.ascontiguousarray(out)
        sav[k + "labels"] = lab
        sav[k + "labels_out"] = np.asarray(lo, np.float32).reshape(-1, 6)
        sav[k + "draws"] = np.array(rec.vals, np.float64)
        dnames.append(name)
        print(name, "draws", rec.vals, flush=True)
    sav["directs"] = np.array(dnames)
    np.savez_compressed(os.path.join(HERE, "augment_golden.npz"), **sav)
    print("wrote augment_golden.npz")


if __name__ == "__main__":
    main()
