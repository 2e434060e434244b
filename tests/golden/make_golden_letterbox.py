#!/usr/bin/env python
"""Golden fixtures of the letterbox step: the REFERENCE's own ``letterbox`` and ``LoadImages`` normalisation
(utils/datasets.py:49-129, :512-546) and ``scale_coords`` (utils/utils.py:181-189), run here on the CPU with cv2.

    letterbox_golden.npz
        case_*          per case: seed, source shape, new_shape, mode; SHA-256 of the fp32 and fp16 network input
                        bytes ([3, H, W] C order); for the small cases and the mostly-border upscales also the
                        letterboxed uint8 image (HWC BGR) itself
        geo_*           a sweep of ~200 shapes: new_unpad, the four borders and (ratiow, ratioh, padw, padh)
        sc_*            scale_coords inputs and outputs
        lab_*           the LoadImagesAndLabels label transform with augment=False (:453-467, :489-490)

Sources are regenerated from seeds by the tests (``source(seed, h, w)``); the fixture stores no source pixels.
Not run by the test-suite (the GPU box has no reference checkout).  Re-run: python tests/golden/make_golden_letterbox.py"""
import hashlib
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

# name, source (h, w), new_shape, mode; ids are the seeds
CASES = [
    ("land_1024x768", (768, 1024), 608, "square"),
    ("hd_1920x1080", (1080, 1920), 608, "square"),
    ("portrait", (1000, 700), 608, "square"),
    ("odd", (333, 517), 320, "square"),
    ("odd_small", (101, 37), 53, "square"),
    ("half_pad", (767, 1024), 608, "square"),
    ("int2x2", (912, 1216), 608, "square"),
    ("int2x2_small", (6, 10), 5, "square"),
    ("int3x3", (1368, 1824), 608, "square"),
    ("int4x3", (3, 32), 8, "square"),
    ("upscale", (300, 400), 608, "square"),
    ("upscale_portrait", (200, 150), 416, "square"),
    ("mixed", (1, 470), 608, "square"),
    ("one_px_wide", (400, 1), 608, "square"),
    ("no_resize", (456, 608), 608, "square"),
    ("no_resize_rect", (320, 608), (352, 608), "rect"),
    ("rect", (768, 1024), (480, 608), "rect"),
    ("rect_hd", (1080, 1920), (352, 608), "rect"),
    ("upscale_small", (60, 80), 96, "square"),
    ("upscale_portrait_small", (50, 37), 128, "square"),
    ("e2e", (97, 133), 128, "square"),
]
# the uint8 letterboxed image itself is stored for cases up to SMALL pixels and for the mostly-border upscale cases
# (they compress to a few kB); the large random-content cases keep digests only
SMALL = 20000
STORE = {"mixed", "one_px_wide"}


def source(seed, h, w):
    """the seeded uint8 BGR source image of a case (the tests regenerate it the same way)"""
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def import_datasets():
    import make_golden as mg
    ia = types.ModuleType("imgaug")
    iaa = types.ModuleType("imgaug.augmenters")
    ia.augmenters = iaa
    sys.modules.update({"imgaug": ia, "imgaug.augmenters": iaa})
    ru = mg.import_reference()[0]
    import utils.datasets as rd  # noqa
    return rd, ru


def main():
    import cv2
    rd, ru = import_datasets()
    sav = {"cv2_version": cv2.__version__}
    tmp = tempfile.mkdtemp()
    for seed, (name, (h, w), new_shape, mode) in enumerate(CASES):
        img0 = source(seed, h, w)
        if mode == "square":                     # LoadImages itself, from a lossless file
            path = os.path.join(tmp, "%s.png" % name)
            cv2.imwrite(path, img0)
            _, x32, back, _ = next(iter(rd.LoadImages(path, img_size=new_shape, half=False)))
            _, x16, _, _ = next(iter(rd.LoadImages(path, img_size=new_shape, half=True)))
            assert (back == img0).all()
        lb, rw, rh, dw, dh = rd.letterbox(img0, new_shape=new_shape, mode=mode)
        if mode == "rect":                       # LoadImagesAndLabels' normalisation (:498-500), fp16 as LoadImages
            x32 = np.ascontiguousarray(lb[:, :, ::-1].transpose(2, 0, 1), dtype=np.float32)
            x32 /= 255.0
            x16 = np.ascontiguousarray(lb[:, :, ::-1].transpose(2, 0, 1), dtype=np.float16)
            x16 /= 255.0
        k = "case_%s_" % name
        sav[k + "seed"] = seed
        sav[k + "src"] = np.array([h, w])
        sav[k + "new_shape"] = np.array(new_shape).reshape(-1)
        sav[k + "mode"] = mode
        sav[k + "meta"] = np.array([rw, rh, dw, dh], np.float64)
        sav[k + "out_hw"] = np.array(x32.shape[1:])
        sav[k + "sha32"] = sha(x32)
        sav[k + "sha16"] = sha(x16)
        if lb.shape[0] * lb.shape[1] <= SMALL or name in STORE:
            sav[k + "lb"] = lb
        print(name, (h, w), "->", x32.shape, flush=True)
    sav["cases"] = np.array([c[0] for c in CASES])

    # geometry sweep: an all-255 source, so the first non-border row / column locates top / left
    rng = np.random.default_rng(1234)
    geo = []
    while len(geo) < 200:
        h, w = (int(v) for v in rng.integers(1, 2400, 2))
        if rng.random() < 0.7:
            mode, ns = "square", int(rng.choice([320, 416, 512, 608, 800]))
        else:
            mode, ns = "rect", (int(rng.choice([320, 352, 480, 608])), 608)
        try:
            lb, rw, rh, dw, dh = rd.letterbox(np.full((h, w, 3), 255, np.uint8), new_shape=ns, mode=mode)
        except cv2.error:
            continue                             # a side resized to 0 pixels: the reference fails too
        ys, xs = np.nonzero(lb[:, :, 0] == 255)
        top, left = int(ys.min()), int(xs.min())
        nh, nw = int(ys.max()) - top + 1, int(xs.max()) - left + 1
        nsh = (ns, ns) if mode == "square" else ns
        geo.append((h, w, nsh[0], nsh[1], mode == "rect", nh, nw, top, lb.shape[0] - top - nh, left,
                    lb.shape[1] - left - nw, rw, rh, dw, dh))
    sav["geo"] = np.array(geo, np.float64)

    # scale_coords: boxes of the letterboxed image back to the source, float32 as the reference's det tensor
    g = torch.Generator().manual_seed(77)
    for i, (img1, img0) in enumerate([((608, 608), (768, 1024)), ((608, 608), (1080, 1920)), ((608, 608), (300, 400)),
                                      ((352, 608), (1080, 1920)), ((608, 608), (1000, 700))]):
        c = torch.rand(50, 5, generator=g) * torch.tensor([608.0, 608.0, 200.0, 100.0, 3.0])
        sav["sc_%d_in" % i] = c.numpy().copy()
        sav["sc_%d_shapes" % i] = np.array([img1, img0])
        sav["sc_%d_out" % i] = ru.scale_coords(img1, c.clone()[:, :4], img0 + (3,)).numpy()

    # labels: the transform of LoadImagesAndLabels.__getitem__ with augment=False, on seeded label rows
    lab_in, lab_out, lab_shapes, lab_meta = [], [], [], []
    for i, (name, (h, w), new_shape, mode) in enumerate(CASES[:6] + CASES[15:18]):
        x = np.random.default_rng(500 + i).random((4, 6)).astype(np.float32)
        _, ratiow, ratioh, padw, padh = rd.letterbox(np.zeros((h, w, 3), np.uint8), new_shape=new_shape, mode=mode)
        img = np.zeros(((new_shape, new_shape) if mode == "square" else new_shape) + (3,), np.uint8)
        labels = x.copy()
        labels[:, 1] = ratiow * w * labels[:, 1] + padw
        labels[:, 2] = ratioh * h * labels[:, 2] + padh
        labels[:, 3] = ratiow * w * labels[:, 3]
        labels[:, 4] = ratioh * h * labels[:, 4]
        labels[:, [2, 4]] /= img.shape[0]
        labels[:, [1, 3]] /= img.shape[1]
        lab_in.append(x)
        lab_out.append(labels)
        lab_shapes.append((h, w) + img.shape[:2])
        lab_meta.append((ratiow, ratioh, padw, padh))
    sav["lab_in"] = np.stack(lab_in)
    sav["lab_out"] = np.stack(lab_out)
    sav["lab_shapes"] = np.array(lab_shapes)
    sav["lab_meta"] = np.array(lab_meta, np.float64)
    np.savez_compressed(os.path.join(HERE, "letterbox_golden.npz"), **sav)
    print("wrote", os.path.join(HERE, "letterbox_golden.npz"))


if __name__ == "__main__":
    main()
