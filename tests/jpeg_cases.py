"""Seeded JPEG test streams written by cv2 (libjpeg-turbo), for the decoder tests: smooth images with detail, every
sampling cv2 writes, grayscale, qualities, optimised tables, restart intervals, Exif orientation segments, and the HRSC
sample of the reference's dataset (tests/golden/hrsc_100001675.jpg)."""
import os

import cv2
import numpy as np

from helpers import GOLDEN

HRSC = os.path.join(GOLDEN, "hrsc_100001675.jpg")
SAMPLINGS = {"444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
             "420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, "440": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440,
             "411": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411}
SIZES = [(1, 1), (7, 9), (8, 8), (15, 17), (16, 16), (33, 47)]


def picture(seed, h, w):
    """a smooth gradient with noise and a few hard edges (every DCT band gets energy), uint8 BGR"""
    r = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.stack([127 + 100 * np.sin(x / (3 + c) + y / (5 + 2 * c) + seed) for c in range(3)], -1)
    img += r.normal(0, 18, img.shape)
    img[(x.astype(int) // 5 + y.astype(int) // 7) % 3 == 0] *= 0.4
    return np.clip(img, 0, 255).astype(np.uint8)


def encode(img, quality=90, sampling="420", optimize=False, restart=0, luma=None, chroma=None, progressive=False):
    params = [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_OPTIMIZE, int(optimize),
              cv2.IMWRITE_JPEG_RST_INTERVAL, restart, cv2.IMWRITE_JPEG_PROGRESSIVE, int(progressive)]
    if img.ndim == 3:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLINGS[sampling]]
    if luma is not None:
        params += [cv2.IMWRITE_JPEG_LUMA_QUALITY, luma]
    if chroma is not None:
        params += [cv2.IMWRITE_JPEG_CHROMA_QUALITY, chroma]
    ok, buf = cv2.imencode(".jpg", img, params)
    assert ok
    return buf.reshape(-1).tobytes()


def with_orientation(blob, orient, big_endian=False):
    """the stream with an APP1 Exif segment holding IFD0 orientation `orient`, spliced in after SOI"""
    bo = "big" if big_endian else "little"
    tiff = (b"MM" if big_endian else b"II") + (42).to_bytes(2, bo) + (8).to_bytes(4, bo) + (1).to_bytes(2, bo)
    tiff += (0x0112).to_bytes(2, bo) + (3).to_bytes(2, bo) + (1).to_bytes(4, bo) + orient.to_bytes(2, bo) + b"\0\0"
    tiff += (0).to_bytes(4, bo)
    payload = b"Exif\0\0" + tiff
    return blob[:2] + b"\xff\xe1" + (len(payload) + 2).to_bytes(2, "big") + payload + blob[2:]


def matrix():
    """(name, blob) over sizes x samplings x qualities x tables x restart intervals, grayscale and orientations"""
    out = []
    for si, (h, w) in enumerate(SIZES):
        img = picture(si, h, w)
        for s in SAMPLINGS:
            for q in (5, 50, 95, 100):
                out.append(("%dx%d_%s_q%d" % (h, w, s, q), encode(img, q, s)))
            out.append(("%dx%d_%s_opt_rst3" % (h, w, s), encode(img, 90, s, optimize=True, restart=3)))
        out.append(("%dx%d_gray" % (h, w), encode(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY), 75)))
    big = picture(7, 121, 163)
    for s in SAMPLINGS:
        for rst in (0, 1, 3, 17):
            out.append(("121x163_%s_rst%d" % (s, rst), encode(big, 85, s, restart=rst)))
        out.append(("121x163_%s_opt_l40_c90" % s, encode(big, 75, s, optimize=True, luma=40, chroma=90)))
        out.append(("121x163_%s_l95_c20" % s, encode(big, 75, s, luma=95, chroma=20)))
    out.append(("121x163_gray_rst1", encode(cv2.cvtColor(big, cv2.COLOR_BGR2GRAY), 95, restart=1)))
    base = encode(picture(9, 37, 53), 80, "420")
    for o in range(1, 9):
        out.append(("orient%d" % o, with_orientation(base, o, big_endian=o % 2 == 0)))
    return out


def no_sync_batch():
    """[a 64 x 256 q50 4:4:4 stream with restart interval 1 (256 small segments), an 800 x 600 stream whose entropy-coded
    segment is all zero bytes]: the second one's chunks do not synchronise"""
    small = encode(picture(13, 64, 256), 50, "444", restart=1)
    big = encode(picture(14, 600, 800), 90, "420")
    sos = big.index(b"\xff\xda")
    start = sos + 2 + int.from_bytes(big[sos + 2:sos + 4], "big")
    zeros = big[:start] + bytes(len(big) - 2 - start) + big[-2:]
    return [small, zeros]


def cmyk(img):
    """a CMYK JPEG (Adobe APP14, four components) of img, or None when PIL is not installed"""
    try:
        from PIL import Image
    except ImportError:
        return None
    import io
    buf = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(img[..., ::-1])).convert("CMYK").save(buf, "JPEG", quality=90)
    return buf.getvalue()


def hrsc():
    with open(HRSC, "rb") as f:
        return f.read()
