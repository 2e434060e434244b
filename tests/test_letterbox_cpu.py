"""CPU checks of the letterbox step (rotate-yolov3_b200/preprocess.py): the host geometry against the reference's
letterbox, the arithmetic the kernel assumes for numpy's /255, and a numpy restatement of the kernel, built from the
same tables, against the reference's network input (fixture digests) and against cv2.resize live."""
import hashlib
import os

import numpy as np
import pytest

from helpers import GOLDEN
from letterbox_cases import letterbox_case, net_input, resize_np

GOLD = os.path.join(GOLDEN, "letterbox_golden.npz")


def _pp():
    import rotate_yolov3_b200.preprocess as pp
    return pp


def letterbox_np(img, new_shape, mode):
    pp = _pp()
    (nh, nw), (top, bottom, left, right), _ = pp.geometry(img.shape[:2], new_shape, mode)
    lb = np.full((top + nh + bottom, left + nw + right, 3), 128, np.uint8)
    lb[top:top + nh, left:left + nw] = resize_np(img, (nh, nw))
    return lb


def test_geometry_sweep_matches_reference():
    pp = _pp()
    geo = np.load(GOLD)["geo"]
    assert len(geo) >= 200
    for h, w, nsh, nsw, rect, nh, nw, top, bottom, left, right, rw, rh, dw, dh in geo:
        ns = (int(nsh), int(nsw)) if rect else int(nsh)
        (gh, gw), borders, meta = pp.geometry((int(h), int(w)), ns, "rect" if rect else "square")
        assert (gh, gw) == (nh, nw) and borders == (top, bottom, left, right), (h, w, ns)
        assert meta == (rw, rh, dw, dh), (h, w, ns)


def test_numpy_division_by_255_is_float32_ieee():
    """numpy's float32 `/= 255.0` is the correctly rounded float32 quotient, and float16 `/=` is that float32 quotient
    rounded once to half: the two things the kernel computes (IEEE __fdiv_rn, then __float2half_rn)."""
    v = np.arange(256)
    a32 = v.astype(np.float32)
    a32 /= 255.0
    exact = np.array([np.float32(np.float64(i) / 255.0) for i in v], np.float32)   # float64 quotient is exact enough
    assert (a32.view(np.uint32) == exact.view(np.uint32)).all()
    a16 = v.astype(np.float16)
    a16 /= 255.0
    assert (a16.view(np.uint16) == exact.astype(np.float16).view(np.uint16)).all()
    assert (a32 != v.astype(np.float32) * np.float32(1 / 255.0)).any()   # a reciprocal multiply would differ


def test_restatement_matches_reference_input():
    """the numpy restatement of the kernel's arithmetic gives the reference's network input bytes for every case"""
    g = np.load(GOLD)
    for name in g["cases"]:
        img, new_shape, mode, k = letterbox_case(g, str(name))
        lb = letterbox_np(img, new_shape, mode)
        if k + "lb" in g:
            assert (lb == g[k + "lb"]).all(), name
        assert hashlib.sha256(net_input(lb, np.float32).tobytes()).hexdigest() == str(g[k + "sha32"]), name
        assert hashlib.sha256(net_input(lb, np.float16).tobytes()).hexdigest() == str(g[k + "sha16"]), name


@pytest.mark.parametrize("src_hw,dst_hw", [((300, 401), (147, 197)), ((912, 1216), (456, 608)), ((300, 300), (100, 100)),
                                           ((9, 64), (3, 16)), ((300, 400), (456, 608)), ((50, 30), (300, 180)),
                                           ((300, 30), (200, 40)), ((400, 1), (608, 2)), ((101, 37), (53, 19)),
                                           ((66, 98), (33, 49))])
def test_restatement_matches_cv2_live(src_hw, dst_hw):
    cv2 = pytest.importorskip("cv2")
    img = np.random.default_rng(sum(src_hw) + sum(dst_hw)).integers(0, 256, src_hw + (3,), dtype=np.uint8)
    ref = cv2.resize(img, dst_hw[::-1], interpolation=cv2.INTER_AREA)
    assert (resize_np(img, dst_hw) == ref).all()


def test_resample_kind_follows_cv2_branches():
    pp = _pp()
    assert pp.resample_tables((912, 1216), (456, 608))[:2] == (pp.AREA_INT, (2, 2))
    assert pp.resample_tables((1368, 1824), (456, 608))[:2] == (pp.AREA_INT, (3, 3))
    assert pp.resample_tables((3, 32), (1, 8))[:2] == (pp.AREA_INT, (4, 3))
    assert pp.resample_tables((768, 1024), (456, 608))[0] == pp.AREA
    assert pp.resample_tables((300, 400), (456, 608))[0] == pp.LINEAR
    assert pp.resample_tables((1, 470), (1, 608))[0] == pp.LINEAR          # one axis at scale 1, one upscaling
    assert pp.resample_tables((456, 608), (456, 608))[0] == pp.AREA         # no resize: unit taps
