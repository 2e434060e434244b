"""CPU checks of multi-scale detection: the sizes detect.py --multi-scale draws, the refusals of detect_multiscale, and
the argument checks of ryolo_merge_scales (status codes, no GPU needed)."""
import ctypes

import numpy as np
import pytest

import helpers


def reference_sizes(img_size):
    """detect.py:54-59 as the reference writes it, on numpy's global RNG"""
    size_num = 2
    img_sz_min = round(img_size / 32 / 1.5) + 1
    img_sz_max = round(img_size / 32 * 1.3) - 1
    img_sizes = np.random.choice(range(img_sz_min * 32, (img_sz_max + 1) * 32, 32), size_num, False)
    return [int(x) for x in img_sizes]


@pytest.mark.parametrize("img_size", [416, 512, 608])
def test_multiscale_sizes_match_reference_draws(img_size):
    from rotate_yolov3_b200 import multiscale_sizes
    seen = set()
    for seed in range(40):
        np.random.seed(seed)
        want = reference_sizes(img_size)
        np.random.seed(seed)
        got = multiscale_sizes(img_size)
        assert got == want and all(type(v) is int for v in got), (seed, got, want)
        assert multiscale_sizes(img_size, np.random.RandomState(seed)) == want
        seen.add(tuple(got))
    assert len(seen) > 5
    lo, hi = min(min(s) for s in seen), max(max(s) for s in seen)
    assert lo % 32 == 0 and hi % 32 == 0 and lo >= img_size / 1.5 and hi <= img_size * 1.3


def _model():
    import rotate_yolov3_b200 as pkg
    return pkg.Darknet(helpers.mini_cfg(64, 64), {"context_factor": 1.0}, arc="default")


def test_detect_multiscale_refusals():
    from rotate_yolov3_b200 import detect_multiscale
    img = [np.zeros((48, 64, 3), np.uint8)]
    m = _model()
    m.train()
    with pytest.raises(ValueError, match="eval"):
        detect_multiscale(m, img, [64], 0.5, 0.5, 100)
    m.eval()
    with pytest.raises(ValueError, match="empty"):
        detect_multiscale(m, img, [], 0.5, 0.5, 100)
    for sizes in ([64, 80], [100], [0], [-32]):
        with pytest.raises(ValueError, match="multiple of 32"):
            detect_multiscale(m, img, sizes, 0.5, 0.5, 100)
    for conf in (-0.1, float("nan")):
        with pytest.raises(ValueError, match="conf_thres"):
            detect_multiscale(m, img, [64], conf, 0.5, 100)
    with pytest.raises(ValueError, match="at most 16"):
        detect_multiscale(m, img, [64] * 17, 0.5, 0.5, 100)
    with pytest.raises(ValueError, match="cap"):
        detect_multiscale(m, img, [64], 0.5, 0.5, 0)


def test_merge_scales_checks_its_arguments():
    import rotate_yolov3_b200 as pkg
    lib = pkg._lib.lib
    buf = ctypes.c_void_p(256)     # never dereferenced: every call below fails its argument checks first
    arr = lambda n, p=buf: (ctypes.c_void_p * max(n, 1))(*([p] * max(n, 1)))
    ok = (arr(2), arr(2), arr(2))
    merge = lib.ryolo_merge_scales
    assert merge(*ok, 0, 4, 100, buf, buf, None) == -1                    # no scale
    assert b"bad argument" in lib.ryolo_last_error()
    assert merge(arr(17), arr(17), arr(17), 17, 4, 100, buf, buf, None) == -1      # more than RYOLO_MERGE_MAX_SCALES
    assert merge(*ok, 2, 0, 100, buf, buf, None) == -1                    # no image
    assert merge(*ok, 2, 65536, 100, buf, buf, None) == -1                # more images than grid rows
    assert merge(*ok, 2, 4, 0, buf, buf, None) == -1                      # cap 0
    assert merge(*ok, 2, 4, 100, None, buf, None) == -1                   # no table
    assert merge(*ok, 2, 4, 100, buf, None, None) == -1                   # no output
    assert merge(None, ok[1], ok[2], 2, 4, 100, buf, buf, None) == -1     # no pointer array
    holed = (ctypes.c_void_p * 2)(buf, None)
    assert merge(ok[0], holed, ok[2], 2, 4, 100, buf, buf, None) == -1    # a null result pointer
    assert b"bad argument" in lib.ryolo_last_error()
    assert pkg._lib.MERGE_MAX_SCALES == 16
