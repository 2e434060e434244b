"""CPU checks of the training augmentation (rotate-yolov3_b200/augment.py, csrc/augment.cu): numpy restatements of
the kernels' arithmetic against cv2 and numpy live (INTER_LINEAR pre-resize tables, the fixed-point warp, the 8-bit
HSV conversions over every colour and every HSV triplet, the gamma table), and the host half of ``train_batch``
(draw replay, target rows) against the reference's own ``__getitem__`` / ``collate_fn`` (fixture)."""
import random

import numpy as np
import pytest

from augment_cases import (DRAW_KEYS_NONE, GEN, Recorder, all_colours, aug_module, augment_golden, batch_case,
                           bgr2hsv_np, f32, gamma_table_np, hsv2bgr_np, hsv_np, source, warp_np)
from letterbox_cases import resize_np

cv2 = pytest.importorskip("cv2")


# ---- restatements against cv2 / numpy live ----------------------------------------------------------------------

@pytest.mark.parametrize("src_hw", [(1080, 1920), (768, 1024), (1216, 912), (611, 613), (1000, 700), (1213, 1900)])
def test_pre_resize_tables_match_cv2_linear(src_hw):
    import rotate_yolov3_b200.preprocess as pp
    aug = aug_module()
    dst = aug.pre_resize_shape(src_hw, 608)
    img = source(sum(src_hw), *src_hw)
    want = cv2.resize(img, (dst[1], dst[0]), interpolation=cv2.INTER_LINEAR)
    orig = pp.resample_tables
    pp.resample_tables = pp.linear_resize_tables
    try:
        got = resize_np(img, dst)
    finally:
        pp.resample_tables = orig
    assert np.array_equal(got, want)


def test_exact_2x_linear_takes_the_area_path():
    import rotate_yolov3_b200.preprocess as pp
    assert pp.linear_resize_tables((1216, 912), (608, 456))[0] == pp.AREA_INT
    assert pp.linear_resize_tables((1215, 912), (607, 456))[0] == pp.LINEAR


def test_rotation_matrix_matches_cv2():
    aug = aug_module()
    rng = np.random.default_rng(3)
    for _ in range(500):
        a, s = float(rng.uniform(-180, 180)), float(rng.uniform(0.5, 1.5))
        c = (float(f32(rng.uniform(0, 700))), float(f32(rng.uniform(0, 700))))
        assert np.array_equal(aug.rotation_matrix(a, c, s), cv2.getRotationMatrix2D(center=c, angle=a, scale=s))


@pytest.mark.parametrize("deg,scale,hw", [(5.0, 0.1, (608, 608)), (50.0, 0.2, (608, 608)), (50.0, 0.2, (352, 608)),
                                          (30.0, 0.5, (97, 131))])
def test_warp_restatement_matches_cv2(deg, scale, hw):
    aug = aug_module()
    rng = random.Random(int(deg) + hw[0])
    img = source(hw[0] + hw[1], *hw)
    for _ in range(4):
        rec = (rng.uniform(-deg, deg), rng.uniform(1 - scale, 1 + scale), rng.uniform(-0.1, 0.1),
               rng.uniform(-0.1, 0.1))
        M = aug.affine_matrix(rec, hw)
        want = cv2.warpAffine(img, M[:2], dsize=(hw[1], hw[0]), flags=cv2.INTER_AREA, borderValue=(128, 128, 128))
        assert np.array_equal(warp_np(img, aug.invert_affine(M)), want)


@pytest.mark.parametrize("w", [4096, 4093, 37, 1])
def test_bgr2hsv_every_colour(w):
    img = all_colours()
    n = img.shape[0] // w * w
    img = img[:n].reshape(-1, w, 3)
    assert np.array_equal(bgr2hsv_np(img), cv2.cvtColor(img, cv2.COLOR_BGR2HSV))


@pytest.mark.parametrize("w", [256, 608, 255, 100, 33, 31, 1])
def test_hsv2bgr_every_triplet(w):
    hh, ss, vv = np.meshgrid(np.arange(180), np.arange(256), np.arange(256), indexing="ij")
    trip = np.stack([hh, ss, vv], -1).reshape(-1, 3).astype(np.uint8)
    trip = np.roll(trip, 7 * w, 0)                 # every triplet at several positions in a row
    n = trip.shape[0] // w * w
    img = trip[:n].reshape(-1, w, 3)
    assert np.array_equal(hsv2bgr_np(img), cv2.cvtColor(img, cv2.COLOR_HSV2BGR))


@pytest.mark.parametrize("a,b", [(1.37, 1.21), (0.61, 0.83), (1.5, 0.7), (0.999999999, 1.0)])
def test_hsv_transform_matches_reference_arithmetic(a, b):
    img = source(9, 64, 608)
    hsv = cv2.cvtColor(img, cv2.COLOR_BGR2HSV)
    S, V = hsv[:, :, 1].astype(np.float32), hsv[:, :, 2].astype(np.float32)
    S *= a
    V *= b
    hsv[:, :, 1] = S if a < 1 else S.clip(None, 255)
    hsv[:, :, 2] = V if b < 1 else V.clip(None, 255)
    want = img.copy()
    cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR, dst=want)
    assert np.array_equal(hsv_np(img, a, b), want)


def test_gamma_tables_every_value_and_maximum():
    rng = random.Random(5)
    gms = [0.8, 1.2, 1.0 - 1e-12] + [rng.uniform(0.8, 1.2) for _ in range(30)]
    v = np.arange(256)
    for gm in gms:
        for m in range(256):
            img = np.minimum(v, m).astype(np.uint8)
            with np.errstate(invalid="ignore"):
                want = np.uint8(np.power(img / float(np.max(img)), gm) * np.max(img)) if m else np.zeros(256, np.uint8)
            assert np.array_equal(gamma_table_np(m, gm)[img], want), (gm, m)


# ---- the host half against the reference (fixture) --------------------------------------------------------------

def test_draw_replay_matches_reference():
    aug = aug_module()
    g = augment_golden()
    for name in g["batches"]:
        seed, hyp, new_shape, mode, img_size, imgs, labs, k = batch_case(g, str(name))
        rec = Recorder(seed)
        for _ in imgs:
            aug.draw(hyp, rec)
        assert np.array_equal(np.array(rec.vals), g[k + "draws"]), name


def test_targets_match_collate_fn_rows():
    aug = aug_module()
    g = augment_golden()
    for name in g["batches"]:
        seed, hyp, new_shape, mode, img_size, imgs, labs, k = batch_case(g, str(name))
        rng = random.Random(seed)
        draws = [aug.draw(hyp, rng) for _ in imgs]
        _, tg = aug.batch_plan([im.shape[:2] for im in imgs], labs, draws, new_shape, mode, img_size)
        assert tg.dtype == np.float32
        assert np.array_equal(tg.view(np.int32), g[k + "targets"].view(np.int32)), name


def test_direct_transforms_match_reference():
    """random_affine, Gamma, HSV and the flips called directly, each forced on: the restated pixels"""
    aug = aug_module()
    g = augment_golden()
    for name in g["directs"]:
        k = "direct_%s_" % name
        img, want, d = g[k + "img"], g[k + "out"], g[k + "draws"]
        rec = dict(DRAW_KEYS_NONE)
        if str(name).startswith("affine"):
            rec["affine"] = tuple(d[:4])
            got = warp_np(img, aug.invert_affine(aug.affine_matrix(rec["affine"], img.shape[:2])))
        elif str(name).startswith("gamma"):
            m = int(img.max())
            got = gamma_table_np(m, d[1])[img]
        elif str(name).startswith("hsv"):
            a, b = d[1] * 0.5 + 1, d[2] * 0.3 + 1
            got = hsv_np(img, a, b)
        else:
            rec[str(name)] = True
            got = img[:, ::-1] if name == "hflip" else img[::-1]
        assert np.array_equal(got, want), name


def test_missing_hyp_key_raises_keyerror():
    aug = aug_module()
    hyp = {"degrees": 5.0, "translate": 0.1, "scale": 0.1, "shear": 0.0, "noise": 0.01, "gamma": 0.2, "blur": 1.3,
           "hsv_s": 0.5, "hsv_v": 0.3, "grayscale": 0.3}
    aug.draw(hyp, random.Random(0))
    for key in hyp:
        bad = {k: v for k, v in hyp.items() if k != key}
        with pytest.raises(KeyError):
            aug.draw(bad, random.Random(0))
        with pytest.raises(KeyError):
            aug.train_batch([np.zeros((8, 8, 3), np.uint8)], [np.zeros((0, 6), np.float32)], bad, new_shape=32)


def test_rect_img_size_sets_the_pre_resize():
    """a dataset img_size that is no multiple of 32: the pre-resize follows it, not the batch shape"""
    aug = aug_module()
    rec = dict(DRAW_KEYS_NONE)
    plan, _ = aug.batch_plan([(1080, 1920)], [np.zeros((0, 6), np.float32)], [rec], (352, 608), "rect", 600)
    assert plan[0][1] == (337, 600)
    plan, _ = aug.batch_plan([(1080, 1920)], [np.zeros((0, 6), np.float32)], [rec], (352, 608), "rect")
    assert plan[0][1] == (342, 608)
    for bad in (0, 600.0, True):
        with pytest.raises(ValueError):
            aug.train_batch([np.zeros((8, 8, 3), np.uint8)], [np.zeros((0, 6), np.float32)], GEN.HYP5,
                            new_shape=(32, 32), mode="rect", img_size=bad)
    with pytest.raises(ValueError):
        aug.train_batch([np.zeros((8, 8, 3), np.uint8)], [np.zeros((0, 6), np.float32)], GEN.HYP5, new_shape=32,
                        img_size=64)
