"""GPU checks of the training augmentation (rotate_yolov3_b200.train_batch): every fixture batch of the reference's
own ``__getitem__`` / ``collate_fn`` bit for bit in fp32 and fp16 with identical target rows, the transforms forced
on one at a time, the device HSV over every colour and the device gamma tables against the host restatements, mixed
and CUDA-resident batches, the launch count, and malformed input."""
import os
import random

import numpy as np
import pytest
import torch

from augment_cases import DRAW_KEYS_NONE, all_colours, batch_case, gamma_table_np, hsv_np
from builders import tensor_sha
from helpers import GOLDEN

pytestmark = pytest.mark.gpu
GOLD = os.path.join(GOLDEN, "augment_golden.npz")
DEV = torch.device("cuda", 0)
HYP = {"degrees": 50.0, "translate": 0.1, "scale": 0.2, "shear": 0.0, "noise": 0.01, "gamma": 0.2, "blur": 1.3,
       "hsv_s": 0.5, "hsv_v": 0.3, "grayscale": 0.3}


def _net(u8, dtype):
    x = np.ascontiguousarray(u8[:, :, ::-1].transpose(2, 0, 1), dtype=np.float32)
    x /= 255.0
    return torch.from_numpy(x if dtype == torch.float32 else x.astype(np.float16))


def _record(**kw):
    rec = dict(DRAW_KEYS_NONE)
    rec.update(kw)
    return rec


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_every_fixture_batch_bitwise(dtype):
    import rotate_yolov3_b200 as pkg
    g = np.load(GOLD)
    for name in g["batches"]:
        seed, hyp, new_shape, mode, img_size, imgs, labs, k = batch_case(g, str(name))
        x, tg, draws = pkg.train_batch(imgs, labs, hyp, new_shape=new_shape, mode=mode, rng=random.Random(seed),
                                       dtype=dtype, img_size=img_size)
        assert tensor_sha(x) == str(g[k + ("sha32" if dtype == torch.float32 else "sha16")]), name
        assert tg.is_cuda and tg.dtype == torch.float32
        assert np.array_equal(tg.cpu().numpy().view(np.int32), g[k + "targets"].view(np.int32)), name
        # the returned draws replay the batch
        x2, tg2, _ = pkg.train_batch(imgs, labs, hyp, new_shape=new_shape, mode=mode, draws=draws, dtype=dtype,
                                     img_size=img_size)
        assert torch.equal(x, x2) and torch.equal(tg, tg2)


def test_direct_transforms_bitwise():
    import rotate_yolov3_b200 as pkg
    g = np.load(GOLD)
    for name in g["directs"]:
        name = str(name)
        k = "direct_%s_" % name
        img, want, d = g[k + "img"], g[k + "out"], g[k + "draws"]
        if name.startswith("affine"):
            rec = _record(affine=tuple(float(v) for v in d[:4]))
        elif name.startswith("gamma"):
            rec = _record(gamma=float(d[1]))
        elif name.startswith("hsv"):
            rec = _record(hsv=(float(d[1]) * 0.5 + 1, float(d[2]) * 0.3 + 1))
        else:
            rec = _record(**{name: True})
        for dtype in (torch.float32, torch.float16):
            x, tg, _ = pkg.train_batch([img], [np.zeros((0, 6), np.float32)], HYP, new_shape=96, draws=[rec],
                                       dtype=dtype)
            assert torch.equal(x[0].cpu(), _net(want, dtype)), (name, dtype)
            assert tg.shape == (0, 7)


@pytest.mark.parametrize("factors", [(1.0, 1.0), (1.37, 0.71), (0.55, 1.29)])
def test_device_hsv_every_colour(factors):
    import rotate_yolov3_b200 as pkg
    img = all_colours().reshape(4096, 4096, 3)
    x, _, _ = pkg.train_batch([img], [np.zeros((0, 6), np.float32)], HYP, new_shape=4096,
                              draws=[_record(hsv=factors)])
    got = torch.round(x[0] * 255).to(torch.uint8).cpu().numpy()[::-1].transpose(1, 2, 0)
    assert np.array_equal(got, hsv_np(img, *factors))
    # rows whose width leaves a scalar tail (100 = 3 x 32 + 4)
    small = all_colours()[::1669][:10000].reshape(100, 100, 3)
    x, _, _ = pkg.train_batch([small], [np.zeros((0, 6), np.float32)], HYP, new_shape=100,
                              draws=[_record(hsv=factors)])
    got = torch.round(x[0] * 255).to(torch.uint8).cpu().numpy()[::-1].transpose(1, 2, 0)
    assert np.array_equal(got, hsv_np(small, *factors))


@pytest.mark.parametrize("flips", [dict(hflip=True), dict(vflip=True), dict(hflip=True, vflip=True)])
def test_device_hsv_with_flips_at_a_width_with_a_scalar_tail(flips):
    """HSV2BGR's vector/scalar path follows a pixel's column before the flips (100 = 3 x 32 + 4)"""
    import rotate_yolov3_b200 as pkg
    small = all_colours()[::1669][:10000].reshape(100, 100, 3)
    want = hsv_np(small, 1.37, 0.71)
    want = want[:, ::-1] if flips.get("hflip") else want
    want = want[::-1] if flips.get("vflip") else want
    x, _, _ = pkg.train_batch([small], [np.zeros((0, 6), np.float32)], HYP, new_shape=100,
                              draws=[_record(hsv=(1.37, 0.71), **flips)])
    assert torch.equal(x[0].cpu(), _net(np.ascontiguousarray(want), torch.float32))


def test_device_gamma_tables_every_value_and_maximum():
    import rotate_yolov3_b200 as pkg
    v = np.arange(256)
    imgs = [np.repeat(np.minimum(v, m).astype(np.uint8).reshape(16, 16, 1), 3, 2) for m in range(256)]
    rng = random.Random(11)
    gms = [0.8, 1.2, 1.0 - 1e-12] + [rng.uniform(0.8, 1.2) for _ in range(40)]
    for gm in gms:
        x, _, _ = pkg.train_batch(imgs, [np.zeros((0, 6), np.float32)] * 256, HYP, new_shape=16,
                                  draws=[_record(gamma=gm)] * 256)
        got = torch.round(x[:, 0] * 255).to(torch.uint8).cpu().numpy().reshape(256, 256)
        want = np.stack([gamma_table_np(m, gm)[np.minimum(v, m)] for m in range(256)])
        assert np.array_equal(got, want), gm


def test_mixed_batch_equals_single_calls_and_cuda_sources():
    import rotate_yolov3_b200 as pkg
    rng = np.random.default_rng(4)
    shapes = [(768, 1024), (1080, 1920), (300, 200), (608, 608), (900, 1300)]
    imgs = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in shapes]
    labs = [np.array([[0, 0.5, 0.5, 0.2, 0.1, 0.3]], np.float32)] * len(imgs)
    x, tg, draws = pkg.train_batch(imgs, labs, HYP, rng=random.Random(3))
    rows = []
    for b, (im, lab, rec) in enumerate(zip(imgs, labs, draws)):
        x1, t1, _ = pkg.train_batch([im], [lab], HYP, draws=[rec])
        assert torch.equal(x1[0], x[b]), b
        t1[:, 0] = b
        rows.append(t1)
    assert torch.equal(torch.cat(rows), tg)
    xc, tc, _ = pkg.train_batch([torch.from_numpy(im).to(DEV) for im in imgs], labs, HYP, draws=draws,
                                dtype=torch.float16)
    xh, th, _ = pkg.train_batch(imgs, labs, HYP, draws=draws, dtype=torch.float16)
    assert torch.equal(xc, xh) and torch.equal(tc, th)


def test_strided_cuda_sources_equal_host_arrays():
    """CUDA images whose pixels or channels are not packed (a CHW decode permuted to HWC, a column-subsampled view, a
    crop) give what the same pixels give as host arrays"""
    import rotate_yolov3_b200 as pkg
    rng = np.random.default_rng(8)
    base = rng.integers(0, 256, (700, 1300, 3), dtype=np.uint8)
    chw = torch.from_numpy(np.ascontiguousarray(base.transpose(2, 0, 1))).to(DEV)
    full = torch.from_numpy(base).to(DEV)
    views = [chw.permute(1, 2, 0), full[:, ::2], full[50:650, 100:1200], full[::3, ::2]]
    assert views[0].stride() == (1300, 1, 700 * 1300) and views[1].stride(1) == 6
    host = [np.ascontiguousarray(v.cpu().numpy()) for v in views]
    labs = [np.array([[0, 0.5, 0.5, 0.2, 0.1, 0.3]], np.float32)] * len(views)
    x, tg, draws = pkg.train_batch(host, labs, HYP, rng=random.Random(5))
    xc, tc, _ = pkg.train_batch(views, labs, HYP, draws=draws)
    assert torch.equal(x, xc) and torch.equal(tg, tc)


def test_launches_per_batch():
    import rotate_yolov3_b200 as pkg
    lib = pkg._lib.lib
    big = np.zeros((1080, 1920, 3), np.uint8)
    small = np.zeros((300, 400, 3), np.uint8)
    lab = [np.zeros((0, 6), np.float32)]
    for imgs, rec, want in (([big], _record(affine=(3.0, 1.0, 0.0, 0.0)), 4),   # pre-resize, letterbox, warp, finish
                            ([small], _record(gamma=1.1), 3),                      # letterbox, max, finish
                            ([small], _record(hsv=(1.1, 0.9), hflip=True), 2)):    # letterbox, finish
        torch.cuda.synchronize()
        n0 = lib.ryolo_launch_count()
        pkg.train_batch(imgs, lab, HYP, draws=[rec])
        torch.cuda.synchronize()
        assert lib.ryolo_launch_count() - n0 == want


def test_malformed_input_raises_before_any_launch():
    import rotate_yolov3_b200 as pkg
    lib = pkg._lib.lib
    ok = np.zeros((20, 30, 3), np.uint8)
    lab = [np.zeros((0, 6), np.float32)]
    bad = [
        dict(images=[], labels=[]),
        dict(images=[ok.astype(np.float32)], labels=lab),
        dict(images=[ok[:, :, :2]], labels=lab),
        dict(images=[ok], labels=[]),
        dict(images=[ok], labels=[np.zeros((2, 5), np.float32)]),
        dict(images=[ok], labels=lab, new_shape=(32, 32)),
        dict(images=[ok], labels=lab, mode="rect", new_shape=32),
        dict(images=[ok], labels=lab, dtype=torch.float64),
        dict(images=[ok], labels=lab, draws=[{"affine": None}]),
        dict(images=[ok], labels=lab, draws=[_record(hsv=(-0.5, 1.0))]),
        dict(images=[ok], labels=lab, draws=[]),
        dict(images=[ok], labels=lab, out=torch.empty(1, 3, 16, 16, device=DEV)),
        dict(images=[ok], labels=lab, new_shape=(20, 32), mode="rect"),
    ]
    torch.cuda.synchronize()
    n0 = lib.ryolo_launch_count()
    for kw in bad:
        kw = dict(kw)
        kw.setdefault("new_shape", 32)
        with pytest.raises(ValueError):
            pkg.train_batch(kw.pop("images"), kw.pop("labels"), HYP, **kw)
    torch.cuda.synchronize()
    assert lib.ryolo_launch_count() == n0
