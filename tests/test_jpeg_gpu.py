"""The device JPEG decoder (rotate_yolov3_b200.decode_images) byte for byte against cv2.imread of the same file written
to a temporary directory: sizes from 1 x 1 to 1920 x 1080 and the reference's HRSC sample, every sampling cv2 writes
and grayscale, qualities 5 to 100 with and without optimised tables and with separate luma / chroma quality, restart
intervals 0, 1, 3 and 17, Exif orientations 1 to 8, chunks small enough that the HRSC sample spans thousands of them,
all mixed in one call; the host fallbacks; repeatability and side streams; letterbox and train_batch fed from it; and
corrupt streams ending as a status and the host decoder."""
import random

import cv2
import numpy as np
import pytest
import torch

from jpeg_cases import cmyk, encode, hrsc, matrix, no_sync_batch, picture

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
HYP = {"degrees": 50.0, "translate": 0.1, "scale": 0.2, "shear": 0.0, "noise": 0.01, "gamma": 0.2, "blur": 1.3,
       "hsv_s": 0.5, "hsv_v": 0.3, "grayscale": 0.3}


def _imread(tmp_path, blobs):
    out = []
    for i, b in enumerate(blobs):
        p = tmp_path / ("%d.jpg" % i)
        p.write_bytes(b)
        out.append(cv2.imread(str(p)))
    return out


def _all_cases():
    cases = matrix()
    cases.append(("hrsc", hrsc()))
    cases.append(("hd_420_q95", encode(picture(11, 1080, 1920), 95, "420")))
    cases.append(("hd_444_q95_rst17", encode(picture(12, 1080, 1920), 95, "444", restart=17)))
    return cases


@pytest.mark.parametrize("chunk", [128, 16])
def test_matrix_in_one_call_bitwise_equals_imread(tmp_path, chunk):
    from rotate_yolov3_b200 import decode_images
    cases = _all_cases()
    names, blobs = [c[0] for c in cases], [c[1] for c in cases]
    want = _imread(tmp_path, blobs)
    imgs, routes = decode_images(blobs, device=DEV, chunk_bytes=chunk)
    torch.cuda.synchronize()
    assert all(r == "device" for r in routes), [(n, r) for n, r in zip(names, routes) if r != "device"]
    for name, img, w in zip(names, imgs, want):
        assert img.is_cuda and img.dtype == torch.uint8 and tuple(img.shape) == w.shape, name
        got = img.cpu().numpy()
        nd = int((got != w).sum())
        assert nd == 0, "%s: %d of %d values differ from cv2.imread" % (name, nd, w.size)


def test_hrsc_in_thousands_of_chunks(tmp_path):
    from rotate_yolov3_b200 import decode_images
    blob = hrsc()
    want = _imread(tmp_path, [blob])[0]
    for chunk in (4, 33):
        imgs, routes = decode_images([np.frombuffer(blob, np.uint8)], chunk_bytes=chunk)
        assert routes == ["device"] and np.array_equal(imgs[0].cpu().numpy(), want), chunk


def test_host_fallbacks_equal_imread(tmp_path):
    from rotate_yolov3_b200 import decode_images
    img = picture(4, 57, 83)
    blobs = [encode(img, 90, "420", progressive=True), encode(img, 80, "422"), encode(img, 70, "444", progressive=True)]
    k = cmyk(img)
    if k is not None:
        blobs.append(k)
    want = _imread(tmp_path, blobs)
    imgs, routes = decode_images(blobs)
    assert routes[0] == "host: progressive" and routes[1] == "device" and routes[2] == "host: progressive"
    if k is not None:
        assert routes[3] == "host: 4 components"
    for i, (a, w) in enumerate(zip(imgs, want)):
        assert np.array_equal(a.cpu().numpy(), w), i


def test_repeatable_and_side_stream():
    from rotate_yolov3_b200 import decode_images
    blobs = [c[1] for c in _all_cases()[::7]] + [hrsc()]
    a, _ = decode_images(blobs)
    b, _ = decode_images(blobs)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        c, _ = decode_images(blobs)
    s.synchronize()
    for x, y, z in zip(a, b, c):
        assert torch.equal(x, y) and torch.equal(x, z)


def test_graph_replay_of_a_staged_batch():
    from rotate_yolov3_b200.decode import Batch
    blobs = [hrsc(), encode(picture(3, 200, 300), 90, "422", restart=5)]
    batch = Batch(blobs, DEV)
    batch.decode()
    want = [im.clone() for im in batch.finish()[0]]
    batch.out.zero_()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g):
            batch.decode()
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    for x, y in zip(batch.images, want):
        assert torch.equal(x, y)


def test_letterbox_and_train_batch_fed_from_decode(tmp_path):
    import rotate_yolov3_b200 as pkg
    blobs = [hrsc(), encode(picture(5, 480, 640), 90, "420"), encode(picture(6, 300, 200), 95, "444", restart=3)]
    host = _imread(tmp_path, blobs)
    dev, routes = pkg.decode_images(blobs)
    assert routes == ["device"] * 3
    x_dev, m_dev = pkg.letterbox(dev, 608)
    x_host, m_host = pkg.letterbox(host, 608)
    assert torch.equal(x_dev, x_host) and torch.equal(m_dev, m_host)
    labs = [np.array([[0, 0.5, 0.5, 0.2, 0.1, 0.3]], np.float32)] * 3
    t_host, tg_host, draws = pkg.train_batch(host, labs, HYP, new_shape=416, rng=random.Random(7))
    t_dev, tg_dev, _ = pkg.train_batch(dev, labs, HYP, new_shape=416, draws=draws)
    assert torch.equal(t_dev, t_host) and torch.equal(tg_dev, tg_host)


def test_corrupt_streams_end_on_the_host(tmp_path):
    """truncated streams and flipped entropy bytes (whose host-build counterparts run in test_jpeg_cpu.py): the device
    sets a status and the image comes from the host decoder, or it decodes to cv2's own image; a stream cv2 rejects
    raises"""
    from rotate_yolov3_b200 import decode_images
    r = np.random.default_rng(5)
    good = encode(picture(6, 96, 128), 90, "420")
    sos = good.index(b"\xff\xda") + 14
    blobs = [good[:len(good) - 30] + b"\xff\xd9", good[:sos + 40] + b"\xff\xd9"]
    while len(blobs) < 24:
        b = bytearray(good)
        p = int(r.integers(sos, len(good) - 2))
        b[p] ^= int(r.integers(1, 256))
        if b[p] != 0xFF and b[p - 1] != 0xFF:
            blobs.append(bytes(b))
    want = _imread(tmp_path, blobs)
    ok = [b for b, w in zip(blobs, want) if w is not None]
    imgs, routes = decode_images(ok)
    assert sum(r_.startswith("host: corrupt") for r_ in routes) >= 2
    for a, w in zip(imgs, [w for w in want if w is not None]):
        assert np.array_equal(a.cpu().numpy(), w)
    for b, w in zip(blobs, want):
        if w is None:
            with pytest.raises(ValueError):
                decode_images([b])


def test_chunk_that_never_synchronises_ends_on_the_host(tmp_path):
    """an 800 x 600 stream whose entropy-coded segment is all zero bytes, batched behind 256 small restart segments
    (its host-build counterpart runs in test_jpeg_cpu.py): the device reports that its chunks do not synchronise, the
    host decodes it, and the other image stays on the device"""
    from rotate_yolov3_b200 import decode_images
    blobs = no_sync_batch()
    want = _imread(tmp_path, blobs)
    imgs, routes = decode_images(blobs)
    assert routes[0] == "device" and routes[1].startswith("host: corrupt"), routes
    for a, w in zip(imgs, want):
        assert np.array_equal(a.cpu().numpy(), w)
