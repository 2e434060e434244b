"""The JPEG decoder without a GPU: the marker parser (rotate_yolov3_b200.decode) on cv2-encoded streams, and the host
build of the device arithmetic (tests/jpeg_host.py) on the staged batch the parser builds, byte for byte against
cv2.imdecode, which decodes as cv2.imread does."""
import cv2
import numpy as np
import pytest

from jpeg_cases import cmyk, encode, hrsc, matrix, no_sync_batch, picture, with_orientation
from jpeg_host import check_equal, cv2_decode, host_decode, make_harness

@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return make_harness(tmp_path_factory)


# ---------------------------------------------------------------------------------------------------------------------
# parser
# ---------------------------------------------------------------------------------------------------------------------

def test_parser_reads_frame_tables_and_restarts():
    from rotate_yolov3_b200.decode import parse
    img = picture(1, 45, 70)
    for s, hv in (("444", (1, 1)), ("422", (2, 1)), ("420", (2, 2)), ("440", (1, 2)), ("411", (4, 1))):
        for rst in (0, 2):
            hd = parse(np.frombuffer(encode(img, 80, s, restart=rst), np.uint8))
            assert (hd.height, hd.width, hd.ncomp) == (45, 70, 3)
            assert (hd.h[0], hd.v[0]) == hv and hd.h[1:] == [1, 1] and hd.v[1:] == [1, 1]
            assert (hd.hmax, hd.vmax) == hv and hd.bpm == hv[0] * hv[1] + 2
            assert hd.mcux == -(-70 // (8 * hv[0])) and hd.mcuy == -(-45 // (8 * hv[1]))
            assert hd.restart == rst and hd.orient == 1 and hd.out_hw == (45, 70)
            starts, ends, first, nmcu = hd.segments
            total = hd.mcux * hd.mcuy
            assert len(starts) == (1 if rst == 0 else -(-total // rst)) and nmcu.sum() == total
            assert np.all(starts[1:] == ends[:-1] + 2) and np.all(ends > starts)
            assert hd.quant[0][0] != 0 and hd.quant[1].shape == (64,)
    g = parse(np.frombuffer(encode(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY), 80), np.uint8))
    assert g.ncomp == 1 and g.bpm == 1 and g.color == 2 and (g.mcux, g.mcuy) == (9, 6)


def test_parser_tables_match_libjpeg_derivation():
    """the 9-bit lookahead and maxcode / valoff agree with a direct canonical-code walk"""
    from rotate_yolov3_b200.decode import derived_table
    for opt in (False, True):
        from rotate_yolov3_b200.decode import parse
        hd = parse(np.frombuffer(encode(picture(2, 64, 64), 90, "420", optimize=opt), np.uint8))
        for t in hd.dc + hd.ac:
            codes = []
            code = 0
            for ln in range(1, 17):
                n = t["maxcode"][ln] - (code if t["maxcode"][ln] >= 0 else 0) + 1 if t["maxcode"][ln] >= 0 else 0
                for k in range(n):
                    codes.append((ln, code + k))
                code = (code + n) << 1
            for idx, (ln, c) in enumerate(codes):
                assert t["vals"][c + t["valoff"][ln]] == t["vals"][idx]
                if ln <= 9:
                    e = int(t["lut"][c << (9 - ln)])
                    assert e >> 8 == ln and (e & 255) == t["vals"][idx]
    with pytest.raises(Exception):
        derived_table(bytes([3] + [0] * 15), bytes([0, 1, 2]), True)   # three 1-bit codes overflow


def test_exif_orientation_and_shapes():
    from rotate_yolov3_b200.decode import parse
    base = encode(picture(3, 20, 31), 85, "420")
    for o in range(1, 9):
        for be in (False, True):
            hd = parse(np.frombuffer(with_orientation(base, o, be), np.uint8))
            assert hd.orient == o and hd.out_hw == ((31, 20) if o >= 5 else (20, 31))
            assert cv2_decode(with_orientation(base, o, be)).shape[:2] == hd.out_hw


def test_routes_of_unsupported_streams():
    from rotate_yolov3_b200.decode import Layout
    img = picture(4, 40, 50)
    prog = encode(img, 90, "420", progressive=True)
    gray = encode(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY), 90)
    blobs = [prog, encode(img, 90, "420", optimize=True), gray]
    k = cmyk(img)
    if k is not None:
        blobs.append(k)
    lay = Layout(blobs)
    assert lay.routes[0] == "host: progressive"
    assert lay.routes[1] == "device" and lay.routes[2] == "device"
    if k is not None:
        assert lay.routes[3] == "host: 4 components"
    for i, r in enumerate(lay.routes):
        if r != "device":
            assert np.array_equal(lay.host[i], cv2_decode(blobs[i]))
    with pytest.raises(ValueError):
        Layout([b"not a jpeg at all"])


# ---------------------------------------------------------------------------------------------------------------------
# the host build of the device arithmetic against cv2
# ---------------------------------------------------------------------------------------------------------------------

def test_host_build_matrix_bitwise_equals_cv2(harness):
    cases = matrix()
    names, blobs = [c[0] for c in cases], [c[1] for c in cases]
    imgs, status, routes = host_decode(harness, blobs)
    assert all(r == "device" for r in routes), [(n, r) for n, r in zip(names, routes) if r != "device"]
    check_equal(imgs, status, blobs, names)


@pytest.mark.parametrize("chunk", [1, 7, 16, 4096])
def test_host_build_chunk_sizes(harness, chunk):
    """tiny chunks force the synchronisation on every image, one huge chunk decodes each segment in one piece"""
    cases = [c for c in matrix() if c[0].startswith(("121x163", "33x47", "orient"))]
    names, blobs = [c[0] for c in cases], [c[1] for c in cases]
    imgs, status, _ = host_decode(harness, blobs, chunk)
    check_equal(imgs, status, blobs, names)


def test_host_build_hrsc_and_hd(harness):
    """the reference's HRSC sample (1167 x 821, 4:2:0, no restarts) in 16-byte chunks (thousands of them), and a
    1920 x 1080 q95 4:4:4 frame with restart interval 17"""
    blobs = [hrsc(), encode(picture(11, 1080, 1920), 95, "444", restart=17)]
    imgs, status, _ = host_decode(harness, blobs, 16)
    check_equal(imgs, status, blobs, ["hrsc", "hd"])


def test_host_build_corrupt_streams_report_status(harness):
    """truncated streams and flipped entropy bytes end as a status (then the host decoder, whose answer is cv2's), or
    as cv2's own image, never as a different image; a stream cv2 rejects is rejected"""
    from rotate_yolov3_b200.decode import Layout
    r = np.random.default_rng(5)
    good = encode(picture(6, 96, 128), 90, "420")
    sos = good.index(b"\xff\xda") + 14
    blobs = [good[:len(good) // 2], good[:-2], good[:len(good) - 30] + b"\xff\xd9", good[:sos + 40] + b"\xff\xd9"]
    while len(blobs) < 24:
        b = bytearray(good)
        p = int(r.integers(sos, len(good) - 2))
        b[p] ^= int(r.integers(1, 256))
        if b[p] != 0xFF and b[p - 1] != 0xFF:
            blobs.append(bytes(b))
    flagged = 0
    for i, blob in enumerate(blobs):
        want = cv2_decode(blob)
        if want is None:
            with pytest.raises(ValueError):
                Layout([blob])
            continue
        imgs, status, routes = host_decode(harness, [blob])
        if routes[0] != "device" or status[0]:
            flagged += 1
            continue
        assert np.array_equal(imgs[0], want), "blob %d decoded differently from cv2" % i
    assert flagged >= 2                                    # the two truncations before EOI at least


def test_host_build_chunk_that_never_synchronises(harness):
    """a 40 KB segment of zero bytes (which cv2 still decodes) keeps its chunks from synchronising: the image gets
    RYOLO_JPEG_ST_NO_SYNC and no chunk of the broken chain writes or reads outside its segment, with many small
    restart segments before it in the batch (so chunk indices run far ahead of the segment's byte offsets)"""
    blobs = no_sync_batch()
    assert cv2_decode(blobs[1]) is not None
    imgs, status, routes = host_decode(harness, blobs)
    assert routes == ["device", "device"]
    assert status[0] == 0 and status[1] & 4, status
    assert np.array_equal(imgs[0], cv2_decode(blobs[0]))
