"""The host build of the device JPEG decoder (tests/jpeg_host.py) against cv2.imdecode, byte for byte, on streams cv2
never writes (tests/jpeg_syntax_cases.py): dequantised coefficients from 2^9 to 2^20 and rewritten quantisation
tables, DC sums past int16, Huffman tables with every code length, 16-bit codes or one symbol, EOB / ZRL edge cases,
byte stuffing on chunk boundaries, every colour rule and samplings cv2 cannot write.  Every stream decodes to cv2's
bytes on the device path or is handed to the host (whose answer is cv2's); the range cases must be handed over with
RYOLO_JPEG_ST_RANGE.  Bug insertions into a copy of the sources must each fail one of these checks."""
import inspect

import numpy as np
import pytest

import jpeg_syntax_cases as cases
import jpeg_writer as jw
from jpeg_cases import encode, hrsc, matrix, picture, SAMPLINGS
from jpeg_host import cv2_decode, host_decode, make_harness

ST_RANGE = 8


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return make_harness(tmp_path_factory)


@pytest.fixture(scope="module")
def syntax_cases():
    return cases.all_cases()


def verify(harness, items, chunk_bytes=128):
    """decode items [(name, blob, expect)] in one batch with the host build; returns the list of failures"""
    from rotate_yolov3_b200.decode import Layout
    bad = []
    ok = []
    for name, blob, expect in items:
        if cv2_decode(blob) is None:
            with pytest.raises(ValueError):
                Layout([blob])
            bad += [] if expect == "reject" else [(name, "cv2 rejects it")]
        else:
            ok.append((name, blob, expect))
    imgs, status, routes = host_decode(harness, [b for _, b, _ in ok], chunk_bytes)
    dev = 0
    for i, (name, blob, expect) in enumerate(ok):
        on_dev = routes[i] == "device"
        st = int(status[dev]) if on_dev else 0
        dev += on_dev
        kept = on_dev and st == 0
        if expect == "device" and not kept:
            bad.append((name, "not kept on the device", routes[i], st))
        if expect == "range" and not (on_dev and st & ST_RANGE):
            bad.append((name, "not handed over with RYOLO_JPEG_ST_RANGE", routes[i], st))
        if expect == "host" and kept:
            bad.append((name, "kept on the device"))
        if kept:
            want = cv2_decode(blob)
            nd = int((imgs[i] != want).sum()) if imgs[i].shape == want.shape else -1
            if nd:
                bad.append((name, "%d values differ from cv2" % nd))
    return bad


def test_writer_reproduces_cv2_streams():
    """the writer, fed the blocks and tables read back from cv2's own streams, writes streams cv2 decodes to the same
    image, for every sampling, with and without restarts, with cv2's tables and with tables from frequencies"""
    for s in SAMPLINGS:
        for rst in (0, 3):
            blob = encode(picture(1, 37, 53), 85, s, restart=rst, optimize=rst == 3)
            w, h, comps, blocks, quant, dc, ac, ri = jw.read_cv2_stream(blob)
            want = cv2_decode(blob)
            assert np.array_equal(cv2_decode(jw.write(w, h, comps, blocks, quant, dc, ac, restart=ri)), want), s
            c2, dc2, ac2 = jw.optimal_tables(w, h, comps, blocks, ri)
            assert np.array_equal(cv2_decode(jw.write(w, h, c2, blocks, quant, dc2, ac2, restart=ri)), want), s


def test_frequency_tables_limit_code_lengths():
    """Annex K.2 tables: lengths up to 16 even for Fibonacci frequencies, whose Huffman code wants 24 bits, and a
    prefix code (Kraft sum below 1, the all-ones code unused)"""
    fib = [1, 1]
    while len(fib) < 25:
        fib.append(fib[-1] + fib[-2])
    for freq, n in ((np.array(fib + [0] * 231), 25), (np.ones(256), 256), (np.arange(1, 257), 256)):
        counts, syms = jw.huff_from_freqs(freq)
        assert len(syms) == n and sum(counts) == n
        assert sum(c * 2.0 ** -(i + 1) for i, c in enumerate(counts)) < 1


def test_reproducer_quant_tables_rewritten(harness):
    """a cv2 q100 4:4:4 40 x 56 stream with only its DQT rewritten: every quantisation value 8 ... 255 (8-bit) and 1000,
    32767 (16-bit, SOF1) puts outputs outside [-512, 511]; the device hands every such image to the host"""
    items = cases.qtable_cases()
    assert not verify(harness, items)
    _, status, _ = host_decode(harness, [b for _, b, _ in items])
    assert all(st & ST_RANGE for (n, _, e), st in zip(items, status) if e == "range")


def test_syntax_cases_equal_cv2_or_go_to_host(harness, syntax_cases):
    bad = verify(harness, syntax_cases)
    assert not bad, bad


@pytest.mark.parametrize("chunk", [1, 2, 3, 7, 16, 1 << 20])
def test_syntax_cases_at_chunk_sizes(harness, syntax_cases, chunk):
    """stuffed bytes on chunk boundaries and every chunk size down to one byte"""
    items = [c for c in syntax_cases if c[0].startswith(("stuffing", "huff", "zrl", "order", "sampling_mixed"))]
    bad = verify(harness, items, chunk)
    assert not bad, bad


def test_colour_rules_follow_libjpeg(syntax_cases):
    from rotate_yolov3_b200.decode import parse
    for name, blob, _ in syntax_cases:
        if name.startswith("colour_"):
            assert parse(np.frombuffer(blob, np.uint8)).color == cases.expected_color(name), name


def test_range_sweep_fires_where_it_must(harness, syntax_cases):
    """the magnitude sweep: no block with dequantised magnitudes up to 2^11 alone is flagged, every frame from 2^13 up
    is; the report gives where the predicate starts to fire"""
    sweep = [c for c in syntax_cases if c[0].startswith("mag_single")]
    _, status, _ = host_decode(harness, [b for _, b, _ in sweep])
    fired = {n: bool(s & ST_RANGE) for (n, _, _), s in zip(sweep, status)}
    print("range status over the single-coefficient sweep:", fired)
    assert not any(fired["mag_single_2^%d" % e] for e in (9, 10, 11))
    assert all(fired["mag_single_2^%d" % e] for e in range(13, 21))


def test_smallest_magnitude_that_fires(harness):
    """one coefficient alone in a block, at each zigzag position: the smallest dequantised magnitude at which the
    predicate fires lies between 2 000 and 4 100 (the DC alone: 4 093, through the output bound (b))"""
    lo = []
    for k in range(64):
        a, b = 1, 1 << 13
        while b - a > 1:
            m = (a + b) // 2
            blk = np.zeros((1, 1, 64), np.int64)
            blk[0, 0, k] = m
            blob = cases._write_opt(8, 8, [{"id": 1, "h": 1, "v": 1, "tq": 0, "td": 0, "ta": 0}], [blk],
                                    {0: [1] * 64})
            _, st, _ = host_decode(harness, [blob])
            a, b = (a, m) if st[0] & ST_RANGE else (m, b)
        lo.append(b)
    print("smallest dequantised magnitude that fires, per zigzag position:", lo)
    assert 2000 < min(lo) and max(lo) <= 4100, lo


def _pass1_matrix():
    """M[n][u]: pass 1 of csrc/jpeg.cuh's idct_islow before its rounding, as an integer matrix (the butterflies of one
    column applied to unit impulses)"""
    m = np.zeros((8, 8), np.int64)
    for u in range(8):
        f = [0] * 8
        f[u] = 1
        z2, z3 = f[2], f[6]
        z1 = (z2 + z3) * 4433
        t2, t3 = z1 + z3 * -15137, z1 + z2 * 6270
        t0, t1 = (f[0] + f[4]) << 13, (f[0] - f[4]) << 13
        t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
        t0, t1, t2, t3 = f[7], f[5], f[3], f[1]
        z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
        z5 = (z3 + z4) * 9633
        t0, t1, t2, t3 = t0 * 2446, t1 * 16819, t2 * 25172, t3 * 12299
        z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069 + z5, z4 * -3196 + z5
        t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
        m[:, u] = [t10 + t3, t11 + t2, t12 + t1, t13 + t0, t13 - t0, t12 - t1, t11 - t2, t10 - t3]
    return m


def test_pass1_gains_behind_the_predicate():
    """the bound the predicate's soundness argument (csrc/jpeg.cuh) rests on: |M[n][0]| = 2^13, |M[n][u]| <= 11387
    (1.39 * 2^13), and 2 * 1.39 <= 3; with it the largest pass-1 value under the column limit is 16385"""
    m = np.abs(_pass1_matrix())
    assert np.all(m[:, 0] == 1 << 13)
    assert m[:, 1:].max() <= 11387, m[:, 1:].max()
    assert 2 * 11387 <= 3 * (1 << 13)
    worst = (4096 * (1 << 13) + (1 << 10)) >> 11
    assert worst + 1 <= 16385 < 1 << 15


STATS = [("jpeg.cuh", "constexpr int kIdctColumnLimit = 8192;",
          "constexpr int kIdctColumnLimit = 8192;\n}}\n#include <stdio.h>\n#define RJ_STATS 1\nnamespace ryolo {\nnamespace jpeg {\nstatic long long rj_col = 0, rj_out = 0, "
          "rj_near = 0, rj_blocks = 0;\nstatic void rj_stats_print() { printf(\"%lld %lld %lld %lld\\n\", rj_col, "
          "rj_out, rj_near, rj_blocks); }"),
         ("jpeg.cuh", "  return v < -128 ? 0 : (v > 127 ? 255 : v + 128);",
          "  if ((v < 0 ? -v : v) > rj_out) rj_out = v < 0 ? -v : v;\n  return v < -128 ? 0 : (v > 127 ? 255 : v + 128);"),
         ("jpeg.cuh", "    bad |= col > kIdctColumnLimit;",
          "    bad |= col > kIdctColumnLimit;\n    if (col > rj_col) rj_col = col;\n    if (c == 0) rj_blocks++;\n"
          "    if (col > kIdctColumnLimit / 2) rj_near++;")]


def test_natural_images_keep_a_margin(tmp_path_factory):
    """the whole matrix, HRSC, a 1920 x 1080 frame and q 1 ... 100 at every sampling stay on the device; reports the
    largest column sum of (a) against its 8192 limit, the largest |output| of (b) against 511, and the number of
    block columns past half the limit"""
    h = make_harness(tmp_path_factory, "jpeg_stats", STATS)
    blobs = [b for _, b in matrix()] + [hrsc(), encode(picture(11, 1080, 1920), 100, "444")]
    img = picture(2, 67, 91)
    for s in SAMPLINGS:
        for q in (1, 5, 10, 25, 50, 75, 90, 95, 100):
            blobs.append(encode(img, q, s))
    _, status, routes = host_decode(h, blobs)
    col, out, near, nblk = (int(x) for x in host_decode.stdout.split())
    print("natural images: %d blocks, largest column sum %d of 8192, largest |output| %d of 511, %d block columns "
          "past 4096" % (nblk, col, out, near))
    assert all(r == "device" for r in routes) and not status.any()
    assert col <= 8192 // 2 and out <= 400


# ---------------------------------------------------------------------------------------------------------------------
# bug insertions: each, put into a copy of the sources, must fail a check above
# ---------------------------------------------------------------------------------------------------------------------

OLD_OUT = """  bad |= (unsigned)(v - kIdctOutMin) > (unsigned)(kIdctOutMax - kIdctOutMin);
  return v < -128 ? 0 : (v > 127 ? 255 : v + 128);"""
INSERTIONS = {
    # the parent's IDCT output: the 10-bit wrap of the range-limit table, nothing flagged
    "wrap_range_limit": [("jpeg.cuh", OLD_OUT, "  const int idx = v & 1023;\n  const int w = (idx < 512 ? "
                          "idx : idx - 1024) + 128;\n  return w < 0 ? 0 : (w > 255 ? 255 : w);"),
                         ("jpeg.cuh", "  return bad ? RYOLO_JPEG_ST_RANGE : 0;", "  return 0;")],
    "predicate_disabled": [("jpeg.cuh", "  return bad ? RYOLO_JPEG_ST_RANGE : 0;", "  return 0;")],
    "zrl_past_64": [("jpeg.cuh", "      if (s.z + 16 > 64) {", "      if (s.z + 16 > 80) {")],
}


@pytest.mark.parametrize("name", sorted(INSERTIONS))
def test_bug_insertion_fails(tmp_path_factory, syntax_cases, name):
    h = make_harness(tmp_path_factory, "jpeg_bug_" + name, INSERTIONS[name])
    assert verify(h, syntax_cases), name


def test_bug_insertion_rgb_ids_dropped(harness, syntax_cases, monkeypatch):
    """the colour rule for component ids 'R','G','B' dropped from the parser"""
    import rotate_yolov3_b200.decode as dec
    src = inspect.getsource(dec._frame).replace("ids == [82, 71, 66]", "False")
    assert "False" in src
    ns = dict(dec.__dict__)
    exec(src, ns)
    monkeypatch.setattr(dec, "_frame", ns["_frame"])
    colour = [c for c in syntax_cases if c[0].startswith("colour_")]
    assert verify(harness, colour)
