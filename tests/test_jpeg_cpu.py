"""The JPEG decoder without a GPU: the marker parser (rotate_yolov3_b200.decode) on cv2-encoded streams, and a host
build of the device arithmetic (csrc/jpeg.cuh, compiled with g++) running the device's passes serially -- chunk pass
A, pass B, the chain resolution, the writers, the DC prefix, the IDCT and the pixel store -- on the staged batch the
parser builds, byte for byte against cv2.imdecode, which decodes as cv2.imread does."""
import os
import shutil
import subprocess

import cv2
import numpy as np
import pytest

from helpers import REPO
from jpeg_cases import cmyk, encode, hrsc, matrix, no_sync_batch, picture, with_orientation

HARNESS = r'''
#include "jpeg.cuh"
#include <stdio.h>
#include <stdlib.h>
#include <vector>
using namespace ryolo::jpeg;
int main(int argc, char** argv) {
  FILE* f = fopen(argv[1], "rb");
  std::vector<uint8_t> st;
  { fseek(f, 0, SEEK_END); long n = ftell(f); fseek(f, 0, SEEK_SET); st.resize(n); fread(st.data(), 1, n, f); fclose(f); }
  const int nimg = atoi(argv[3]), nsegs = atoi(argv[4]), nchunks = atoi(argv[5]), C = atoi(argv[6]);
  long off[6];
  for (int i = 0; i < 6; i++) off[i] = atol(argv[7 + i]);
  const long area_bytes = atol(argv[13]), out_bytes = atol(argv[14]);
  const ryolo_jpeg_image* im = (const ryolo_jpeg_image*)(st.data() + off[0]);
  const ryolo_jpeg_segment* sg = (const ryolo_jpeg_segment*)(st.data() + off[1]);
  const int32_t* cs = (const int32_t*)(st.data() + off[2]);
  const ryolo_jpeg_huff* hf = (const ryolo_jpeg_huff*)(st.data() + off[3]);
  const uint16_t* q = (const uint16_t*)(st.data() + off[4]);
  const uint8_t* d = st.data() + off[5];
  std::vector<uint8_t> area(area_bytes + 16), out(out_bytes);
  std::vector<uint32_t> exits(2 * nchunks);
  std::vector<int> jump(nchunks), nblk(nchunks), base(nchunks, -1), status(nimg, 0);
  for (int c = 0; c < nchunks; c++) {
    const ryolo_jpeg_segment& s = sg[cs[c]];
    pack(chunk_pass_a(d, s, im[s.image], hf, c - s.first_chunk, C), &exits[2 * c]);
  }
  for (int c = 0; c < nchunks; c++) {
    const ryolo_jpeg_segment& s = sg[cs[c]];
    const int k = c - s.first_chunk;
    const State s0 = k == 0 ? segment_start(s) : unpack(&exits[2 * (c - 1)]);
    const int j = chunk_pass_b(d, s, im[s.image], hf, k, C, s0, &exits[2 * s.first_chunk], &nblk[c]);
    jump[c] = j < 0 ? -1 : s.first_chunk + j;
  }
  for (int g = 0; g < nsegs; g++) {                 // jpeg_resolve_kernel, one 32-chunk window per step
    const int end = sg[g].first_chunk + sg[g].nchunk;
    int p = sg[g].first_chunk, b = 0, broken = 0;
    while (p < end) {
      int first = 32;
      for (int i = 0; i < 32 && p + i < end; i++)
        if (jump[p + i] != p + i) { first = i; break; }
      const int jf = jump[p + (first & 31) < end ? p + (first & 31) : p];
      for (int i = 0; i < 32 && p + i < end; i++)
        if (on_chain(i, first, jf)) { base[p + i] = b; b += nblk[p + i]; }
      p = next_chain(p, first, jf);
      if (p < 0) { broken = 1; break; }
    }
    if (broken) status[sg[g].image] |= RYOLO_JPEG_ST_NO_SYNC;
    else if (b < sg[g].nmcu * im[sg[g].image].bpm) status[sg[g].image] |= RYOLO_JPEG_ST_TRUNCATED;
  }
  for (int c = 0; c < nchunks; c++) {               // jpeg_write_kernel
    if (base[c] < 0 || jump[c] < 0) continue;
    const ryolo_jpeg_segment& s = sg[cs[c]];
    const ryolo_jpeg_image& m = im[s.image];
    const int k = c - s.first_chunk;
    const State s0 = k == 0 ? segment_start(s) : unpack(&exits[2 * (c - 1)]);
    int16_t* blocks = (int16_t*)(area.data() + m.coef_off) + (int64_t)s.first_mcu * m.bpm * 64;
    status[s.image] |= chunk_write(d, s, m, hf, jump[c] - s.first_chunk, C, s0, base[c], blocks);
  }
  for (int g = 0; g < nsegs; g++) {
    const ryolo_jpeg_image& m = im[sg[g].image];
    int16_t* coefs = (int16_t*)(area.data() + m.coef_off);
    for (int ci = 0; ci < m.ncomp; ci++) {
      uint32_t run = 0;
      const int64_t n = (int64_t)sg[g].nmcu * m.h[ci] * m.v[ci];
      for (int64_t e = 0; e < n; e++) {
        int16_t* c0 = coefs + dc_block(m, sg[g], ci, e) * 64;
        run += (uint32_t)(int32_t)*c0;
        *c0 = (int16_t)(run & 0xFFFFu);
      }
    }
  }
  for (int i = 0; i < nimg; i++) {
    const ryolo_jpeg_image& m = im[i];
    for (int64_t b = 0; b < (int64_t)m.mcux * m.mcuy * m.bpm; b++) {
      int row, col;
      const int ci = block_position(m, b, row, col);
      idct_islow((const int16_t*)(area.data() + m.coef_off) + b * 64, q + m.qtab[ci],
                 area.data() + m.plane_off[ci] + (int64_t)row * m.pitch[ci] + col, m.pitch[ci]);
    }
    for (int oy = 0; oy < m.out_h; oy++)
      for (int ox = 0; ox < m.out_w; ox++)
        pixel_bgr(m, area.data(), ox, oy, out.data() + m.out_off + 3 * ((int64_t)oy * m.out_w + ox));
  }
  FILE* g = fopen(argv[2], "wb");
  fwrite(status.data(), 4, nimg, g);
  fwrite(out.data(), 1, out_bytes, g);
  fclose(g);
  return 0;
}
'''


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    d = tmp_path_factory.mktemp("jpeg_host")
    src = d / "h.cpp"
    src.write_text(HARNESS)
    exe = d / "h"
    cmd = ["g++", "-O2", "-std=c++17", "-I" + os.path.join(REPO, "rotate-yolov3_b200", "csrc"), "-o", str(exe), str(src)]
    # with AddressSanitizer where the toolchain has it, so that a read or write outside a buffer fails the test
    if subprocess.run(cmd + ["-fsanitize=address"], capture_output=True).returncode != 0:
        subprocess.run(cmd, check=True)
    return exe, d


def host_decode(harness, blobs, chunk_bytes=128):
    """decode_images' device path run by the host build: (images of the device-routed streams or None, status, routes)"""
    from rotate_yolov3_b200.decode import Layout
    exe, d = harness
    lay = Layout(blobs, chunk_bytes)
    if lay.stage is None:
        return [None] * len(blobs), np.zeros(0, np.int32), lay.routes
    (d / "stage.bin").write_bytes(lay.stage.tobytes())
    args = [str(exe), str(d / "stage.bin"), str(d / "out.bin"), lay.nimg, lay.nsegs, lay.nchunks, lay.chunk_bytes]
    args += list(lay.offsets) + [lay.area, int(lay.out_offs[-1])]
    subprocess.run([str(a) for a in args], check=True)
    raw = np.fromfile(d / "out.bin", np.uint8)
    status = raw[:4 * lay.nimg].view(np.int32)
    out = raw[4 * lay.nimg:]
    imgs = [None] * len(blobs)
    for i in lay.dev_idx:
        hh, ww = lay.shapes[i]
        o = int(lay.out_offs[i])
        imgs[i] = out[o:o + 3 * hh * ww].reshape(hh, ww, 3)
    return imgs, status, lay.routes


def _cv2(blob):
    return cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)


def _check_equal(imgs, status, blobs, names):
    assert not status.any(), [(n, s) for n, s in zip(names, status) if s]
    for name, img, blob in zip(names, imgs, blobs):
        want = _cv2(blob)
        assert img is not None, name
        assert img.shape == want.shape, (name, img.shape, want.shape)
        nd = int((img != want).sum())
        assert nd == 0, "%s: %d of %d values differ from cv2 (max |d| %d)" % (
            name, nd, want.size, int(np.abs(img.astype(int) - want).max()))


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
            assert _cv2(with_orientation(base, o, be)).shape[:2] == hd.out_hw


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
            assert np.array_equal(lay.host[i], _cv2(blobs[i]))
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
    _check_equal(imgs, status, blobs, names)


@pytest.mark.parametrize("chunk", [1, 7, 16, 4096])
def test_host_build_chunk_sizes(harness, chunk):
    """tiny chunks force the synchronisation on every image, one huge chunk decodes each segment in one piece"""
    cases = [c for c in matrix() if c[0].startswith(("121x163", "33x47", "orient"))]
    names, blobs = [c[0] for c in cases], [c[1] for c in cases]
    imgs, status, _ = host_decode(harness, blobs, chunk)
    _check_equal(imgs, status, blobs, names)


def test_host_build_hrsc_and_hd(harness):
    """the reference's HRSC sample (1167 x 821, 4:2:0, no restarts) in 16-byte chunks (thousands of them), and a
    1920 x 1080 q95 4:4:4 frame with restart interval 17"""
    blobs = [hrsc(), encode(picture(11, 1080, 1920), 95, "444", restart=17)]
    imgs, status, _ = host_decode(harness, blobs, 16)
    _check_equal(imgs, status, blobs, ["hrsc", "hd"])


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
        want = _cv2(blob)
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
    assert _cv2(blobs[1]) is not None
    imgs, status, routes = host_decode(harness, blobs)
    assert routes == ["device", "device"]
    assert status[0] == 0 and status[1] & 4, status
    assert np.array_equal(imgs[0], _cv2(blobs[0]))
