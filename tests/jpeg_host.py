"""The host build of the device JPEG decoder: csrc/jpeg.cuh compiled with g++ into a program that runs the device's
passes serially -- chunk pass A, pass B, the chain resolution, the writers, the DC prefix, the IDCT and the pixel store
-- on the batch rotate_yolov3_b200.decode.Layout stages, so that the decoder can be compared with cv2.imdecode on
machines without a GPU."""
import os
import shutil
import subprocess

import cv2
import numpy as np
import pytest

from helpers import REPO

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
      status[i] |= idct_islow((const int16_t*)(area.data() + m.coef_off) + b * 64, q + m.qtab[ci],
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
#ifdef RJ_STATS
  rj_stats_print();
#endif
  return 0;
}
'''


def build_harness(d, patches=()):
    """compile HARNESS against csrc/jpeg.cuh into directory d: (executable, d).  patches: (file, old, new) edits, file
    "harness" or "jpeg.cuh", applied to copies of the sources (each `old` must occur), for bug insertions and
    instrumented builds.  With AddressSanitizer where the toolchain has it, so that a read or write outside a buffer
    fails the test."""
    src = {"harness": HARNESS, "jpeg.cuh": open(os.path.join(REPO, "rotate-yolov3_b200", "csrc", "jpeg.cuh")).read()}
    for f, old, new in patches:
        assert old in src[f], (f, old)
        src[f] = src[f].replace(old, new)
    csrc = d / "pkg" / "csrc"
    csrc.mkdir(parents=True, exist_ok=True)
    (d / "include").mkdir(exist_ok=True)
    shutil.copy(os.path.join(REPO, "include", "ryolo.h"), d / "include" / "ryolo.h")
    (csrc / "jpeg.cuh").write_text(src["jpeg.cuh"])
    (d / "h.cpp").write_text(src["harness"])
    exe = d / "h"
    cmd = ["g++", "-O2", "-std=c++17", "-I" + str(csrc), "-o", str(exe), str(d / "h.cpp")]
    if subprocess.run(cmd + ["-fsanitize=address"], capture_output=True).returncode != 0:
        subprocess.run(cmd, check=True)
    return exe, d


def make_harness(tmp_path_factory, name="jpeg_host", patches=()):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    return build_harness(tmp_path_factory.mktemp(name), patches)


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
    run = subprocess.run([str(a) for a in args], check=True, capture_output=True, text=True)
    host_decode.stdout = run.stdout
    raw = np.fromfile(d / "out.bin", np.uint8)
    status = raw[:4 * lay.nimg].view(np.int32)
    out = raw[4 * lay.nimg:]
    imgs = [None] * len(blobs)
    for i in lay.dev_idx:
        hh, ww = lay.shapes[i]
        o = int(lay.out_offs[i])
        imgs[i] = out[o:o + 3 * hh * ww].reshape(hh, ww, 3)
    return imgs, status, lay.routes


def cv2_decode(blob):
    """what cv2.imread returns for a file holding blob (None when cv2 rejects it)"""
    return cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)


def check_equal(imgs, status, blobs, names):
    assert not status.any(), [(n, s) for n, s in zip(names, status) if s]
    for name, img, blob in zip(names, imgs, blobs):
        want = cv2_decode(blob)
        assert img is not None, name
        assert img.shape == want.shape, (name, img.shape, want.shape)
        nd = int((img != want).sum())
        assert nd == 0, "%s: %d of %d values differ from cv2 (max |d| %d)" % (
            name, nd, want.size, int(np.abs(img.astype(int) - want).max()))
