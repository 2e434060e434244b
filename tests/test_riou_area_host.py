"""csrc/riou_area.cuh (the clamp integral of the rotated-IoU kernels, second formulation) evaluated ON THE HOST in fp32 --
the header compiles with g++, the `.sat` clamps become fmin/fmax -- against the float64 convex-clip oracle: random boxes,
axis-aligned boxes with integer coordinates and collinear / identical edges, 90-degree rotations, near-identical pairs.
Tolerance = the GPU tests' (1e-4 relative + 1e-6).  This pins the arithmetic of the formulation without a GPU; the kernels'
own parity tests are in test_riou_gpu.py / test_riou_loss_gpu.py."""
import os
import shutil
import subprocess

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r'''
#include <stdio.h>
#include <stdlib.h>
#include <math.h>
#include "riou_area.cuh"
extern "C" double orc_skew_iou(const double* box1, const double* box2, int mode);
static double urand() { return rand() / (RAND_MAX + 1.0); }
static void gen(double* b, double canvas, int kind) {
  b[0] = urand() * canvas; b[1] = urand() * canvas;
  double area = 792 + urand() * (15803 - 792), ratio = 4 + urand() * 5;
  b[2] = sqrt(area * ratio); b[3] = sqrt(area / ratio);
  b[4] = (urand() - 0.5) * M_PI;
  if (kind == 1) { b[4] = 0; b[0] = floor(b[0]); b[1] = floor(b[1]); b[2] = floor(b[2]); b[3] = floor(b[3]) + 1; }
  if (kind == 2) { b[4] = (rand() % 4) * M_PI / 2 - M_PI / 2; }
}
static float iou32(const float* a, const float* b) {
  float c = cosf(a[4]), s = sinf(a[4]), hw = 0.5f * a[2], hh = 0.5f * a[3];
  ryolo::canonical_frame(c, s, hw, hh);
  float inter = ryolo::clamp_integral_area2(a[0], a[1], c, s, hw, hh, b[0], b[1],
                                            cosf(b[4]), sinf(b[4]), 0.5f * b[2], 0.5f * b[3]);
  const float aa = a[2] * a[3], ab = b[2] * b[3];
  inter = fminf(inter, fminf(aa, ab));
  const float u = aa + ab - inter;
  return u == 0.f ? 0.f : inter / u;
}
int main() {
  srand(7);
  long bad = 0, nonzero = 0;
  for (int kind = 0; kind < 4; kind++) {
    for (long it = 0; it < 250000; it++) {
      double a[5], b[5];
      const double canvas = kind == 3 ? 100.0 : 300.0;
      gen(a, canvas, kind == 3 ? 0 : kind); gen(b, canvas, kind == 3 ? 0 : kind);
      if (kind == 1 && (it & 3) == 0) { b[1] = a[1]; b[3] = a[3]; }            /* collinear top / bottom edges */
      if (kind == 1 && (it & 7) == 1) { for (int i = 0; i < 5; i++) b[i] = a[i]; }
      if (kind == 3) { for (int i = 0; i < 5; i++) b[i] = a[i] + (urand() - 0.5) * 1e-3 * (it % 1000); }
      float fa[5], fb[5]; double da[5], db[5];
      for (int i = 0; i < 5; i++) { fa[i] = (float)a[i]; fb[i] = (float)b[i]; da[i] = fa[i]; db[i] = fb[i]; }
      const double ref = orc_skew_iou(da, db, 0), got = iou32(fa, fb);
      if (ref > 0) nonzero++;
      if (fabs(got - ref) > 1e-4 * fabs(ref) + 1e-6) bad++;
    }
  }
  printf("%ld %ld\n", bad, nonzero);
  return bad != 0;
}
'''


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
def test_clamp_integral_on_the_host_vs_float64_oracle(tmp_path):
    orc = os.path.join(REPO, "oracle", "librbox_oracle.so")
    if not os.path.exists(orc):
        pytest.skip("oracle/librbox_oracle.so not built (python -c 'import __graft_entry__ as g; g.build()')")
    src = tmp_path / "t.cpp"
    src.write_text(SRC)
    exe = tmp_path / "t"
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-I" + os.path.join(REPO, "rotate-yolov3_b200", "csrc"), "-o", str(exe),
                    str(src), orc, "-Wl,-rpath," + os.path.join(REPO, "oracle"), "-lm"], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    bad, nonzero = (int(v) for v in out.stdout.split())
    assert out.returncode == 0 and bad == 0, out.stdout
    assert nonzero > 400000          # the sets actually overlap
