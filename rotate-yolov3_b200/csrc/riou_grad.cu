// Rotated-IoU as a DIFFERENTIABLE op: IoU of paired rotated boxes plus its analytic gradient with respect to both boxes
// (SURVEY.md 8f item 4: the README's "riou loss", README.md:18, which model/loss.py never implemented -- its regression
// loss is SmoothL1 + a horizontal wh_iou, SURVEY D1).  Extension with no reference counterpart; the oracle is the float64
// convex-clip IoU of oracle/rbox_oracle.c differentiated numerically (tests/test_riou_loss_gpu.py).
//
// Gradient of the intersection area I = area(a ∩ b) by the boundary-velocity (Reynolds transport) formula: when a
// parameter p of box b changes, I changes by the integral over the part of b's boundary that lies INSIDE a of the
// boundary's normal velocity,
//        dI/dp = sum over the 4 edges e of b of  ∫_{e ∩ a} n_e · (∂x/∂p) ds .
// For a rectangle x = c + R(θ)(u, v):  ∂x/∂c = identity,  ∂x/∂θ = perp(x − c),  the edges u = ±w/2 move along their
// normal by ±dw/2 (the other two edges slide tangentially: no normal velocity), likewise h.  All integrands are linear
// along an edge, so with L_e = length of e ∩ a, m_e = its midpoint:
//        dI/dc = Σ L_e n_e,   dI/dθ = Σ L_e n_e · perp(m_e − c),   dI/dw = ½ Σ_{e ∈ {u = ±w/2}} L_e,   dI/dh likewise.
// e ∩ a is one parametric interval per edge (Liang–Barsky against a's four half-planes in a's frame) -- no polygon
// clipping, no vertex arrays.  The gradient w.r.t. box a is the same computation with the roles swapped.
// IoU = I / U, U = A_a + A_b − I:   dIoU = ((U + I) dI − I dA) / U².  The value of I itself: clamp integral (see below).
#include "common.cuh"
#include "riou_area.cuh"

namespace ryolo {

struct GBox {
  float cx, cy, w, h, c, s;
};

__device__ __forceinline__ GBox load_gbox(const float* __restrict__ p) {
  GBox b;
  b.cx = p[0]; b.cy = p[1]; b.w = fabsf(p[2]); b.h = fabsf(p[3]);
  sincosf(p[4], &b.s, &b.c);
  return b;
}

// d(area(inner ∩ outer)) / d(cx, cy, w, h, theta of `inner`)
__device__ __forceinline__ void edge_terms(const GBox& in, const GBox& out, float* g /*[5]*/) {
  // inner box in outer's frame
  const float dx = in.cx - out.cx, dy = in.cy - out.cy;
  const float rx = dx * out.c + dy * out.s, ry = dy * out.c - dx * out.s;
  const float cd = out.c * in.c + out.s * in.s, sd = out.c * in.s - out.s * in.c;   // relative rotation
  const float hw = 0.5f * in.w, hh = 0.5f * in.h, HW = 0.5f * out.w, HH = 0.5f * out.h;
  // local axes of inner in outer's frame
  const float ux = cd, uy = sd, vx = -sd, vy = cd;
  float gx = 0.f, gy = 0.f, gw = 0.f, gh = 0.f, gt = 0.f;
#pragma unroll
  for (int e = 0; e < 4; e++) {
    // edge e, counter-clockwise: 0: v = -hh (u from -hw to hw), 1: u = +hw, 2: v = +hh, 3: u = -hw
    float ax, ay, ex, ey, nx, ny;
    if (e == 0) { ax = rx - hw * ux - hh * vx; ay = ry - hw * uy - hh * vy; ex = 2.f * hw * ux; ey = 2.f * hw * uy; nx = -vx; ny = -vy; }
    else if (e == 1) { ax = rx + hw * ux - hh * vx; ay = ry + hw * uy - hh * vy; ex = 2.f * hh * vx; ey = 2.f * hh * vy; nx = ux; ny = uy; }
    else if (e == 2) { ax = rx + hw * ux + hh * vx; ay = ry + hw * uy + hh * vy; ex = -2.f * hw * ux; ey = -2.f * hw * uy; nx = vx; ny = vy; }
    else { ax = rx - hw * ux + hh * vx; ay = ry - hw * uy + hh * vy; ex = -2.f * hh * vx; ey = -2.f * hh * vy; nx = -ux; ny = -uy; }
    // Liang-Barsky: t in [t0, t1] with |ax + t ex| <= HW and |ay + t ey| <= HH
    float t0 = 0.f, t1 = 1.f;
    bool ok = true;
    {
      if (ex == 0.f) ok = ok && fabsf(ax) <= HW;
      else {
        const float inv = 1.f / ex;
        float ta = (-HW - ax) * inv, tb = (HW - ax) * inv;
        if (ta > tb) { const float t = ta; ta = tb; tb = t; }
        t0 = fmaxf(t0, ta); t1 = fminf(t1, tb);
      }
      if (ey == 0.f) ok = ok && fabsf(ay) <= HH;
      else {
        const float inv = 1.f / ey;
        float ta = (-HH - ay) * inv, tb = (HH - ay) * inv;
        if (ta > tb) { const float t = ta; ta = tb; tb = t; }
        t0 = fmaxf(t0, ta); t1 = fminf(t1, tb);
      }
    }
    if (!ok || !(t1 > t0)) continue;
    const float elen = (e & 1) ? 2.f * hh : 2.f * hw;       // |edge|
    const float L = (t1 - t0) * elen;
    const float tm = 0.5f * (t0 + t1);
    const float mx = ax + tm * ex - rx, my = ay + tm * ey - ry;    // midpoint relative to inner's centre (outer frame)
    gx += L * nx;
    gy += L * ny;
    gt += L * (nx * (-my) + ny * mx);
    if (e & 1) gw += 0.5f * L; else gh += 0.5f * L;
  }
  // rotate the centre gradient back to the world frame
  g[0] = gx * out.c - gy * out.s;
  g[1] = gx * out.s + gy * out.c;
  g[2] = gw;
  g[3] = gh;
  g[4] = gt;
}

// separated on one of the four box axes by more than the fp32 rounding of the projections (8 u of their scale)
__device__ __forceinline__ bool separated(const GBox& a, const GBox& b) {
  const float dx = b.cx - a.cx, dy = b.cy - a.cy;
  const float C = fabsf(a.c * b.c + a.s * b.s), S = fabsf(a.c * b.s - a.s * b.c);
  const float ha = 0.5f * a.w, ka = 0.5f * a.h, hb = 0.5f * b.w, kb = 0.5f * b.h;
  const float slack = 4.76837158e-7f * (fabsf(dx) + fabsf(dy) + ha + ka + hb + kb);   // 8 * 2^-24
  return fabsf(dx * a.c + dy * a.s) - (ha + hb * C + kb * S) > slack ||
         fabsf(dy * a.c - dx * a.s) - (ka + hb * S + kb * C) > slack ||
         fabsf(dx * b.c + dy * b.s) - (hb + ha * C + ka * S) > slack ||
         fabsf(dy * b.c - dx * b.s) - (kb + ha * S + ka * C) > slack;
}

__global__ void __launch_bounds__(128) riou_grad_kernel(const float* __restrict__ a, const float* __restrict__ b, int n,
                                                        int sa, int sb, const float* __restrict__ gout,
                                                        float* __restrict__ iou_out, float* __restrict__ ga,
                                                        float* __restrict__ gb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* pa = a + (size_t)i * sa;
  const float* pb = b + (size_t)i * sb;
  const GBox A = load_gbox(pa), B = load_gbox(pb);
  float dIa[5], dIb[5];
  edge_terms(A, B, dIa);      // a's edges inside b: dI/d(a)
  edge_terms(B, A, dIb);      // b's edges inside a: dI/d(b)
  // The area VALUE comes from the clamp integral of riou_area.cuh (the matrix kernel's routine): continuous and free of tie
  // rules.  The edge terms above would give it too (Euler's theorem for the degree-2 homogeneity under common scaling:
  // 2 I = w_a I_wa + h_a I_ha + w_b I_wb + h_b I_hb + (c_b − c_a)·∇_{c_b} I), but that sum counts a run where an edge of a
  // lies ON an edge of b twice (once in each box's terms) -- exactly the axis-aligned, equal-height boxes detection data is
  // full of; there the gradient is one-sided anyway, the value must still be right.
  float fc = A.c, fs = A.s, fhw = 0.5f * A.w, fhh = 0.5f * A.h;
  canonical_frame(fc, fs, fhw, fhh);
  float I = clamp_integral_area2(A.cx, A.cy, fc, fs, fhw, fhh, B.cx, B.cy, B.c, B.s, 0.5f * B.w, 0.5f * B.h);
  const float Aa = A.w * A.h, Ab = B.w * B.h;
  const bool finite = isfinite(pa[0]) && isfinite(pa[1]) && isfinite(pa[2]) && isfinite(pa[3]) && isfinite(pa[4]) &&
                      isfinite(pb[0]) && isfinite(pb[1]) && isfinite(pb[2]) && isfinite(pb[3]) && isfinite(pb[4]);
  I = fminf(fmaxf(I, 0.f), fminf(Aa, Ab));
  const float U = Aa + Ab - I;
  // Separated boxes have IoU 0 and zero gradients, whatever rounding residue the clamp integral leaves for them (a few
  // 1e-7 of the areas): that residue would otherwise turn into a w / h gradient through the union.
  const bool live = finite && Aa > 0.f && Ab > 0.f && U > 0.f && !separated(A, B);
  const float iou = live ? I / U : 0.f;
  if (iou_out) iou_out[i] = iou;
  if (!live) {   // disjoint, zero-area or invalid: the edge terms may hold inf or NaN, so no 0 * dI here
#pragma unroll
    for (int k = 0; k < 5; k++) {
      if (ga) ga[(size_t)i * 5 + k] = 0.f;
      if (gb) gb[(size_t)i * 5 + k] = 0.f;
    }
    return;
  }
  const float go = gout ? gout[i] : 1.f;
  const float k1 = go * (U + I) / (U * U);     // multiplies dI
  const float k2 = go * I / (U * U);           // multiplies dA
  // sign of w, h: the box uses |w|, |h|
  const float swa = pa[2] < 0.f ? -1.f : 1.f, sha = pa[3] < 0.f ? -1.f : 1.f;
  const float swb = pb[2] < 0.f ? -1.f : 1.f, shb = pb[3] < 0.f ? -1.f : 1.f;
  if (ga) {
    float* o = ga + (size_t)i * 5;
    o[0] = k1 * dIa[0];
    o[1] = k1 * dIa[1];
    o[2] = swa * (k1 * dIa[2] - k2 * A.h);
    o[3] = sha * (k1 * dIa[3] - k2 * A.w);
    o[4] = k1 * dIa[4];
  }
  if (gb) {
    float* o = gb + (size_t)i * 5;
    o[0] = k1 * dIb[0];
    o[1] = k1 * dIb[1];
    o[2] = swb * (k1 * dIb[2] - k2 * B.h);
    o[3] = shb * (k1 * dIb[3] - k2 * B.w);
    o[4] = k1 * dIb[4];
  }
}

}  // namespace ryolo

using namespace ryolo;

extern "C" int ryolo_riou_paired_grad(const float* a, const float* b, int n, int stride_a, int stride_b,
                                      const float* grad_out, float* iou_out, float* grad_a, float* grad_b, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(n >= 0 && stride_a >= 5 && stride_b >= 5);
  if (n == 0) return RYOLO_OK;
  RYOLO_ARG_CHECK(a && b && (iou_out || grad_a || grad_b));
  riou_grad_kernel<<<(n + 127) / 128, 128, 0, stream>>>(a, b, n, stride_a, stride_b, grad_out, iou_out, grad_a, grad_b);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}
