// area(a ∩ b) of two rotated rectangles by the CLAMP INTEGRAL, second formulation (round 2).
//
// As in round 1 (riou.cu header): the intersection area equals the area enclosed by the image of b's boundary under the
// Euclidean projection onto a -- in a's frame the coordinate-wise clamp -- a continuous, branch-free function of the
// inputs with no topological decisions.  What changed is how the integral is taken, to cut its instruction count from
// ~300 to ~140 per pair:
//   * a's frame is NORMALISED to the unit square [0,1]^2 (x'' = (x + hw)/(2 hw)), so every clamp is the free `.sat`
//     modifier of the FADD/FFMA that produces the value (no FMNMX pairs: round 1 spent 136 of them per pair);
//   * Green's theorem with the 1-form x dy instead of (x dy - y dx)/2:  area = closed-integral of X dY over the clamped
//     curve.  On one edge Y(t) = sat(ay + t ey) moves only for t in [ty_lo, ty_hi] (its two clamp breakpoints), with
//     dY = ey dt there, so the edge contributes  ey * integral_{ty_lo}^{ty_hi} sat(ax + t ex) dt : a clamped linear
//     function over ONE interval = three trapezoids between (ty_lo, s1, s2, ty_hi), s1/s2 = X's breakpoints clamped into
//     the interval.  No sorting network, 4 evaluations of X per edge instead of 2 x 5.
//   * the breakpoints of one coordinate are  -c + min(r,0)  and  -c + max(r,0)  with r = 1/e, c = a*r: already ordered.
// Degenerate edges (e = 0 -> r = inf, c = inf or NaN) only produce arbitrary breakpoints in [0,1] (`.sat` maps NaN to 0),
// which subdivide a piece on which the clamped coordinate is constant: harmless, as in round 1.
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define RY_HD __host__ __device__ __forceinline__
#else
#define RY_HD static inline
#endif

namespace ryolo {

#if defined(__CUDA_ARCH__)
RY_HD float ry_sat(float x) { return __saturatef(x); }
RY_HD float ry_rcp(float x) {   // bare MUFU.RCP (1 ulp); 1/0 = inf, handled by the .sat breakpoints
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
#else
RY_HD float ry_sat(float x) { return fminf(fmaxf(x, 0.f), 1.f); }   // fmaxf(NaN, 0) = 0, like .sat
RY_HD float ry_rcp(float x) { return 1.f / x; }
#endif

// one edge: start (ax, ay), vector (ex, ey) in the normalised frame; (rxn, rxp) = (min(1/ex,0), max(1/ex,0)), same for y
RY_HD float clamp_edge_xdy(float ax, float ay, float ex, float ey, float rx, float rxn, float rxp, float ry, float ryn,
                           float ryp) {
  const float cx = ax * rx, cy = ay * ry;
  const float tx_lo = ry_sat(rxn - cx), tx_hi = ry_sat(rxp - cx);
  const float ty_lo = ry_sat(ryn - cy), ty_hi = ry_sat(ryp - cy);
  const float s1 = fmaxf(ty_lo, fminf(tx_lo, ty_hi));
  const float s2 = fmaxf(ty_lo, fminf(tx_hi, ty_hi));
  const float xa = ry_sat(fmaf(ty_lo, ex, ax));
  const float xb = ry_sat(fmaf(s1, ex, ax));
  const float xc = ry_sat(fmaf(s2, ex, ax));
  const float xd = ry_sat(fmaf(ty_hi, ex, ax));
  float in = (xa + xb) * (s1 - ty_lo);
  in = fmaf(xb + xc, s2 - s1, in);
  in = fmaf(xc + xd, ty_hi - s2, in);
  return ey * in;     // twice the contribution
}

// The frame box a should have its long side along y (canonical_frame): b's edges enter the integral weighted by ey, and each
// breakpoint's rounding (~u in t) moves an edge's dY by ~u |ey|, multiplied by X in [0, 1].  With a thin box along x
// crossed at a steep angle, |ey| reaches ~50 (b's length over a's height): two aspect-50 boxes crossing at 75 degrees put
// the IoU 1e-6 off, past the 1e-4 relative + 1e-6 contract.  With a's long side along y, |ey| is at most b's length over
// a's long side.
RY_HD void canonical_frame(float& c, float& s, float& hw, float& hh) {
  if (hw > hh) {   // the same rectangle turned by +90 degrees: exact (a swap and a negation)
    const float t = c;
    c = -s;
    s = t;
    const float h = hw;
    hw = hh;
    hh = h;
  }
}

// a: centre (acx, acy), cos/sin (ac, as), half extents (ahw, ahh) in canonical_frame; b likewise (any frame).  Returns
// area(a ∩ b) >= 0.
RY_HD float clamp_integral_area2(float acx, float acy, float ac, float as, float ahw, float ahh, float bcx, float bcy,
                                 float bc, float bs, float bhw, float bhh) {
  const float dx = bcx - acx, dy = bcy - acy;
  const float rx = fmaf(dx, ac, dy * as);
  const float ry = fmaf(dy, ac, -dx * as);
  const float cd = fmaf(ac, bc, as * bs);    // cos(theta_b - theta_a)
  const float sd = fmaf(ac, bs, -as * bc);   // sin(theta_b - theta_a)
  const float iw = ry_rcp(ahw), ih = ry_rcp(ahh);     // 2 * (1 / (2 hw)), 2 * (1 / (2 hh))
  // b's full edge vectors U = 2u, V = 2v in the normalised frame (x'' = x / (2 hw) + 1/2)
  const float kx = bhw * iw, ky = bhw * ih, lx = bhh * iw, ly = bhh * ih;
  const float Ux = cd * kx, Uy = sd * ky, Vx = -sd * lx, Vy = cd * ly;
  const float ox = fmaf(rx, 0.5f * iw, 0.5f), oy = fmaf(ry, 0.5f * ih, 0.5f);    // b's centre
  // corners counter-clockwise: p0 = o - U/2 - V/2, p1 = p0 + U, p2 = p1 + V, p3 = p0 + V
  const float p0x = fmaf(-0.5f, Vx, fmaf(-0.5f, Ux, ox)), p0y = fmaf(-0.5f, Vy, fmaf(-0.5f, Uy, oy));
  const float p1x = p0x + Ux, p1y = p0y + Uy;
  const float p2x = p1x + Vx, p2y = p1y + Vy;
  const float p3x = p0x + Vx, p3y = p0y + Vy;
  const float rUx = ry_rcp(Ux), rUy = ry_rcp(Uy), rVx = ry_rcp(Vx), rVy = ry_rcp(Vy);
  const float rUxn = fminf(rUx, 0.f), rUxp = fmaxf(rUx, 0.f), rUyn = fminf(rUy, 0.f), rUyp = fmaxf(rUy, 0.f);
  const float rVxn = fminf(rVx, 0.f), rVxp = fmaxf(rVx, 0.f), rVyn = fminf(rVy, 0.f), rVyp = fmaxf(rVy, 0.f);
  float acc = clamp_edge_xdy(p0x, p0y, Ux, Uy, rUx, rUxn, rUxp, rUy, rUyn, rUyp);      // p0 -> p1 along +U
  acc += clamp_edge_xdy(p1x, p1y, Vx, Vy, rVx, rVxn, rVxp, rVy, rVyn, rVyp);           // p1 -> p2 along +V
  acc += clamp_edge_xdy(p2x, p2y, -Ux, -Uy, -rUx, -rUxp, -rUxn, -rUy, -rUyp, -rUyn);   // p2 -> p3 along -U
  acc += clamp_edge_xdy(p3x, p3y, -Vx, -Vy, -rVx, -rVxp, -rVxn, -rVy, -rVyp, -rVyn);   // p3 -> p0 along -V
  // acc = 2 * area in the unit square; a's area is (2 hw)(2 hh)
  return fmaxf(acc * (2.f * ahw * ahh), 0.f);
}

}  // namespace ryolo
