// Rotated-box IoU for sm_90a with skew_bbox_iou semantics (reference: utils/utils.py:290-320,
// skewiou :663-699, get_rotated_coors :702-725).  The reference computes one pair at a time in Python
// through cv2 + shapely (float64 GEOS); here one launch produces the whole N x M matrix (or the N paired values).
//
// Geometry.  Box b is expressed in box a's local frame (centre difference rotated by -theta_a, relative rotation
// theta_b - theta_a from the per-box sin/cos), which keeps fp32 cancellation at box scale instead of canvas scale.
// The intersection area is the area enclosed by the image of b's boundary under the Euclidean PROJECTION onto a
// (for an axis-aligned box: the coordinate-wise clamp).  For z in int(a) the winding number of that image curve
// about z equals the winding number of the boundary of b (the segment from w to clamp(w) never enters int(a)), and it
// is 0 outside a, so
//        area(a ∩ b) = (1/2) * closed-integral over clamp(boundary b) of (x dy - y dx) = sum over edges of
//                      sum over the linear pieces between clamp breakpoints of (X_i + X_{i+1}) (Y_{i+1} - Y_i) / 2.
// Each edge has at most 4 breakpoints (x = ±hw, y = ±hh); they are sorted with a 5-comparator network, extra or
// coincident breakpoints are harmless (they only subdivide a linear piece), so the routine is branch-free, needs no
// vertex arrays, and is a continuous function of its inputs (identical boxes -> 1, touching boxes -> 0, no
// topological decisions as in edge-crossing enumeration).  ~300 fp32 instructions per pair, all lanes converged.
//
// Pairwise kernel: CTA tile = 32 rows x 128 columns, 256 threads.  Stage A1: bounding-circle test for every pair
// (10 instructions, one LDS.128 broadcast); survivors (~28 %) are compacted once per thread into queue 1.
// Stage A2: separating-axis test on queue 1 with converged warps -> queue 2 (~12 % of all pairs).  Stage B: clamp
// integral on queue 2.  The output tile lives in shared memory (pre-zeroed) and is written back with 128-bit
// streaming stores, so HBM sees exactly one coalesced write of the matrix.
#include "common.cuh"
#include "f32x2.cuh"
#include "riou_area.cuh"

namespace ryolo {

constexpr int RT = 32;    // tile rows
constexpr int CT = 128;   // tile columns
constexpr int RIOU_THREADS = 256;

struct RBox {  // per-box derived data, two float4
  float cx, cy, rad, area;  // rad < 0 marks a box whose IoU with anything is 0 (invalid or zero area)
  float c, s, hw, hh;
};

__device__ __forceinline__ RBox make_rbox(const float* __restrict__ p) {
  RBox b;
  const float cx = p[0], cy = p[1], w = p[2], h = p[3], th = p[4];
  b.cx = cx;
  b.cy = cy;
  b.hw = 0.5f * fabsf(w);
  b.hh = 0.5f * fabsf(h);
  sincosf(th, &b.s, &b.c);
  b.area = fabsf(w * h);  // Polygon(...).convex_hull.area of the 4 corners (utils/utils.py:667-668)
  const bool live = isfinite(cx) && isfinite(cy) && isfinite(w) && isfinite(h) && isfinite(th) &&
                    b.area != 0.f && isfinite(b.area);  // invalid polygon / zero area -> 0 (utils/utils.py:669-673)
  b.rad = live ? sqrtf(b.hw * b.hw + b.hh * b.hh) : -1.f;
  return b;
}

// a's frame: |x| <= hw, |y| <= hh.  Returns area(a ∩ b).
__device__ __forceinline__ float clamp_integral_area(const RBox& a, const RBox& b) {
  const float dx = b.cx - a.cx, dy = b.cy - a.cy;
  const float rx = dx * a.c + dy * a.s;
  const float ry = dy * a.c - dx * a.s;
  const float cd = a.c * b.c + a.s * b.s;   // cos(theta_b - theta_a)
  const float sd = a.c * b.s - a.s * b.c;   // sin(theta_b - theta_a)
  const float ux = cd * b.hw, uy = sd * b.hw;
  const float vx = -sd * b.hh, vy = cd * b.hh;
  const float hw = a.hw, hh = a.hh;
  // corners, counter-clockwise (u x v = hw_b * hh_b > 0)
  const float px[4] = {rx - ux - vx, rx + ux - vx, rx + ux + vx, rx - ux + vx};
  const float py[4] = {ry - uy - vy, ry + uy - vy, ry + uy + vy, ry - uy + vy};
  float cxp[4], cyp[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    cxp[i] = fminf(fmaxf(px[i], -hw), hw);
    cyp[i] = fminf(fmaxf(py[i], -hh), hh);
  }
  float acc = 0.f;
  // edge vectors are +2u, +2v, -2u, -2v: four reciprocals serve the eight x/y breakpoint slopes
  const float ru_x = __fdividef(0.5f, ux), ru_y = __fdividef(0.5f, uy), rv_x = __fdividef(0.5f, vx), rv_y = __fdividef(0.5f, vy);
#pragma unroll
  for (int e = 0; e < 4; e++) {
    const int f = (e + 1) & 3;
    const float ax = px[e], ay = py[e];
    const float ex = px[f] - ax, ey = py[f] - ay;
    const float rex = e == 0 ? ru_x : (e == 1 ? rv_x : (e == 2 ? -ru_x : -rv_x));
    const float rey = e == 0 ? ru_y : (e == 1 ? rv_y : (e == 2 ? -ru_y : -rv_y));
    // breakpoints (clamped to [0,1]; NaN from 0*inf is dropped by fmaxf/fminf)
    float t0 = fminf(fmaxf((-hw - ax) * rex, 0.f), 1.f);
    float t1 = fminf(fmaxf((hw - ax) * rex, 0.f), 1.f);
    float t2 = fminf(fmaxf((-hh - ay) * rey, 0.f), 1.f);
    float t3 = fminf(fmaxf((hh - ay) * rey, 0.f), 1.f);
    float lo, hi;
    lo = fminf(t0, t1); hi = fmaxf(t0, t1); t0 = lo; t1 = hi;
    lo = fminf(t2, t3); hi = fmaxf(t2, t3); t2 = lo; t3 = hi;
    lo = fminf(t0, t2); hi = fmaxf(t0, t2); t0 = lo; t2 = hi;
    lo = fminf(t1, t3); hi = fmaxf(t1, t3); t1 = lo; t3 = hi;
    lo = fminf(t1, t2); hi = fmaxf(t1, t2); t1 = lo; t2 = hi;
    float X0 = cxp[e], Y0 = cyp[e];
    const float ts[4] = {t0, t1, t2, t3};
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const float X1 = fminf(fmaxf(fmaf(ts[k], ex, ax), -hw), hw);
      const float Y1 = fminf(fmaxf(fmaf(ts[k], ey, ay), -hh), hh);
      acc = fmaf(X0 + X1, Y1 - Y0, acc);
      X0 = X1;
      Y0 = Y1;
    }
    acc = fmaf(X0 + cxp[f], cyp[f] - Y0, acc);
  }
  return fmaxf(0.5f * acc, 0.f);
}

// axis-aligned envelope of the 8 corners (mode 'giou', utils/utils.py:682-685), taken relative to a's centre: at 1e5 px
// cx +- extent rounds by up to 4e-3 px, which put the envelope of a 100 x 10 px pair 4e-4 off
__device__ __forceinline__ float envelope_area(const RBox& a, const RBox& b) {
  const float ax = fabsf(a.c) * a.hw + fabsf(a.s) * a.hh, ay = fabsf(a.s) * a.hw + fabsf(a.c) * a.hh;
  const float bx = fabsf(b.c) * b.hw + fabsf(b.s) * b.hh, by = fabsf(b.s) * b.hw + fabsf(b.c) * b.hh;
  const float dx = b.cx - a.cx, dy = b.cy - a.cy;
  const float x0 = fminf(-ax, dx - bx), x1 = fmaxf(ax, dx + bx);
  const float y0 = fminf(-ay, dy - by), y1 = fmaxf(ay, dy + by);
  return (x1 - x0) * (y1 - y0);
}

// strictly-separated test on the 4 box axes (tiny relative slack: touching boxes go on to the integral)
__device__ __forceinline__ bool sat_disjoint(const RBox& a, const RBox& b) {
  const float dx = b.cx - a.cx, dy = b.cy - a.cy;
  const float k = 1.0001f;
  const float C = fabsf(a.c * b.c + a.s * b.s);
  const float S = fabsf(a.c * b.s - a.s * b.c);
  if (fabsf(dx * a.c + dy * a.s) > k * (a.hw + b.hw * C + b.hh * S)) return true;
  if (fabsf(dy * a.c - dx * a.s) > k * (a.hh + b.hw * S + b.hh * C)) return true;
  if (fabsf(dx * b.c + dy * b.s) > k * (b.hw + a.hw * C + a.hh * S)) return true;
  if (fabsf(dy * b.c - dx * b.s) > k * (b.hh + a.hw * S + a.hh * C)) return true;
  return false;
}

__device__ __forceinline__ float iou_from_inter(const RBox& a, const RBox& b, float inter, int mode) {
  inter = fminf(inter, fminf(a.area, b.area));
  const float uni = mode == RYOLO_IOU_MODE_GIOU ? envelope_area(a, b) : a.area + b.area - inter;
  return uni == 0.f ? 0.f : inter / uni;   // union == 0 -> 0 (utils/utils.py:693-694)
}

__global__ void __launch_bounds__(256) riou_paired_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                          int n, int sa, int sb, int mode, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const RBox ba = make_rbox(a + (size_t)i * sa);
  const RBox bb = make_rbox(b + (size_t)i * sb);
  float r = 0.f;
  if (ba.rad >= 0.f && bb.rad >= 0.f) {
    const float dx = bb.cx - ba.cx, dy = bb.cy - ba.cy, R = (ba.rad + bb.rad) * 1.0001f;
    if (!(dx * dx + dy * dy > R * R) && !sat_disjoint(ba, bb)) r = iou_from_inter(ba, bb, clamp_integral_area(ba, bb), mode);
  }
  out[i] = r;
}

// ---------------------------------------------------------------------------------------------------------------
// Pairwise kernel, round 2.  A CTA owns a strip of CT = 128 columns (their derived data -- sincosf included -- is computed
// once) and walks ROW_TILES row tiles of RT = 32 rows; per 32 x 128 tile:
//   A1  bounding circles for all 4096 pairs with PACKED fp32x2 math, two rows per instruction: d^2 - R^2 from 7 packed
//       ops per 2 pairs, its sign bit shifted into a 16-bit pass mask by one funnel shift per pair (no compare, no
//       predicate) -- 5.5 instructions per pair (round 1: 23).  Survivors (~28 %) -> queue 1.
//   A2  separating axes on queue 1 in converged warps (branch-free, one comparison) -> queue 2 (~12 %).
//   B   clamp integral (riou_area.cuh, ~140 instructions, round 1: ~350) on queue 2 -> output tile in shared memory.
//   W   the tile goes out with 128-bit streaming stores and is re-zeroed in the same pass; warp 0 derives the next row
//       tile's boxes meanwhile.
// Invalid boxes (non-finite or zero area: IoU 0 with everything, utils/utils.py:669-673) are moved to x = +-1e18 so that the
// circle test rejects them without a flag.
// ---------------------------------------------------------------------------------------------------------------
constexpr int ROW_TILES = 8;

struct RiouSmem {
  float4 col0[CT], col1[CT];   // (cx, cy, 1.0001 rad, area), (c, s, hw, hh)
  float4 row0[RT], row1[RT];
  float4 rnxy[RT / 2];         // (-x[2j], -x[2j+1], -y[2j], -y[2j+1])
  float4 rrr[RT / 2];          // (R[2j], R[2j+1], -R[2j], -R[2j+1]),  R = 1.0001 rad
  float out[RT * CT];
  unsigned short q1[RT * CT];
  unsigned short q2[RT * CT];
  int cnt1, cnt2;
};

constexpr float FAR_AWAY = 1e18f;

// row boxes (far > 0) are the frame of the clamp integral: canonical_frame, once per box.  SAT and envelope only see the
// same rectangle.
__device__ __forceinline__ void derive_box(const float* __restrict__ p, bool in_range, float far, float4& d0, float4& d1) {
  RBox bx;
  bool live = false;
  if (in_range) {
    bx = make_rbox(p);
    live = bx.rad >= 0.f;
    if (far > 0.f) canonical_frame(bx.c, bx.s, bx.hw, bx.hh);
  }
  if (live) {
    d0 = make_float4(bx.cx, bx.cy, bx.rad * 1.0001f, bx.area);
    d1 = make_float4(bx.c, bx.s, bx.hw, bx.hh);
  } else {
    d0 = make_float4(far, 0.f, 0.f, 0.f);
    d1 = make_float4(1.f, 0.f, 0.f, 0.f);
  }
}

// stage A1 for one pair, lane for lane the packed arithmetic of the pairwise kernel: true when the bounding circles of row
// box r and column box c may overlap (sign of d^2 - R^2)
__device__ __forceinline__ bool circle_overlap(const float4& r0, const float4& c0) {
  const float dx = __fadd_rn(c0.x, -r0.x), dy = __fadd_rn(c0.y, -r0.y);
  const float R = __fadd_rn(c0.z, r0.z), Rn = __fadd_rn(-c0.z, -r0.z);
  float s = __fmul_rn(dy, dy);
  s = __fmaf_rn(dx, dx, s);
  s = __fmaf_rn(R, Rn, s);
  return (__float_as_uint(s) >> 31) != 0u;
}

// stage A2 for one pair: false when some box axis separates the boxes (branch-free, one comparison)
__device__ __forceinline__ bool sat_overlap(const float4& a0, const float4& a1, const float4& b0, const float4& b1) {
  const float dx = b0.x - a0.x, dy = b0.y - a0.y;
  const float rx = fmaf(dx, a1.x, dy * a1.y), ry = fmaf(dy, a1.x, -dx * a1.y);      // offset in a's frame
  const float cd = fmaf(a1.x, b1.x, a1.y * b1.y), sd = fmaf(a1.x, b1.y, -a1.y * b1.x);
  const float px = fmaf(rx, cd, ry * sd), py = fmaf(ry, cd, -rx * sd);              // offset in b's frame
  const float C = fabsf(cd), S = fabsf(sd);
  const float k = -1.0001f;      // tiny relative slack: touching boxes go on to the integral
  const float m1 = fmaf(k, fmaf(b1.w, S, fmaf(b1.z, C, a1.z)), fabsf(rx));
  const float m2 = fmaf(k, fmaf(b1.w, C, fmaf(b1.z, S, a1.w)), fabsf(ry));
  const float m3 = fmaf(k, fmaf(a1.w, S, fmaf(a1.z, C, b1.z)), fabsf(px));
  const float m4 = fmaf(k, fmaf(a1.w, C, fmaf(a1.z, S, b1.w)), fabsf(py));
  const float worst = fmaxf(fmaxf(m1, m2), fmaxf(m3, m4));      // > 0: separated on some axis
  return !(worst > 0.f);
}

// stage B for one pair that passed A1 and A2: the clamp integral (riou_area.cuh) and the IoU
__device__ __forceinline__ float pair_iou(const float4& a0, const float4& a1, const float4& b0, const float4& b1, int mode) {
  float inter = clamp_integral_area2(a0.x, a0.y, a1.x, a1.y, a1.z, a1.w, b0.x, b0.y, b1.x, b1.y, b1.z, b1.w);
  inter = fminf(inter, fminf(a0.w, b0.w));
  float uni = a0.w + b0.w - inter;
  if (mode == RYOLO_IOU_MODE_GIOU) {
    RBox ra, rb;
    ra.cx = a0.x; ra.cy = a0.y; ra.c = a1.x; ra.s = a1.y; ra.hw = a1.z; ra.hh = a1.w;
    rb.cx = b0.x; rb.cy = b0.y; rb.c = b1.x; rb.s = b1.y; rb.hw = b1.z; rb.hh = b1.w;
    uni = envelope_area(ra, rb);
  }
  return uni == 0.f ? 0.f : inter / uni;   // union == 0 -> 0 (utils/utils.py:693-694)
}

__device__ __forceinline__ void store_row(RiouSmem& sm, int t, const float4& d0, const float4& d1) {
  sm.row0[t] = d0;
  sm.row1[t] = d1;
  float* nxy = reinterpret_cast<float*>(sm.rnxy) + (t >> 1) * 4 + (t & 1);
  nxy[0] = -d0.x;
  nxy[2] = -d0.y;
  float* rr = reinterpret_cast<float*>(sm.rrr) + (t >> 1) * 4 + (t & 1);
  rr[0] = d0.z;
  rr[2] = -d0.z;
}

__global__ void __launch_bounds__(RIOU_THREADS, 4) riou_pairwise_kernel(const float* __restrict__ a, int n, int sa,
                                                                        const float* __restrict__ b, int m, int sb,
                                                                        int mode, float* __restrict__ out) {
  __shared__ RiouSmem sm;
  const int tid = threadIdx.x, lane = tid & 31;
  const int c0 = blockIdx.x * CT;
  const int tile0 = blockIdx.y * ROW_TILES;
  const int n_tiles = min(ROW_TILES, (n + RT - 1) / RT - tile0);

  if (tid < RT) {
    float4 d0, d1;
    const int r = tile0 * RT + tid;
    derive_box(a + (size_t)r * sa, r < n, FAR_AWAY, d0, d1);
    store_row(sm, tid, d0, d1);
  } else if (tid >= 64 && tid < 64 + CT) {
    const int j = tid - 64;
    float4 d0, d1;
    derive_box(b + (size_t)(c0 + j) * sb, c0 + j < m, -FAR_AWAY, d0, d1);
    sm.col0[j] = d0;
    sm.col1[j] = d1;
  }
  if (tid == 0) { sm.cnt1 = 0; sm.cnt2 = 0; }
  {  // zero the output tile once; the write-back pass re-zeroes what it reads
    float4* o4 = reinterpret_cast<float4*>(sm.out);
#pragma unroll
    for (int e = 0; e < (RT * CT / 4) / RIOU_THREADS; e++) o4[tid + e * RIOU_THREADS] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  __syncthreads();

  const int cols = min(CT, m - c0);
  const bool vec_store = (m & 3) == 0 && cols == CT && (reinterpret_cast<uintptr_t>(out) & 15) == 0;

#pragma unroll 1
  for (int t = 0; t < n_tiles; t++) {
    const int r0 = (tile0 + t) * RT;
    // ---- stage A1: bounding circles; thread = one column x 16 rows, two rows per packed instruction ----
    {
      const int c = tid & (CT - 1);
      const int rg = tid >> 7;
      const float4 cb = sm.col0[c];
      const uint64_t cx2 = f2pack(cb.x, cb.x), cy2 = f2pack(cb.y, cb.y), cr2 = f2pack(cb.z, cb.z), crn2 = f2pack(-cb.z, -cb.z);
      unsigned pass = 0;
#pragma unroll
      for (int j = 0; j < RT / 4; j++) {
        const float4 xy = sm.rnxy[rg * (RT / 4) + j];   // broadcast
        const float4 rr = sm.rrr[rg * (RT / 4) + j];
        const uint64_t dx = f2add(cx2, f2pack(xy.x, xy.y));
        const uint64_t dy = f2add(cy2, f2pack(xy.z, xy.w));
        const uint64_t R = f2add(cr2, f2pack(rr.x, rr.y));
        const uint64_t Rn = f2add(crn2, f2pack(rr.z, rr.w));
        uint64_t s = f2mul(dy, dy);
        s = f2fma(dx, dx, s);
        s = f2fma(R, Rn, s);       // d^2 - R^2 : negative <=> the circles overlap
        float s0, s1;
        f2unpack(s, s0, s1);
        pass = __funnelshift_l(__float_as_uint(s0), pass, 1);
        pass = __funnelshift_l(__float_as_uint(s1), pass, 1);
      }
      // row k of this thread's 16 sits in bit 15 - k.  One compaction per thread: warp scan of the counts, one atomic
      const int cnt = __popc(pass);
      int incl = cnt;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
      }
      int base = 0;
      if (lane == 31) base = atomicAdd(&sm.cnt1, incl);
      base = __shfl_sync(0xffffffffu, base, 31) + incl - cnt;
      const int row_hi = rg * (RT / 2) + 15;
      while (pass) {
        const int bp = 31 - __clz(pass);
        pass ^= 1u << bp;
        sm.q1[base++] = (unsigned short)(((row_hi - bp) << 7) | c);
      }
      if (tid == 0) sm.cnt2 = 0;
    }
    __syncthreads();
    // ---- stage A2: separating axes on queue 1 (converged warps, branch-free); ONE compaction per thread ----
    {
      const int cnt1 = sm.cnt1;
      unsigned kept = 0;               // bit i: my entry of round i (queue index i * 256 + tid) survives
#pragma unroll 1
      for (int q = tid, round = 0; q < cnt1; q += RIOU_THREADS, round++) {
        const int e = sm.q1[q];
        const float4 a0 = sm.row0[e >> 7], a1 = sm.row1[e >> 7], b0 = sm.col0[e & (CT - 1)], b1 = sm.col1[e & (CT - 1)];
        kept |= (sat_overlap(a0, a1, b0, b1) ? 1u : 0u) << round;
      }
      const int cnt = __popc(kept);
      int incl = cnt;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
      }
      int base = 0;
      if (lane == 31 && incl) base = atomicAdd(&sm.cnt2, incl);
      base = __shfl_sync(0xffffffffu, base, 31) + incl - cnt;
      while (kept) {
        const int round = __ffs(kept) - 1;
        kept &= kept - 1;
        sm.q2[base++] = sm.q1[round * RIOU_THREADS + tid];
      }
    }
    __syncthreads();
    // ---- stage B: clamp integral on queue 2 ----
    {
      const int cnt2 = sm.cnt2;
      if (tid == 0) sm.cnt1 = 0;      // queue 1 is consumed
      for (int q = tid; q < cnt2; q += RIOU_THREADS) {
        const int e = sm.q2[q];
        const int r = e >> 7, c = e & (CT - 1);
        sm.out[r * CT + c] = pair_iou(sm.row0[r], sm.row1[r], sm.col0[c], sm.col1[c], mode);
      }
    }
    __syncthreads();
    // ---- write back (and re-zero); warp 0 first derives the next row tile ----
    if (tid < RT && t + 1 < n_tiles) {
      float4 d0, d1;
      const int r = r0 + RT + tid;
      derive_box(a + (size_t)r * sa, r < n, FAR_AWAY, d0, d1);
      store_row(sm, tid, d0, d1);
    }
    const int rows = min(RT, n - r0);
    if (vec_store) {
      // thread = (row tid/32 + 8k, columns 4*(tid%32) ..): one LDS.128 + STS.128 + STG.128 per 4 pairs
      const int c4 = tid & 31;
      float4* src = reinterpret_cast<float4*>(sm.out) + tid;
      float4* dst = reinterpret_cast<float4*>(out + (size_t)(r0 + (tid >> 5)) * m + c0) + c4;
      const size_t dstep = (size_t)(RIOU_THREADS / 32) * m / 4;
#pragma unroll
      for (int k = 0; k < RT / (RIOU_THREADS / 32); k++) {
        if ((tid >> 5) + k * (RIOU_THREADS / 32) < rows) {
          const float4 v = src[k * RIOU_THREADS];
          src[k * RIOU_THREADS] = make_float4(0.f, 0.f, 0.f, 0.f);
          __stcs(dst + k * dstep, v);        // streaming: the matrix is written once and not re-read by this kernel
        }
      }
    } else {
      for (int e = tid; e < rows * CT; e += RIOU_THREADS) {
        const int r = e / CT, c = e % CT;
        const float v = sm.out[r * CT + c];
        sm.out[r * CT + c] = 0.f;
        if (c < cols) out[(size_t)(r0 + r) * m + c0 + c] = v;
      }
    }
    __syncthreads();
  }
}

// The same-image (prediction, target) pairs of an evaluation batch in one launch (ryolo_match_batched).  pbox [batch*cap, 5]:
// image b's num_keep[b] predictions from row b*cap; tbox [*, 5]: the targets grouped by image, image b's from row
// tstart[b] to tstart[b+1], timg = image of each grouped row.  Image b's matrix is written row-major at
// iou + cap * tstart[b] (row stride t_b), so the buffer holds cap * nt values whatever the split of the targets.  Each
// value is the pairwise kernel's for the same boxes, bit for bit: the same derived boxes and the same three stages.
__global__ void __launch_bounds__(256) riou_image_pairs_kernel(const float* __restrict__ pbox, int cap,
                                                               const int* __restrict__ num_keep,
                                                               const float* __restrict__ tbox,
                                                               const int* __restrict__ timg,
                                                               const int* __restrict__ tstart, int batch,
                                                               float* __restrict__ iou) {
  const long long total = (long long)cap * tstart[batch];
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int b = timg[e / cap];
    const int t0 = tstart[b], t = tstart[b + 1] - t0;
    const long long local = e - (long long)cap * t0;
    const int i = (int)(local / t), j = (int)(local - (long long)i * t);
    if (i >= num_keep[b]) continue;
    float4 r0, r1, c0, c1;
    derive_box(pbox + ((size_t)b * cap + i) * 5, true, FAR_AWAY, r0, r1);
    derive_box(tbox + (size_t)(t0 + j) * 5, true, -FAR_AWAY, c0, c1);
    float v = 0.f;
    if (circle_overlap(r0, c0) && sat_overlap(r0, r1, c0, c1)) v = pair_iou(r0, r1, c0, c1, RYOLO_IOU_MODE_IOU);
    iou[e] = v;
  }
}

int launch_riou_image_pairs(const float* pbox, int cap, const int* num_keep, const float* tbox, const int* timg,
                            const int* tstart, int batch, int nt, float* iou, cudaStream_t stream) {
  const long long blocks = ((long long)cap * nt + 255) / 256, limit = (long long)device_sm_count() * 16;
  if (blocks == 0) return RYOLO_OK;
  riou_image_pairs_kernel<<<(unsigned)(blocks < limit ? blocks : limit), 256, 0, stream>>>(pbox, cap, num_keep, tbox, timg,
                                                                                         tstart, batch, iou);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

}  // namespace ryolo

using namespace ryolo;

extern "C" int ryolo_riou_paired(const float* a, const float* b, int n, int stride_a, int stride_b, int mode, float* out,
                                 void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(n >= 0 && stride_a >= 5 && stride_b >= 5);
  RYOLO_ARG_CHECK(mode == RYOLO_IOU_MODE_IOU || mode == RYOLO_IOU_MODE_GIOU);
  if (n == 0) return RYOLO_OK;
  RYOLO_ARG_CHECK(a && b && out);
  riou_paired_kernel<<<(n + 255) / 256, 256, 0, stream>>>(a, b, n, stride_a, stride_b, mode, out);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_riou_pairwise(const float* a, int n, int stride_a, const float* b, int m, int stride_b, int mode,
                                   float* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(n >= 0 && m >= 0 && stride_a >= 5 && stride_b >= 5);
  RYOLO_ARG_CHECK(mode == RYOLO_IOU_MODE_IOU || mode == RYOLO_IOU_MODE_GIOU);
  if (n == 0 || m == 0) return RYOLO_OK;
  RYOLO_ARG_CHECK(a && b && out);
  dim3 grid((m + CT - 1) / CT, ((n + RT - 1) / RT + ROW_TILES - 1) / ROW_TILES);
  RYOLO_ARG_CHECK(grid.y <= 65535);
  riou_pairwise_kernel<<<grid, RIOU_THREADS, 0, stream>>>(a, n, stride_a, b, m, stride_b, mode, out);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}
