// TMA-fed versions of the three read-limited BN / PReLU passes: statistics, backward reduce, backward apply (included by
// bnact.cu; same arithmetic, same results).
//
// Work split: the grid of <= 2 x SMs persistent CTAs strides over the row pieces together (piece = blockIdx + k * gridDim), so
// the whole grid reads one moving front of the tensor.
// Why: the direct versions keep ONE 16-byte load in flight per thread; at the 50-70 % occupancy their register budgets
// allow that is ~23 KB in flight per SM, less than Little's law (HBM bandwidth x latency) asks for to saturate HBM, and
// unrolling for more loads per thread costs occupancy.  Here the bytes in flight are decoupled from the thread count: an interior row of
// the padded-NHWC tensor is contiguous (w x c bf16 when the channel stride equals c, true for every z / dz buffer), so a
// CTA takes row PIECES (<= 20 KB) grid-stride, one elected thread issues `cp.async.bulk` (1-D TMA) copies of
// the next pieces into a ring of shared-memory stages, completion on an mbarrier, and the 256 threads consume a stage
// with LDS.128 -- 2 CTAs x 80 KB of stages per SM.  Stores go straight from registers (coalesced 16 B).
#pragma once

namespace ryolo {

constexpr int PIPE_ITEMS = 1280;                    // 16-byte items per stage (20 KB)
constexpr int PIPE_STAGE_BYTES = PIPE_ITEMS * 16;

struct PieceGeo {
  int ppr;       // pieces per interior row
  int px;        // pixels per piece (the last piece of a row may be shorter)
  int total;     // pieces in the tensor
  int per_cta;   // pieces per CTA (grid = ceil(total / per_cta); the CTAs stride over the pieces together)
  int rev;       // 1: the grid walks the tensor from the END (see "Traversal order" below)
};

// Traversal order.  A pass over a tensor larger than the 50 MB L2 that runs in the same direction as the pass before it
// finds nothing of it in L2 (the lines it needs first were evicted first), while the opposite direction starts on the
// ~100 MB the previous kernel touched LAST.  The chain per layer is  conv (writes z ascending) -> statistics -> bn_act_fwd
// and  dgrad (writes dy ascending) -> reduce -> apply: statistics and reduce walk DESCENDING, bn_act_fwd and apply
// ascending, so every pass begins inside its predecessor's tail.

__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}

struct Piece {
  int b, y, x0, npx;
};
__device__ __forceinline__ Piece piece_at(const Geo& g, const PieceGeo& pg, int p) {
  Piece q;
  const int row = p / pg.ppr, j = p - row * pg.ppr;
  q.b = row / g.h;
  q.y = row - q.b * g.h;
  q.x0 = j * pg.px;
  q.npx = min(pg.px, g.w - q.x0);
  return q;
}

// K inputs per stage (each tensor with channel stride == c), NST stages.  Shared-memory layout: [NST][K][PIPE_ITEMS] uint4,
// then NST mbarriers.
template <int K, int NST>
struct RowPipe {
  uint32_t buf0, bar0;
  const uint4* gen;       // generic-address view of the stage ring
  int p_begin, p_end, rev;

  // ring slot p (0 <= p < p_end, consumed in increasing order) -> piece of the tensor: the grid strides over the pieces
  // together, ascending or descending, so that the whole grid works on one moving front of the tensor
  int total;
  __device__ __forceinline__ int phys(int p) const {
    const int k = blockIdx.x + p * gridDim.x;
    return rev ? total - 1 - k : k;
  }

  __device__ __forceinline__ void init(unsigned char* smem, const PieceGeo& pg) {
    buf0 = (uint32_t)__cvta_generic_to_shared(smem);
    bar0 = buf0 + NST * K * PIPE_STAGE_BYTES;
    gen = reinterpret_cast<const uint4*>(smem);
    rev = pg.rev;
    total = pg.total;
    p_begin = 0;
    p_end = (int)blockIdx.x < pg.total ? (pg.total - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    if (threadIdx.x == 0) {
#pragma unroll
      for (int s = 0; s < NST; s++) mbar_init(bar0 + 8u * s, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
  }
  static constexpr size_t smem_bytes() { return (size_t)NST * K * PIPE_STAGE_BYTES + 8 * NST; }

  // thread 0 only
  __device__ __forceinline__ void issue(const Geo& g, const PieceGeo& pg, int p, const __nv_bfloat16* const* src) {
    const int s = (p - p_begin) % NST;
    const Piece q = piece_at(g, pg, phys(p));
    const uint32_t bytes = (uint32_t)q.npx * g.c * 2;
    const size_t off = pad_off(q.b, q.y, q.x0, g.h, g.w, g.c);
    mbar_expect_tx(bar0 + 8u * s, bytes * K);
#pragma unroll
    for (int k = 0; k < K; k++) bulk_g2s(buf0 + (s * K + k) * PIPE_STAGE_BYTES, src[k] + off, bytes, bar0 + 8u * s);
  }
  __device__ __forceinline__ void prologue(const Geo& g, const PieceGeo& pg, const __nv_bfloat16* const* src) {
    if (threadIdx.x == 0)
      for (int s = 0; s < NST && p_begin + s < p_end; s++) issue(g, pg, p_begin + s, src);
  }
  __device__ __forceinline__ const uint4* wait(int p, int k) const {
    const int it = p - p_begin, s = it % NST;
    mbar_wait(bar0 + 8u * s, (uint32_t)(it / NST) & 1u);
    return gen + (size_t)(s * K + k) * PIPE_ITEMS;
  }
  // every thread has finished reading piece p's stage: refill it with piece p + NST
  __device__ __forceinline__ void release(const Geo& g, const PieceGeo& pg, int p, const __nv_bfloat16* const* src) {
    __syncthreads();
    if (threadIdx.x == 0 && p + NST < p_end) issue(g, pg, p + NST, src);
  }
};

// ---------------------------------------------------------------------------------------------------------------
// BN finalisation, fused into the reduction of the statistics' partial rows (bn_sums_reduce_kernel)
struct BnFinalize {
  const float *gamma, *beta;        // gamma == nullptr: statistics only
  float *mean, *invstd, *scale, *shift, *running_mean, *running_var;
  float count, eps, momentum;
};
__device__ __forceinline__ void bn_finalize_channel(const BnFinalize& f, int c, int ch, float s1, float s2) {
  const float mean = s1 / f.count;
  const float var = fmaxf(s2 / f.count - mean * mean, 0.f);
  const float invstd = rsqrtf(var + f.eps);
  const float sc = f.gamma[ch] * invstd;
  f.mean[ch] = mean;
  f.invstd[ch] = invstd;
  f.scale[ch] = sc;
  f.shift[ch] = f.beta[ch] - mean * sc;
  if (f.running_mean) {
    f.running_mean[ch] = (1.f - f.momentum) * f.running_mean[ch] + f.momentum * mean;
    f.running_var[ch] = (1.f - f.momentum) * f.running_var[ch] + f.momentum * var * (f.count / fmaxf(f.count - 1.f, 1.f));
  }
}

// sums[j] and sums[c + j] (and sums[2c] for has_extra) = the rows of `partials` [rows][2c (+1)] added in a fixed order:
// thread (column j, part q) adds rows q, q + 8, q + 16, ...; the 8 parts are then added in order.  CTA = 32 columns;
// with has_extra one more CTA takes sums[2c].  fin.gamma: finalise the batch statistics of channel j as well.
constexpr int kReduceParts = 8;
__global__ void __launch_bounds__(32 * kReduceParts) bn_sums_reduce_kernel(const float* __restrict__ partials, int rows, int c,
                                                                          int has_extra, float* __restrict__ sums,
                                                                          BnFinalize fin) {
  __shared__ float s_part[2][kReduceParts][32];
  const int n = 2 * c + has_extra, lane = threadIdx.x & 31, q = threadIdx.x >> 5;
  const bool extra = has_extra && blockIdx.x == gridDim.x - 1;
  const int j = blockIdx.x * 32 + lane;
  const int i1 = extra ? 2 * c : j, i2 = extra ? 2 * c : c + j;
  const bool live = extra ? lane == 0 : j < c;
  float s1 = 0.f, s2 = 0.f;
  if (live) {
#pragma unroll 4
    for (int r = q; r < rows; r += kReduceParts) {
      s1 += __ldcg(partials + (size_t)r * n + i1);
      s2 += __ldcg(partials + (size_t)r * n + i2);
    }
  }
  s_part[0][q][lane] = s1;
  s_part[1][q][lane] = s2;
  __syncthreads();
  if (q != 0 || !live) return;
  float t1 = 0.f, t2 = 0.f;
#pragma unroll
  for (int k = 0; k < kReduceParts; k++) {
    t1 += s_part[0][k][lane];
    t2 += s_part[1][k][lane];
  }
  if (extra) {
    sums[2 * c] = t1;
    return;
  }
  sums[j] = t1;
  sums[c + j] = t2;
  if (fin.gamma) bn_finalize_channel(fin, c, j, t1, t2);
}

__global__ void __launch_bounds__(BNT, 2) bn_stats_pipe_kernel(const __nv_bfloat16* __restrict__ z, Geo g, PieceGeo pg,
                                                               float* __restrict__ partials /*[gridDim.x][2*c]*/) {
  extern __shared__ __align__(128) unsigned char dsm[];
  using Pipe = RowPipe<1, 4>;
  Pipe pipe;
  pipe.init(dsm, pg);
  float* s_acc = reinterpret_cast<float*>(dsm + Pipe::smem_bytes());   // [kAccFloats]
  __syncthreads();
  const __nv_bfloat16* src[1] = {z};
  pipe.prologue(g, pg, src);
  const RowSpan rs = row_span(g);
  uint64_t p1[4], p2[4];
#pragma unroll
  for (int e = 0; e < 4; e++) p1[e] = p2[e] = 0ull;
  for (int p = pipe.p_begin; p < pipe.p_end; p++) {
    const uint4* st = pipe.wait(p, 0);
    const Piece q = piece_at(g, pg, pipe.phys(p));
    const int items = q.npx << rs.cgs_log2;
    for (int i = threadIdx.x; i < items; i += BNT) {
      const uint4 v = st[i];
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 4; e++) {
        const uint64_t f2 = bf2_to_f2(w[e]);
        p1[e] = f2add(p1[e], f2);
        p2[e] = f2fma(f2, f2, p2[e]);
      }
    }
    pipe.release(g, pg, p, src);
  }
  float s1[8], s2[8];
#pragma unroll
  for (int e = 0; e < 4; e++) {
    f2unpack(p1[e], s1[2 * e], s1[2 * e + 1]);
    f2unpack(p2[e], s2[2 * e], s2[2 * e + 1]);
  }
  block_partials(rs, g.c, s1, s2, 0.f, false, s_acc, partials);
}

// ---------------------------------------------------------------------------------------------------------------
// Backward passes.  Where dy comes from:
//   DYP = 0  through load_dy (upsample adjoint, or a concat buffer with a wider channel stride): only z rides the pipe;
//   DYP = 1  a plain tensor with channel stride == c: rides the pipe next to z (stage = z piece + dy piece);
//   DYP = 2  the space-to-depth dgrad output of a following 3x3/stride-2 block (channel stride == 4c): ONE s2d row holds the
//            dy of TWO image rows, so a piece is a ROW PAIR: stage = z piece of row 2k, z piece of row 2k+1 (10 KB each) and
//            the matching run of the s2d row (20 KB, contiguous).  These are the three largest tensors of the network
//            (608^2 x 32, 304^2 x 64, 152^2 x 128); through load_dy they stay far below HBM bandwidth.
template <int DYP>
struct BwdPipe {
  static constexpr int NST = DYP == 0 ? 4 : 2;
  static constexpr int Z_ITEMS = DYP == 2 ? PIPE_ITEMS / 2 : PIPE_ITEMS;          // 16-byte items of one z piece
  static constexpr int STAGE_ITEMS = DYP == 0 ? PIPE_ITEMS : 2 * PIPE_ITEMS;
  static constexpr int ROWS = DYP == 2 ? 2 : 1;                                    // image rows per piece
  static constexpr size_t smem_bytes() { return (size_t)NST * STAGE_ITEMS * 16 + 8 * NST; }

  uint32_t buf0, bar0;
  const uint4* gen;
  int p_begin, p_end, rev, total;
  const __nv_bfloat16 *z, *dy;

  __device__ __forceinline__ void init(unsigned char* smem, const PieceGeo& pg, const __nv_bfloat16* z_,
                                       const __nv_bfloat16* dy_) {
    buf0 = (uint32_t)__cvta_generic_to_shared(smem);
    bar0 = buf0 + NST * STAGE_ITEMS * 16;
    gen = reinterpret_cast<const uint4*>(smem);
    z = z_;
    dy = dy_;
    rev = pg.rev;
    total = pg.total;
    p_begin = 0;
    p_end = (int)blockIdx.x < pg.total ? (pg.total - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    if (threadIdx.x == 0) {
#pragma unroll
      for (int s = 0; s < NST; s++) mbar_init(bar0 + 8u * s, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
  }
  // ring slot p -> (b, first image row, x0, npx); for DYP = 2 the piece index runs over row PAIRS
  __device__ __forceinline__ Piece piece(const Geo& g, const PieceGeo& pg, int p) const {
    Geo gg = g;
    gg.h = g.h / ROWS;
    const int k = blockIdx.x + p * gridDim.x;                          // grid-stride, see "Traversal order"
    Piece q = piece_at(gg, pg, rev ? total - 1 - k : k);
    q.y *= ROWS;
    return q;
  }
  __device__ __forceinline__ void issue(const Geo& g, const PieceGeo& pg, int p) {   // thread 0 only
    const int s = (p - p_begin) % NST;
    const Piece q = piece(g, pg, p);
    const uint32_t bytes = (uint32_t)q.npx * g.c * 2;
    const uint32_t st = buf0 + s * STAGE_ITEMS * 16, bar = bar0 + 8u * s;
    if (DYP == 0) {
      mbar_expect_tx(bar, bytes);
      bulk_g2s(st, z + pad_off(q.b, q.y, q.x0, g.h, g.w, g.c), bytes, bar);
    } else if (DYP == 1) {
      const size_t off = pad_off(q.b, q.y, q.x0, g.h, g.w, g.c);
      mbar_expect_tx(bar, 2 * bytes);
      bulk_g2s(st, z + off, bytes, bar);
      bulk_g2s(st + Z_ITEMS * 16, dy + off, bytes, bar);
    } else {
      mbar_expect_tx(bar, 4 * bytes);
      bulk_g2s(st, z + pad_off(q.b, q.y, q.x0, g.h, g.w, g.c), bytes, bar);
      bulk_g2s(st + Z_ITEMS * 16, z + pad_off(q.b, q.y + 1, q.x0, g.h, g.w, g.c), bytes, bar);
      bulk_g2s(st + 2 * Z_ITEMS * 16, dy + pad_off(q.b, q.y >> 1, q.x0 >> 1, g.h >> 1, g.w >> 1, 4 * g.c), 2 * bytes, bar);
    }
  }
  __device__ __forceinline__ void prologue(const Geo& g, const PieceGeo& pg) {
    if (threadIdx.x == 0)
      for (int s = 0; s < NST && p_begin + s < p_end; s++) issue(g, pg, p_begin + s);
  }
  __device__ __forceinline__ const uint4* wait(int p) const {
    const int it = p - p_begin, s = it % NST;
    mbar_wait(bar0 + 8u * s, (uint32_t)(it / NST) & 1u);
    return gen + (size_t)s * STAGE_ITEMS;
  }
  __device__ __forceinline__ void release(const Geo& g, const PieceGeo& pg, int p) {
    __syncthreads();
    if (threadIdx.x == 0 && p + NST < p_end) issue(g, pg, p + NST);
  }
  // dy of item i (pixel x0 + i / cgs, my channel group) of image row q.y + r, from the stage
  __device__ __forceinline__ uint4 dy_item(const uint4* st, int i, int r, const RowSpan& rs, int cgs) const {
    if (DYP == 1) return st[Z_ITEMS + i];
    // s2d row: pixel pair j = (x - x0) / 2 holds 4 * cgs items, quadrant (row & 1) * 2 + (x & 1)   (x0 is even)
    const int px = i >> rs.cgs_log2;
    return st[2 * Z_ITEMS + (((px >> 1) * 4 + r * 2 + (px & 1)) << rs.cgs_log2) + rs.cg];
  }
};

template <int DYP>
__global__ void __launch_bounds__(BNT, 2) bn_act_bwd_reduce_pipe_kernel(
    const __nv_bfloat16* __restrict__ dy, int dcs, int up, const __nv_bfloat16* __restrict__ z, Geo g, PieceGeo pg,
    const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ mean,
    const float* __restrict__ invstd, float slope, int has_act, float* __restrict__ partials /*[gridDim.x][2*c + 1]*/,
    const float* __restrict__ slope_dev) {
  extern __shared__ __align__(128) unsigned char dsm[];
  using Pipe = BwdPipe<DYP>;
  Pipe pipe;
  pipe.init(dsm, pg, z, dy);
  float* s_acc = reinterpret_cast<float*>(dsm + Pipe::smem_bytes());   // [kAccFloats]
  __syncthreads();
  pipe.prologue(g, pg);
  if (slope_dev) slope = __ldg(slope_dev);
  const RowSpan rs = row_span(g);
  const int cgs = g.c >> 3;
  float sc[8], sh[8], mu[8], is[8];
  load8(scale, rs.cg, sc);
  load8(shift, rs.cg, sh);
  load8(mean, rs.cg, mu);
  load8(invstd, rs.cg, is);
  float asl = 0.f;
  uint64_t sc2[4], sh2[4], nmu2[4], is2[4], q1[4], q2[4];
#pragma unroll
  for (int e = 0; e < 4; e++) {
    sc2[e] = f2pack(sc[2 * e], sc[2 * e + 1]);
    sh2[e] = f2pack(sh[2 * e], sh[2 * e + 1]);
    nmu2[e] = f2pack(-mu[2 * e], -mu[2 * e + 1]);
    is2[e] = f2pack(is[2 * e], is[2 * e + 1]);
    q1[e] = q2[e] = 0ull;
  }
  for (int p = pipe.p_begin; p < pipe.p_end; p++) {
    const Piece q = pipe.piece(g, pg, p);
    const uint4* st = pipe.wait(p);
    const int items = q.npx << rs.cgs_log2;
#pragma unroll
    for (int r = 0; r < Pipe::ROWS; r++) {
      const uint4* zs = st + r * Pipe::Z_ITEMS;
      for (int i = threadIdx.x; i < items; i += BNT) {
        const uint4 zv = zs[i];
        float d[8];
        if (DYP) unpack8(pipe.dy_item(st, i, r, rs, cgs), d);
        else load_dy(dy, dcs, g, q.b, q.y, q.x0 + (i >> rs.cgs_log2), rs.cg, up, d);
        const uint32_t zw[4] = {zv.x, zv.y, zv.z, zv.w};
#pragma unroll
        for (int e = 0; e < 4; e++) {
          const uint64_t f2 = bf2_to_f2(zw[e]);
          float u0, u1;
          f2unpack(f2fma(f2, sc2[e], sh2[e]), u0, u1);
          float du0 = d[2 * e], du1 = d[2 * e + 1];
          if (has_act) {
            if (!(u0 > 0.f)) { asl = fmaf(du0, u0, asl); du0 *= slope; }
            if (!(u1 > 0.f)) { asl = fmaf(du1, u1, asl); du1 *= slope; }
          }
          const uint64_t du2 = f2pack(du0, du1);
          const uint64_t zh2 = f2mul(f2add(f2, nmu2[e]), is2[e]);
          q1[e] = f2add(q1[e], du2);
          q2[e] = f2fma(du2, zh2, q2[e]);
        }
      }
    }
    pipe.release(g, pg, p);
  }
  float a1[8], a2[8];
#pragma unroll
  for (int e = 0; e < 4; e++) {
    f2unpack(q1[e], a1[2 * e], a1[2 * e + 1]);
    f2unpack(q2[e], a2[2 * e], a2[2 * e + 1]);
  }
  for (int o = 16; o > 0; o >>= 1) asl += __shfl_xor_sync(0xffffffffu, asl, o);
  block_partials(rs, g.c, a1, a2, asl, true, s_acc, partials);
}

template <int DYP>
__global__ void __launch_bounds__(BNT, 2) bn_act_bwd_apply_pipe_kernel(
    const __nv_bfloat16* __restrict__ dy, int dcs, int up, __nv_bfloat16* __restrict__ z /*in: z, out: dz*/, Geo g,
    PieceGeo pg, const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ mean,
    const float* __restrict__ invstd, float slope, int has_act, int has_bn, const float* __restrict__ sums, float inv_n,
    __nv_bfloat16* __restrict__ gres, int gcs, int gres_acc, const float* __restrict__ slope_dev) {
  extern __shared__ __align__(128) unsigned char dsm[];
  using Pipe = BwdPipe<DYP>;
  Pipe pipe;
  pipe.init(dsm, pg, z, dy);
  __syncthreads();
  pipe.prologue(g, pg);
  if (slope_dev) slope = __ldg(slope_dev);
  const RowSpan rs = row_span(g);
  const int cgs = g.c >> 3;
  float sc[8], sh[8], mu[8], is[8], m1[8], m2[8];
  load8(scale, rs.cg, sc);
  load8(shift, rs.cg, sh);
  load8(mean, rs.cg, mu);
  load8(invstd, rs.cg, is);
  load8(sums, rs.cg, m1);
  load8(sums + g.c, rs.cg, m2);
  uint64_t sc2[4], sh2[4], nmu2[4], is2[4], nm12[4], nm22[4];
#pragma unroll
  for (int e = 0; e < 4; e++) {
    sc2[e] = f2pack(sc[2 * e], sc[2 * e + 1]);
    sh2[e] = f2pack(sh[2 * e], sh[2 * e + 1]);
    nmu2[e] = f2pack(-mu[2 * e], -mu[2 * e + 1]);
    is2[e] = f2pack(is[2 * e], is[2 * e + 1]);
    nm12[e] = f2pack(-m1[2 * e] * inv_n, -m1[2 * e + 1] * inv_n);
    nm22[e] = f2pack(-m2[2 * e] * inv_n, -m2[2 * e + 1] * inv_n);
  }
  for (int p = pipe.p_begin; p < pipe.p_end; p++) {
    const Piece q = pipe.piece(g, pg, p);
    const uint4* st = pipe.wait(p);
    const int items = q.npx << rs.cgs_log2;
#pragma unroll
    for (int r = 0; r < Pipe::ROWS; r++) {
      const int b = q.b, y = q.y + r;
      __nv_bfloat16* zr = z + pad_off(b, y, 0, g.h, g.w, g.c) + rs.cg * 8;
      __nv_bfloat16* gr = gres ? gres + pad_off(b, y, 0, g.h, g.w, gcs) + rs.cg * 8 : nullptr;
      const uint4* zs = st + r * Pipe::Z_ITEMS;
      for (int i = threadIdx.x; i < items; i += BNT) {
        const int x = q.x0 + (i >> rs.cgs_log2);
        const uint4 zv = zs[i];
        float d[8];
        if (DYP) unpack8(pipe.dy_item(st, i, r, rs, cgs), d);
        else load_dy(dy, dcs, g, b, y, x, rs.cg, up, d);
        if (gr) {  // shortcut branch: d(residual) (+)= dy   (never combined with upsample)
          float o[8];
          if (gres_acc) {
            unpack8(*reinterpret_cast<const uint4*>(gr + (size_t)x * gcs), o);
#pragma unroll
            for (int e = 0; e < 8; e++) o[e] += d[e];
          } else {
#pragma unroll
            for (int e = 0; e < 8; e++) o[e] = d[e];
          }
          *reinterpret_cast<uint4*>(gr + (size_t)x * gcs) = pack8(o);
        }
        float out[8];
        const uint32_t zw[4] = {zv.x, zv.y, zv.z, zv.w};
#pragma unroll
        for (int e = 0; e < 4; e++) {
          const uint64_t f2 = bf2_to_f2(zw[e]);
          float u0, u1;
          f2unpack(f2fma(f2, sc2[e], sh2[e]), u0, u1);
          float du0 = d[2 * e], du1 = d[2 * e + 1];
          if (has_act) {
            if (!(u0 > 0.f)) du0 *= slope;
            if (!(u1 > 0.f)) du1 *= slope;
          }
          if (has_bn) {
            const uint64_t zh2 = f2mul(f2add(f2, nmu2[e]), is2[e]);
            const uint64_t t2 = f2fma(zh2, nm22[e], f2add(f2pack(du0, du1), nm12[e]));
            f2unpack(f2mul(sc2[e], t2), out[2 * e], out[2 * e + 1]);
          } else {
            out[2 * e] = du0;
            out[2 * e + 1] = du1;
          }
        }
        *reinterpret_cast<uint4*>(zr + (size_t)x * g.c) = pack8(out);
      }
    }
    pipe.release(g, pg, p);
  }
}

// host side ------------------------------------------------------------------------------------------------------
// The pipe needs the rows of the tensor to be contiguous (channel stride == c) and 256 threads to tile the channel groups.
// Only the read-limited passes (statistics, the backward pair) take it: the forward pass is write-limited, so its direct
// version gains nothing from the pipe.
static inline bool pipe_ok(const Geo& g, int cstride) { return cstride == g.c && (g.c >> 3) <= BNT; }
// rows_per_piece = 2: row pairs with even piece boundaries and half-size z pieces (BwdPipe<2>)
static inline PieceGeo mk_pieces(const Geo& g, int* grid, int rows_per_piece = 1) {
  PieceGeo pg;
  const int cgs = g.c >> 3;
  int max_px = PIPE_ITEMS / rows_per_piece / cgs;      // >= 10 for c <= 1024
  if (rows_per_piece == 2) max_px &= ~1;
  pg.ppr = (g.w + max_px - 1) / max_px;
  pg.px = (g.w + pg.ppr - 1) / pg.ppr;
  if (rows_per_piece == 2 && (pg.px & 1)) pg.px++;
  pg.total = g.batch * (g.h / rows_per_piece) * pg.ppr;
  const int ctas = 2 * device_sm_count();
  pg.per_cta = (pg.total + ctas - 1) / ctas;
  pg.rev = 0;
  *grid = (pg.total + pg.per_cta - 1) / pg.per_cta;
  return pg;
}

}  // namespace ryolo
