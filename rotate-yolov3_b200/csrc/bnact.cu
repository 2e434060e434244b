// Training-mode BatchNorm2d + PReLU (+ shortcut add, + nearest x2 upsample) around the wgmma convolutions, forward
// and backward, on padded-NHWC bf16 activations.  Reference semantics: nn.BatchNorm2d(momentum=0.1, eps=1e-5) with
// batch statistics -> nn.PReLU(num_parameters=1) (model/models.py:62-65), shortcut add (models.py:281-282), nn.Upsample
// nearest x2 (models.py:93-94), differentiated by autograd (train.py:278-282).
//
// Memory-bound passes, 16-byte (8-channel) accesses, channels innermost:
//   bn_stats          z -> per-channel sum, sum of squares                      (1 read)
//   bn_act_fwd        y = prelu(z*scale + shift) [+ res], optional 2x2 replicated store      (1 read [+1], 1 write)
//   bn_act_bwd_reduce dy, z -> per-channel sum(du), sum(du * zhat), scalar d(slope)            (2 reads)
//   bn_act_bwd_apply  dz = scale*(du - mean(du) - zhat*mean(du*zhat)) written over z; dres (+)= dy   (2 reads, 1-2 writes)
// plus the small layout kernels of the training graph (zero insertion for stride-2 adjoints, im2col of the 3-channel
// image so that the first layer runs on the same GEMMs).
#include <cuda_bf16.h>

#include "common.cuh"
#include "f32x2.cuh"
#include "sm90.cuh"

namespace ryolo {

__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int e = 0; e < 4; e++) {
    const float2 t = __bfloat1622float2(h[e]);
    f[2 * e] = t.x;
    f[2 * e + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  __nv_bfloat162 h[4];
#pragma unroll
  for (int e = 0; e < 4; e++) h[e] = __floats2bfloat162_rn(f[2 * e], f[2 * e + 1]);
  return *reinterpret_cast<uint4*>(h);
}

struct Geo {
  int batch, h, w, c;   // interior size, real channels (multiple of 8; c/8 is a power of two for every Darknet width)
};

// generic thread -> (interior pixel, 8-channel group) decode for the small layout kernels below
__device__ __forceinline__ bool decode_item(const Geo& g, size_t item, int& b, int& y, int& x, int& cg) {
  const int cgs = g.c >> 3;
  const size_t npix = (size_t)g.batch * g.h * g.w;
  if (item >= npix * cgs) return false;
  cg = (int)(item % cgs);
  const size_t pix = item / cgs;
  x = (int)(pix % g.w);
  y = (int)((pix / g.w) % g.h);
  b = (int)(pix / ((size_t)g.w * g.h));
  return true;
}
__device__ __forceinline__ size_t pad_off(int b, int y, int x, int h, int w, int cs) {  // element offset of padded pixel
  return (((size_t)b * (h + 2) + y + 1) * (w + 2) + x + 1) * cs;
}

// The four BN/PReLU kernels share one work decomposition: a CTA owns a contiguous span of interior ROWS (b, y);
// thread t owns channel group (t mod cgs) for the whole kernel -- its 8 scale/shift/mean/invstd values live in
// registers -- and walks the pixels of the span with stride blockDim/cgs.  No integer division in the inner loop
// (cgs is a power of two), 16-byte accesses, consecutive threads on consecutive channel groups of the same pixel.
constexpr int BNT = 256;

struct RowSpan {
  int cg, cgs_log2, px0, pstep;   // my channel group, log2(cgs), first pixel index within a row, pixel stride
};
__device__ __forceinline__ RowSpan row_span(const Geo& g) {
  RowSpan r;
  const int cgs = g.c >> 3;
  r.cgs_log2 = 31 - __clz(cgs);
  r.cg = threadIdx.x & (cgs - 1);
  r.px0 = threadIdx.x >> r.cgs_log2;
  r.pstep = BNT >> r.cgs_log2;
  return r;
}
__device__ __forceinline__ void load8(const float* __restrict__ p, int cg, float* o) {
  const float4 a = *reinterpret_cast<const float4*>(p + cg * 8), b = *reinterpret_cast<const float4*>(p + cg * 8 + 4);
  o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
}

// Per-channel sums are reduced in a FIXED order, so that a training step computes the same numbers every run: float
// atomics (shared or global) would add the contributions in arrival order, and train-mode BatchNorm amplifies the
// last-bit differences through the network.  Each CTA stages its threads' 8 + 8 channel values in shared memory, adds
// the threads of one channel in thread order and writes ONE partial row [2c (+1)] to `partials`; bn_sums_reduce_kernel
// then adds the rows of all CTAs in a fixed partition and order.
constexpr int kAccFloats = 16 * BNT + BNT / 32;   // shared staging of block_partials (>= 2 * 2048 + 1 floats)
constexpr size_t kAccBytes = kAccFloats * sizeof(float);
__device__ __forceinline__ void block_partials(const RowSpan& rs, int c, const float (&v1)[8], const float (&v2)[8],
                                               float warp_extra, bool has_extra, float* s_buf, float* __restrict__ partials) {
  const int n = 2 * c + (has_extra ? 1 : 0);
  __syncthreads();
#pragma unroll
  for (int e = 0; e < 8; e++) {
    s_buf[e * BNT + threadIdx.x] = v1[e];
    s_buf[(8 + e) * BNT + threadIdx.x] = v2[e];
  }
  if (has_extra && (threadIdx.x & 31) == 0) s_buf[16 * BNT + (threadIdx.x >> 5)] = warp_extra;
  __syncthreads();
  const int cgs = c >> 3;
  float* row = partials + (size_t)blockIdx.x * n;
  for (int i = threadIdx.x; i < n; i += BNT) {
    float s = 0.f;
    if (i < 2 * c) {
      const int ch = i < c ? i : i - c, e = (ch & 7) + (i < c ? 0 : 8), cg = ch >> 3;
      for (int k = 0; k < rs.pstep; k++) s += s_buf[e * BNT + cg + k * cgs];
    } else {
      for (int wi = 0; wi < BNT / 32; wi++) s += s_buf[16 * BNT + wi];
    }
    row[i] = s;
  }
}

// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(BNT) bn_stats_kernel(const __nv_bfloat16* __restrict__ z, int zcs, Geo g,
                                                       float* __restrict__ partials /*[gridDim.x][2*c]*/,
                                                       int rows_per_block) {
  extern __shared__ float s_acc[];  // [kAccFloats]
  const RowSpan rs = row_span(g);
  const int nrows = g.batch * g.h;
  const int row_begin = blockIdx.x * rows_per_block, row_end = min(nrows, row_begin + rows_per_block);
  // packed fp32x2 accumulators: 16 instructions per 16-byte load instead of 24
  uint64_t p1[4], p2[4];
#pragma unroll
  for (int e = 0; e < 4; e++) p1[e] = p2[e] = 0ull;
  for (int row = row_begin; row < row_end; row++) {
    const int b = row / g.h, y = row - b * g.h;
    const __nv_bfloat16* zr = z + pad_off(b, y, 0, g.h, g.w, zcs) + rs.cg * 8;
    for (int x = rs.px0; x < g.w; x += rs.pstep) {
      const uint4 v = *reinterpret_cast<const uint4*>(zr + (size_t)x * zcs);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 4; e++) {
        const uint64_t f2 = bf2_to_f2(w[e]);
        p1[e] = f2add(p1[e], f2);
        p2[e] = f2fma(f2, f2, p2[e]);
      }
    }
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
__global__ void __launch_bounds__(BNT) bn_act_fwd_kernel(const __nv_bfloat16* __restrict__ z, int zcs, Geo g,
                                                         const float* __restrict__ scale, const float* __restrict__ shift,
                                                         float slope, int has_act, const __nv_bfloat16* __restrict__ res,
                                                         int rcs, __nv_bfloat16* __restrict__ y, int ycs, int up,
                                                         int rows_per_block, const float* __restrict__ slope_dev,
                                                         __nv_bfloat16* __restrict__ xs, int xcs) {
  if (slope_dev) slope = __ldg(slope_dev);
  const RowSpan rs = row_span(g);
  float sc[8], sh[8];
  load8(scale, rs.cg, sc);
  load8(shift, rs.cg, sh);
  const int nrows = g.batch * g.h;
  const int row_begin = blockIdx.x * rows_per_block, row_end = min(nrows, row_begin + rows_per_block);
  for (int row = row_begin; row < row_end; row++) {
    const int b = row / g.h, yy = row - b * g.h;
    const __nv_bfloat16* zr = z + pad_off(b, yy, 0, g.h, g.w, zcs) + rs.cg * 8;
    const __nv_bfloat16* rr = res ? res + pad_off(b, yy, 0, g.h, g.w, rcs) + rs.cg * 8 : nullptr;
    for (int x = rs.px0; x < g.w; x += rs.pstep) {
      float f[8], r[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      unpack8(*reinterpret_cast<const uint4*>(zr + (size_t)x * zcs), f);
      if (rr) unpack8(*reinterpret_cast<const uint4*>(rr + (size_t)x * rcs), r);
#pragma unroll
      for (int e = 0; e < 8; e++) {
        float u = fmaf(f[e], sc[e], sh[e]);
        if (has_act) u = u > 0.f ? u : slope * u;
        f[e] = u + r[e];
      }
      const uint4 o = pack8(f);
      if (!up) {
        *reinterpret_cast<uint4*>(y + pad_off(b, yy, x, g.h, g.w, ycs) + rs.cg * 8) = o;
        // second copy in the space-to-depth layout of a following 3x3/stride-2 block (saves its s2d pass over y)
        if (xs) *reinterpret_cast<uint4*>(xs + pad_off(b, yy >> 1, x >> 1, g.h >> 1, g.w >> 1, xcs) +
                                          ((yy & 1) * 2 + (x & 1)) * g.c + rs.cg * 8) = o;
      } else {
#pragma unroll
        for (int ry = 0; ry < 2; ry++)
#pragma unroll
          for (int rx = 0; rx < 2; rx++)
            *reinterpret_cast<uint4*>(y + pad_off(b, 2 * yy + ry, 2 * x + rx, 2 * g.h, 2 * g.w, ycs) + rs.cg * 8) = o;
      }
    }
  }
}

// dy for one 8-channel group; up = 1: at 2x resolution (sum of the 2x2 block = adjoint of nearest upsample); up = 2: dy
// lives in the space-to-depth layout of the consuming 3x3/stride-2 block (its dgrad output, read in place instead of
// being scattered back by a depth_to_space pass)
__device__ __forceinline__ const __nv_bfloat16* dy_s2d_ptr(const __nv_bfloat16* __restrict__ dy, int dcs, const Geo& g, int b,
                                                           int y, int x, int cg) {
  return dy + pad_off(b, y >> 1, x >> 1, g.h >> 1, g.w >> 1, dcs) + ((y & 1) * 2 + (x & 1)) * g.c + cg * 8;
}
__device__ __forceinline__ void load_dy(const __nv_bfloat16* __restrict__ dy, int dcs, const Geo& g, int b, int y, int x,
                                        int cg, int up, float* d) {
  if (up == 2) {
    unpack8(*reinterpret_cast<const uint4*>(dy_s2d_ptr(dy, dcs, g, b, y, x, cg)), d);
  } else if (!up) {
    unpack8(*reinterpret_cast<const uint4*>(dy + pad_off(b, y, x, g.h, g.w, dcs) + cg * 8), d);
  } else {
#pragma unroll
    for (int e = 0; e < 8; e++) d[e] = 0.f;
#pragma unroll
    for (int ry = 0; ry < 2; ry++)
#pragma unroll
      for (int rx = 0; rx < 2; rx++) {
        float t[8];
        unpack8(*reinterpret_cast<const uint4*>(dy + pad_off(b, 2 * y + ry, 2 * x + rx, 2 * g.h, 2 * g.w, dcs) + cg * 8), t);
#pragma unroll
        for (int e = 0; e < 8; e++) d[e] += t[e];
      }
  }
}

__global__ void __launch_bounds__(BNT, 3) bn_act_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ dy, int dcs, int up,
                                                                const __nv_bfloat16* __restrict__ z, int zcs, Geo g,
                                                                const float* __restrict__ scale,
                                                                const float* __restrict__ shift,
                                                                const float* __restrict__ mean,
                                                                const float* __restrict__ invstd, float slope, int has_act,
                                                                float* __restrict__ partials /*[gridDim.x][2*c + 1]*/,
                                                                int rows_per_block, const float* __restrict__ slope_dev) {
  if (slope_dev) slope = __ldg(slope_dev);
  extern __shared__ float s_acc[];  // [kAccFloats]
  __syncthreads();
  const RowSpan rs = row_span(g);
  float sc[8], sh[8], mu[8], is[8];
  load8(scale, rs.cg, sc);
  load8(shift, rs.cg, sh);
  load8(mean, rs.cg, mu);
  load8(invstd, rs.cg, is);
  const int nrows = g.batch * g.h;
  const int row_begin = blockIdx.x * rows_per_block, row_end = min(nrows, row_begin + rows_per_block);
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
  for (int row = row_begin; row < row_end; row++) {
    const int b = row / g.h, y = row - b * g.h;
    const __nv_bfloat16* zr = z + pad_off(b, y, 0, g.h, g.w, zcs) + rs.cg * 8;
    for (int x = rs.px0; x < g.w; x += rs.pstep) {
      const uint4 zv = *reinterpret_cast<const uint4*>(zr + (size_t)x * zcs);
      float d[8];
      load_dy(dy, dcs, g, b, y, x, rs.cg, up, d);
      const uint32_t zw[4] = {zv.x, zv.y, zv.z, zv.w};
#pragma unroll
      for (int e = 0; e < 4; e++) {
        // two channels per step in packed fp32x2: u = z*scale + shift, zhat = (z - mean) * invstd
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
  float a1[8], a2[8];
#pragma unroll
  for (int e = 0; e < 4; e++) {
    f2unpack(q1[e], a1[2 * e], a1[2 * e + 1]);
    f2unpack(q2[e], a2[2 * e], a2[2 * e + 1]);
  }
  // the slope term: a fixed butterfly per warp, then the warps in order
  for (int o = 16; o > 0; o >>= 1) asl += __shfl_xor_sync(0xffffffffu, asl, o);
  block_partials(rs, g.c, a1, a2, asl, true, s_acc, partials);
}

__global__ void __launch_bounds__(BNT) bn_act_bwd_apply_kernel(const __nv_bfloat16* __restrict__ dy, int dcs, int up,
                                                               __nv_bfloat16* __restrict__ z /*in: z, out: dz*/, int zcs,
                                                               Geo g, const float* __restrict__ scale,
                                                               const float* __restrict__ shift,
                                                               const float* __restrict__ mean,
                                                               const float* __restrict__ invstd, float slope, int has_act,
                                                               int has_bn, const float* __restrict__ sums, float inv_n,
                                                               __nv_bfloat16* __restrict__ gres, int gcs, int gres_acc,
                                                               int rows_per_block, const float* __restrict__ slope_dev) {
  if (slope_dev) slope = __ldg(slope_dev);
  const RowSpan rs = row_span(g);
  float sc[8], sh[8], mu[8], is[8], m1[8], m2[8];
  load8(scale, rs.cg, sc);
  load8(shift, rs.cg, sh);
  load8(mean, rs.cg, mu);
  load8(invstd, rs.cg, is);
  load8(sums, rs.cg, m1);
  load8(sums + g.c, rs.cg, m2);
#pragma unroll
  for (int e = 0; e < 8; e++) {
    m1[e] *= inv_n;
    m2[e] *= inv_n;
  }
  uint64_t sc2[4], sh2[4], nmu2[4], is2[4], nm12[4], nm22[4];
#pragma unroll
  for (int e = 0; e < 4; e++) {
    sc2[e] = f2pack(sc[2 * e], sc[2 * e + 1]);
    sh2[e] = f2pack(sh[2 * e], sh[2 * e + 1]);
    nmu2[e] = f2pack(-mu[2 * e], -mu[2 * e + 1]);
    is2[e] = f2pack(is[2 * e], is[2 * e + 1]);
    nm12[e] = f2pack(-m1[2 * e], -m1[2 * e + 1]);
    nm22[e] = f2pack(-m2[2 * e], -m2[2 * e + 1]);
  }
  const int nrows = g.batch * g.h;
  const int row_begin = blockIdx.x * rows_per_block, row_end = min(nrows, row_begin + rows_per_block);
  constexpr int U = 2;   // pixels per iteration, all loads issued before the arithmetic
  for (int row = row_begin; row < row_end; row++) {
    const int b = row / g.h, y = row - b * g.h;
    __nv_bfloat16* zr = z + pad_off(b, y, 0, g.h, g.w, zcs) + rs.cg * 8;
    const __nv_bfloat16* dr = dy + pad_off(b, y, 0, g.h, g.w, dcs) + rs.cg * 8;
    __nv_bfloat16* gr = gres ? gres + pad_off(b, y, 0, g.h, g.w, gcs) + rs.cg * 8 : nullptr;
    for (int x0 = rs.px0; x0 < g.w; x0 += U * rs.pstep) {
      uint4 zv[U], dv[U], gv[U];
      float d[U][8];
#pragma unroll
      for (int q = 0; q < U; q++) {
        const int x = x0 + q * rs.pstep;
        if (x < g.w) {
          zv[q] = *reinterpret_cast<const uint4*>(zr + (size_t)x * zcs);
          if (!up) dv[q] = __ldg(reinterpret_cast<const uint4*>(dr + (size_t)x * dcs));
          else if (up == 2) dv[q] = __ldg(reinterpret_cast<const uint4*>(dy_s2d_ptr(dy, dcs, g, b, y, x, rs.cg)));
          if (gr && gres_acc) gv[q] = *reinterpret_cast<const uint4*>(gr + (size_t)x * gcs);
        }
      }
#pragma unroll
      for (int q = 0; q < U; q++) {
        const int x = x0 + q * rs.pstep;
        if (x >= g.w) continue;
        if (up != 1) unpack8(dv[q], d[q]);
        else load_dy(dy, dcs, g, b, y, x, rs.cg, up, d[q]);
        if (gr) {  // shortcut branch: d(residual) (+)= dy   (never combined with upsample)
          float o[8];
          if (gres_acc) {
            unpack8(gv[q], o);
#pragma unroll
            for (int e = 0; e < 8; e++) o[e] += d[q][e];
          } else {
#pragma unroll
            for (int e = 0; e < 8; e++) o[e] = d[q][e];
          }
          *reinterpret_cast<uint4*>(gr + (size_t)x * gcs) = pack8(o);
        }
        float out[8];
        const uint32_t zw[4] = {zv[q].x, zv[q].y, zv[q].z, zv[q].w};
#pragma unroll
        for (int e = 0; e < 4; e++) {      // two channels per step, packed fp32x2
          const uint64_t f2 = bf2_to_f2(zw[e]);
          float u0, u1;
          f2unpack(f2fma(f2, sc2[e], sh2[e]), u0, u1);
          float du0 = d[q][2 * e], du1 = d[q][2 * e + 1];
          if (has_act) {
            if (!(u0 > 0.f)) du0 *= slope;
            if (!(u1 > 0.f)) du1 *= slope;
          }
          if (has_bn) {
            // sc * (du - m1 - zhat * m2),  zhat = (z - mean) * invstd
            const uint64_t zh2 = f2mul(f2add(f2, nmu2[e]), is2[e]);
            const uint64_t t2 = f2fma(zh2, nm22[e], f2add(f2pack(du0, du1), nm12[e]));
            f2unpack(f2mul(sc2[e], t2), out[2 * e], out[2 * e + 1]);
          } else {
            out[2 * e] = du0;
            out[2 * e + 1] = du1;
          }
        }
        *reinterpret_cast<uint4*>(zr + (size_t)x * zcs) = pack8(out);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// adjoint of "keep the even pixels" (stride-2 conv): small grid gradient placed on the even interior pixels of the
// (pre-zeroed, never otherwise written) input-resolution buffer
__global__ void __launch_bounds__(256) zero_insert2x_kernel(const __nv_bfloat16* __restrict__ src, int scs, Geo g /*small*/,
                                                            __nv_bfloat16* __restrict__ dst, int dcs, int ih, int iw) {
  const size_t item = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int b, y, x, cg;
  if (!decode_item(g, item, b, y, x, cg)) return;
  const uint4 v = *reinterpret_cast<const uint4*>(src + pad_off(b, y, x, g.h, g.w, scs) + cg * 8);
  *reinterpret_cast<uint4*>(dst + pad_off(b, 2 * y, 2 * x, ih, iw, dcs) + cg * 8) = v;
}

// space-to-depth for the stride-2 convolutions: xs[b, Y, X, (py*2+px)*C + c] = x[b, 2Y+py, 2X+px, c] (interior coordinates,
// H and W even).  On xs a 3x3/stride-2/pad-1 conv is a 2x2-tap stride-1 conv (tap offsets -1..0) with 4C input channels
// (7 of the 16 (tap, phase) weight blocks are zero) -- the same flat implicit GEMM, 1.78x instead of 4x MMA work.
__global__ void __launch_bounds__(256) space_to_depth_kernel(const __nv_bfloat16* __restrict__ x, int xcs, Geo g /*of x*/,
                                                             __nv_bfloat16* __restrict__ xs, int scs) {
  const size_t item = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int b, y, xx, cg;
  if (!decode_item(g, item, b, y, xx, cg)) return;
  const uint4 v = *reinterpret_cast<const uint4*>(x + pad_off(b, y, xx, g.h, g.w, xcs) + cg * 8);
  const int ph = (y & 1) * 2 + (xx & 1);
  *reinterpret_cast<uint4*>(xs + pad_off(b, y >> 1, xx >> 1, g.h >> 1, g.w >> 1, scs) + ph * g.c + cg * 8) = v;
}
// adjoint: gx[b, 2Y+py, 2X+px, c] (+)= dxs[b, Y, X, (py*2+px)*C + c]
__global__ void __launch_bounds__(256) depth_to_space_kernel(const __nv_bfloat16* __restrict__ dxs, int scs, Geo g /*of gx*/,
                                                             __nv_bfloat16* __restrict__ gx, int gcs, int accumulate) {
  const size_t item = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int b, y, xx, cg;
  if (!decode_item(g, item, b, y, xx, cg)) return;
  const int ph = (y & 1) * 2 + (xx & 1);
  float d[8];
  unpack8(*reinterpret_cast<const uint4*>(dxs + pad_off(b, y >> 1, xx >> 1, g.h >> 1, g.w >> 1, scs) + ph * g.c + cg * 8), d);
  __nv_bfloat16* gp = gx + pad_off(b, y, xx, g.h, g.w, gcs) + cg * 8;
  if (accumulate) {
    float o[8];
    unpack8(*reinterpret_cast<const uint4*>(gp), o);
#pragma unroll
    for (int e = 0; e < 8; e++) d[e] += o[e];
  }
  *reinterpret_cast<uint4*>(gp) = pack8(d);
}

// Phase decomposition of the dilated 3x3 convolutions ([d-convolutional] blocks, dilation (dh, dw), pad (dh, dw)):
// xp[(b*dh + ry)*dw + rx, Y, X, c] = x[b, Y*dh + ry, X*dw + rx, c], zero where that pixel is past the edge.  On every
// phase image the dilated conv is an ordinary pad-1 3x3 conv.  One thread per 16-byte group of the phase image; the
// stores are contiguous, the loads contiguous within each pixel.
__global__ void __launch_bounds__(256) dilate_split_kernel(const __nv_bfloat16* __restrict__ x, int xcs, Geo g /*of x*/,
                                                           Geo gp /*of xp*/, int dh, int dw, __nv_bfloat16* __restrict__ xp,
                                                           int pcs) {
  const size_t item = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int n, py, px, cg;
  if (!decode_item(gp, item, n, py, px, cg)) return;
  const int rx = n % dw, ry = (n / dw) % dh, b = n / (dw * dh);
  const int y = py * dh + ry, xx = px * dw + rx;
  uint4 v = make_uint4(0u, 0u, 0u, 0u);
  if (y < g.h && xx < g.w) v = *reinterpret_cast<const uint4*>(x + pad_off(b, y, xx, g.h, g.w, xcs) + cg * 8);
  *reinterpret_cast<uint4*>(xp + pad_off(n, py, px, gp.h, gp.w, pcs) + cg * 8) = v;
}
// its inverse on the interior pixels and its adjoint: y[b, y, x] = xp[phase of (y, x)] (+ residual) (+ y), summed in fp32
// in that order and rounded to bf16 once
__global__ void __launch_bounds__(256) dilate_merge_kernel(const __nv_bfloat16* __restrict__ xp, int pcs, Geo gp /*of xp*/,
                                                           Geo g /*of y*/, int dh, int dw,
                                                           const __nv_bfloat16* __restrict__ res, int rcs, int accumulate,
                                                           __nv_bfloat16* __restrict__ y, int ycs) {
  const size_t item = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int b, yy, xx, cg;
  if (!decode_item(g, item, b, yy, xx, cg)) return;
  const int n = (b * dh + yy % dh) * dw + xx % dw;
  float d[8];
  unpack8(*reinterpret_cast<const uint4*>(xp + pad_off(n, yy / dh, xx / dw, gp.h, gp.w, pcs) + cg * 8), d);
  if (res) {
    float r[8];
    unpack8(*reinterpret_cast<const uint4*>(res + pad_off(b, yy, xx, g.h, g.w, rcs) + cg * 8), r);
#pragma unroll
    for (int e = 0; e < 8; e++) d[e] += r[e];
  }
  __nv_bfloat16* yp = y + pad_off(b, yy, xx, g.h, g.w, ycs) + cg * 8;
  if (accumulate) {
    float o[8];
    unpack8(*reinterpret_cast<const uint4*>(yp), o);
#pragma unroll
    for (int e = 0; e < 8; e++) d[e] += o[e];
  }
  *reinterpret_cast<uint4*>(yp) = pack8(d);
}

// 2x2 max pooling on padded NHWC (reference: nn.MaxPool2d(2, stride) blocks of cfg/yolov3-tiny.cfg, model/models.py:79-87).
// stride 2: out[y, x] = max over in[2y..2y+1, 2x..2x+1].  stride 1: the reference zero-pads right/bottom
// (nn.ZeroPad2d((0,1,0,1))) and pools with stride 1 -> out[y, x] = max over in[y..y+1, x..x+1] where the row/column past
// the edge reads ZERO -- which is exactly the zero halo of the padded layout.
__global__ void __launch_bounds__(256) maxpool2x2_kernel(const __nv_bfloat16* __restrict__ x, int xcs, int ih, int iw,
                                                         Geo g /*output*/, int stride, __nv_bfloat16* __restrict__ y, int ycs) {
  const size_t item = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int b, oy, ox, cg;
  if (!decode_item(g, item, b, oy, ox, cg)) return;
  const int y0 = oy * stride, x0 = ox * stride;
  __nv_bfloat162 m[4];
  bool first = true;
#pragma unroll
  for (int dy = 0; dy < 2; dy++)
#pragma unroll
    for (int dx = 0; dx < 2; dx++) {
      const uint4 v = *reinterpret_cast<const uint4*>(x + pad_off(b, y0 + dy, x0 + dx, ih, iw, xcs) + cg * 8);
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
      for (int e = 0; e < 4; e++) m[e] = first ? h[e] : __hmax2(m[e], h[e]);
      first = false;
    }
  *reinterpret_cast<uint4*>(y + pad_off(b, oy, ox, g.h, g.w, ycs) + cg * 8) = *reinterpret_cast<uint4*>(m);
}

// im2col of the 3-channel image for the first 3x3/stride-1/pad-1 conv: column index = c*9 + kh*3 + kw (the flattening
// of nn.Conv2d.weight[co]), 27 real + zero padding to 64 channels, bf16 padded NHWC.  A thread builds one pixel's
// 128-byte row in shared memory; the block then stores its rows as 16-byte chunks in address order, so a warp writes
// 4 consecutive pixels (512 contiguous bytes) per instruction instead of 16 bytes in each of 32 rows.
__global__ void __launch_bounds__(256) im2col_first_kernel(const float* __restrict__ img, int batch, int h, int w,
                                                           __nv_bfloat16* __restrict__ dst /*cs = 64*/) {
  __shared__ uint4 rows[256 * 8];      // [pixel][chunk ^ (pixel % 8)]: the per-pixel writes hit distinct banks
  __shared__ size_t offs[256];         // element offset of the pixel's row in dst
  const size_t npix = (size_t)batch * h * w;
  const size_t pix0 = (size_t)blockIdx.x * 256;
  const int t = threadIdx.x;
  const size_t pix = pix0 + t;
  if (pix < npix) {
    const int x = (int)(pix % w);
    const int y = (int)((pix / w) % h);
    const int b = (int)(pix / ((size_t)w * h));
    float v[32];
#pragma unroll
    for (int k = 0; k < 32; k++) v[k] = 0.f;
#pragma unroll
    for (int c = 0; c < 3; c++)
#pragma unroll
      for (int dy = 0; dy < 3; dy++)
#pragma unroll
        for (int dx = 0; dx < 3; dx++) {
          const int yy = y + dy - 1, xx = x + dx - 1;
          if (yy >= 0 && yy < h && xx >= 0 && xx < w) v[c * 9 + dy * 3 + dx] = __ldg(img + (((size_t)b * 3 + c) * h + yy) * w + xx);
        }
#pragma unroll
    for (int q = 0; q < 4; q++) rows[t * 8 + (q ^ (t & 7))] = pack8(v + q * 8);
#pragma unroll
    for (int q = 4; q < 8; q++) rows[t * 8 + (q ^ (t & 7))] = make_uint4(0, 0, 0, 0);
    offs[t] = pad_off(b, y, x, h, w, 64);
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const int k = i * 256 + t, px = k >> 3, q = k & 7;
    if (pix0 + px < npix) *reinterpret_cast<uint4*>(dst + offs[px] + q * 8) = rows[px * 8 + (q ^ (px & 7))];
  }
}

static inline Geo mk_geo(int batch, int h, int w, int c) {
  Geo g;
  g.batch = batch; g.h = h; g.w = w; g.c = c;
  return g;
}
static inline size_t n_items(const Geo& g) { return (size_t)g.batch * g.h * g.w * (g.c >> 3); }
// rows per CTA so that a CTA streams ~16k 16-byte items and the grid still has >= ~4 CTAs per SM
static inline int rows_per_block(const Geo& g) {
  constexpr long long kItemsPerCta = 16384;
  const int cgs = g.c >> 3;
  long long per_row = (long long)g.w * cgs;
  int r = (int)((kItemsPerCta + per_row - 1) / per_row);
  const int nrows = g.batch * g.h;
  const int max_r = (nrows + 591) / 592;
  if (r > max_r) r = max_r;
  return r < 1 ? 1 : r;
}
static inline bool pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

}  // namespace ryolo

#include "bnpipe.cuh"

namespace ryolo {

// per-CTA partial rows of the BN reductions
static float* bn_partials(cudaStream_t stream, size_t floats) {
  return static_cast<float*>(stream_scratch(stream, SCRATCH_BN, floats * sizeof(float)));
}

static int bn_sums_reduce(const float* partials, int rows, int c, int has_extra, float* sums, const BnFinalize& fin,
                          cudaStream_t stream) {
  bn_sums_reduce_kernel<<<(c + 31) / 32 + has_extra, 32 * kReduceParts, 0, stream>>>(partials, rows, c, has_extra, sums, fin);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

}  // namespace ryolo

using namespace ryolo;

#define GEO_CHECK() RYOLO_ARG_CHECK(batch > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0 && c <= 2048)
#define GEO_CHECK_P2() RYOLO_ARG_CHECK(pow2(c >> 3))

// statistics (and, with fin.gamma, their finalisation): per-CTA partial rows, then one ordered reduction
static int bn_stats_impl(const void* z, int z_cstride, const Geo& g, float* sums, const BnFinalize& fin, cudaStream_t stream) {
  const int c = g.c;
  int grid;
  PieceGeo pg;
  const bool piped = pipe_ok(g, z_cstride);
  const int rpb = rows_per_block(g);
  if (piped) {
    pg = mk_pieces(g, &grid);
    pg.rev = 1;   // descending: it starts in the tail the conv just wrote
  } else {
    grid = (g.batch * g.h + rpb - 1) / rpb;
  }
  float* partials = bn_partials(stream, (size_t)grid * 2 * c);
  if (!partials) return RYOLO_E_CUDA;
  if (piped) {
    constexpr size_t kMax = RowPipe<1, 4>::smem_bytes() + kAccBytes;
    RYOLO_SMEM_OPT_IN(bn_stats_pipe_kernel, kMax);
    bn_stats_pipe_kernel<<<grid, BNT, kMax, stream>>>(static_cast<const __nv_bfloat16*>(z), g, pg, partials);
  } else {
    bn_stats_kernel<<<grid, BNT, kAccBytes, stream>>>(static_cast<const __nv_bfloat16*>(z), z_cstride, g, partials, rpb);
  }
  RYOLO_LAUNCH_CHECK();
  return bn_sums_reduce(partials, grid, c, 0, sums, fin, stream);
}

static int bn_act_fwd_impl(const void* z, int z_cstride, int batch, int h, int w, int c, const float* scale,
                           const float* shift, float slope, int has_act, const void* residual, int res_cstride, void* y,
                           int y_cstride, int upsample2x, const float* slope_dev, void* xs, int xs_cstride, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(z && scale && shift && y);
  GEO_CHECK();
  RYOLO_ARG_CHECK(!(residual && upsample2x));
  RYOLO_ARG_CHECK(!xs || (!upsample2x && h % 2 == 0 && w % 2 == 0 && xs_cstride >= 4 * c && xs_cstride % 8 == 0));
  GEO_CHECK_P2();
  const Geo g = mk_geo(batch, h, w, c);
  const int rpb = rows_per_block(g);
  bn_act_fwd_kernel<<<(unsigned)((batch * h + rpb - 1) / rpb), BNT, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(z), z_cstride, g, scale, shift, slope, has_act,
      static_cast<const __nv_bfloat16*>(residual), res_cstride, static_cast<__nv_bfloat16*>(y), y_cstride, upsample2x, rpb,
      slope_dev, static_cast<__nv_bfloat16*>(xs), xs_cstride);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_bn_act_fwd(const void* z, int z_cstride, int batch, int h, int w, int c, const float* scale,
                                const float* shift, float slope, int has_act, const void* residual, int res_cstride,
                                void* y, int y_cstride, int upsample2x, const float* slope_dev, void* stream_) {
  return bn_act_fwd_impl(z, z_cstride, batch, h, w, c, scale, shift, slope, has_act, residual, res_cstride, y, y_cstride,
                         upsample2x, slope_dev, nullptr, 0, stream_);
}

extern "C" int ryolo_bn_act_fwd_s2d(const void* z, int z_cstride, int batch, int h, int w, int c, const float* scale,
                                    const float* shift, float slope, int has_act, const void* residual, int res_cstride,
                                    void* y, int y_cstride, const float* slope_dev, void* xs, int xs_cstride,
                                    void* stream_) {
  RYOLO_ARG_CHECK(xs != nullptr);
  return bn_act_fwd_impl(z, z_cstride, batch, h, w, c, scale, shift, slope, has_act, residual, res_cstride, y, y_cstride, 0,
                         slope_dev, xs, xs_cstride, stream_);
}

extern "C" int ryolo_bn_act_bwd(const void* dy, int dy_cstride, int upsample2x, void* z_dz, int z_cstride, int batch, int h,
                                int w, int c, const float* scale, const float* shift, const float* mean,
                                const float* invstd, float slope, int has_act, int has_bn, float* sums, void* gres,
                                int gres_cstride, int gres_accumulate, const float* slope_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(dy && z_dz && scale && shift && mean && invstd && sums);
  GEO_CHECK();
  RYOLO_ARG_CHECK(upsample2x >= 0 && upsample2x <= 2 && !(gres && upsample2x == 1));
  RYOLO_ARG_CHECK(upsample2x != 2 || (h % 2 == 0 && w % 2 == 0 && dy_cstride >= 4 * c));
  GEO_CHECK_P2();
  const Geo g = mk_geo(batch, h, w, c);
  const float inv_cnt = 1.0f / ((float)batch * h * w);
  if (pipe_ok(g, z_cstride)) {
    // how dy reaches the kernels: 1 = plain tensor on the pipe, 2 = space-to-depth dgrad output on the pipe (row pairs),
    // 0 = direct loads (upsample adjoint, concat buffers)
    const int dyp = (upsample2x == 0 && dy_cstride == c) ? 1
                    : (upsample2x == 2 && dy_cstride == 4 * c && (c >> 3) * 2 <= PIPE_ITEMS / 2) ? 2 : 0;
    int grid;
    const PieceGeo pg = mk_pieces(g, &grid, dyp == 2 ? 2 : 1);
    constexpr size_t kMax = BwdPipe<0>::smem_bytes() + kAccBytes;
    static_assert(BwdPipe<0>::smem_bytes() == BwdPipe<1>::smem_bytes() + 16 && BwdPipe<1>::smem_bytes() == BwdPipe<2>::smem_bytes(),
                  "stage rings of equal size");
    const __nv_bfloat16* dyb = static_cast<const __nv_bfloat16*>(dy);
    __nv_bfloat16* zb = static_cast<__nv_bfloat16*>(z_dz);
    __nv_bfloat16* grb = static_cast<__nv_bfloat16*>(gres);
    float* partials = bn_partials(stream, (size_t)grid * (2 * c + 1));
    if (!partials) return RYOLO_E_CUDA;
    PieceGeo pg_red = pg;                       // the reduction walks descending (it starts in the tail dgrad just wrote),
    pg_red.rev = 1;                             // the apply pass ascending (it starts where the reduction ended)
#define RYOLO_BWD_PIPE(D)                                                                                                  \
  do {                                                                                                                   \
    RYOLO_SMEM_OPT_IN(bn_act_bwd_reduce_pipe_kernel<D>, kMax);                                                           \
    RYOLO_SMEM_OPT_IN(bn_act_bwd_apply_pipe_kernel<D>, kMax);                                                            \
    bn_act_bwd_reduce_pipe_kernel<D><<<grid, BNT, BwdPipe<D>::smem_bytes() + kAccBytes, stream>>>(                       \
        dyb, dy_cstride, upsample2x, zb, g, pg_red, scale, shift, mean, invstd, slope, has_act, partials, slope_dev);       \
    RYOLO_LAUNCH_CHECK();                                                                                                \
    if (bn_sums_reduce(partials, grid, c, 1, sums, BnFinalize{}, stream) != RYOLO_OK) return RYOLO_E_CUDA;              \
    bn_act_bwd_apply_pipe_kernel<D><<<grid, BNT, BwdPipe<D>::smem_bytes(), stream>>>(                                    \
        dyb, dy_cstride, upsample2x, zb, g, pg, scale, shift, mean, invstd, slope, has_act, has_bn, sums, inv_cnt, grb,  \
        gres_cstride, gres_accumulate, slope_dev);                                                                       \
    RYOLO_LAUNCH_CHECK();                                                                                                \
  } while (0)
    if (dyp == 1) RYOLO_BWD_PIPE(1);
    else if (dyp == 2) RYOLO_BWD_PIPE(2);
    else RYOLO_BWD_PIPE(0);
#undef RYOLO_BWD_PIPE
    return RYOLO_OK;
  }
  const int rpb = rows_per_block(g);
  const unsigned blocks = (unsigned)((batch * h + rpb - 1) / rpb);
  float* partials = bn_partials(stream, (size_t)blocks * (2 * c + 1));
  if (!partials) return RYOLO_E_CUDA;
  bn_act_bwd_reduce_kernel<<<blocks, BNT, kAccBytes, stream>>>(
      static_cast<const __nv_bfloat16*>(dy), dy_cstride, upsample2x, static_cast<const __nv_bfloat16*>(z_dz), z_cstride, g,
      scale, shift, mean, invstd, slope, has_act, partials, rpb, slope_dev);
  RYOLO_LAUNCH_CHECK();
  if (bn_sums_reduce(partials, (int)blocks, c, 1, sums, BnFinalize{}, stream) != RYOLO_OK) return RYOLO_E_CUDA;
  const float inv_n = 1.0f / ((float)batch * h * w);
  bn_act_bwd_apply_kernel<<<blocks, BNT, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(dy), dy_cstride, upsample2x, static_cast<__nv_bfloat16*>(z_dz), z_cstride, g, scale,
      shift, mean, invstd, slope, has_act, has_bn, sums, inv_n, static_cast<__nv_bfloat16*>(gres), gres_cstride,
      gres_accumulate, rpb, slope_dev);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_bn_stats_finalize(const void* z, int z_cstride, int batch, int h, int w, int c, float* sums, float eps,
                                       float momentum, const float* gamma, const float* beta, float* mean, float* invstd,
                                       float* scale, float* shift, float* running_mean, float* running_var, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(z && sums && gamma && beta && mean && invstd && scale && shift);
  RYOLO_ARG_CHECK((running_mean == nullptr) == (running_var == nullptr));
  GEO_CHECK();
  GEO_CHECK_P2();
  const Geo g = mk_geo(batch, h, w, c);
  const float count = (float)batch * h * w;
  BnFinalize fin;
  fin.gamma = gamma; fin.beta = beta; fin.mean = mean; fin.invstd = invstd; fin.scale = scale; fin.shift = shift;
  fin.running_mean = running_mean; fin.running_var = running_var; fin.count = count; fin.eps = eps; fin.momentum = momentum;
  return bn_stats_impl(z, z_cstride, g, sums, fin, stream);
}

extern "C" int ryolo_zero_insert2x(const void* src, int src_cstride, int batch, int h, int w, int c, void* dst,
                                   int dst_cstride, int dst_h, int dst_w, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(src && dst);
  GEO_CHECK();
  RYOLO_ARG_CHECK(dst_h >= 2 * h - 1 && dst_w >= 2 * w - 1);
  const Geo g = mk_geo(batch, h, w, c);
  const size_t items = n_items(g);
  zero_insert2x_kernel<<<(unsigned)((items + 255) / 256), 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(src),
                                                                           src_cstride, g, static_cast<__nv_bfloat16*>(dst),
                                                                           dst_cstride, dst_h, dst_w);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_space_to_depth(const void* x, int x_cstride, int batch, int h, int w, int c, void* xs, int xs_cstride,
                                    void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(x && xs);
  GEO_CHECK();
  RYOLO_ARG_CHECK(h % 2 == 0 && w % 2 == 0 && xs_cstride >= 4 * c);
  const Geo g = mk_geo(batch, h, w, c);
  const size_t items = n_items(g);
  space_to_depth_kernel<<<(unsigned)((items + 255) / 256), 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), x_cstride,
                                                                            g, static_cast<__nv_bfloat16*>(xs), xs_cstride);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_depth_to_space(const void* dxs, int dxs_cstride, int batch, int h, int w, int c, void* gx,
                                    int gx_cstride, int accumulate, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(dxs && gx);
  GEO_CHECK();
  RYOLO_ARG_CHECK(h % 2 == 0 && w % 2 == 0 && dxs_cstride >= 4 * c);
  const Geo g = mk_geo(batch, h, w, c);
  const size_t items = n_items(g);
  depth_to_space_kernel<<<(unsigned)((items + 255) / 256), 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(dxs),
                                                                            dxs_cstride, g, static_cast<__nv_bfloat16*>(gx),
                                                                            gx_cstride, accumulate);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int ryolo_dilate_split(const void* x, int x_cstride, int batch, int h, int w, int c, int dh, int dw, void* xp,
                                  int xp_cstride, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(x && xp && aligned16(x) && aligned16(xp));
  GEO_CHECK();
  RYOLO_ARG_CHECK(dh >= 1 && dw >= 1 && (long long)batch * dh * dw < (1ll << 24));
  RYOLO_ARG_CHECK(x_cstride >= c && x_cstride % 8 == 0 && xp_cstride >= c && xp_cstride % 8 == 0);
  const Geo g = mk_geo(batch, h, w, c);
  const Geo gp = mk_geo(batch * dh * dw, (h + dh - 1) / dh, (w + dw - 1) / dw, c);
  const size_t items = n_items(gp);
  dilate_split_kernel<<<(unsigned)((items + 255) / 256), 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), x_cstride,
                                                                          g, gp, dh, dw, static_cast<__nv_bfloat16*>(xp),
                                                                          xp_cstride);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_dilate_merge(const void* xp, int xp_cstride, int batch, int h, int w, int c, int dh, int dw,
                                  const void* residual, int res_cstride, int accumulate, void* y, int y_cstride,
                                  void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(xp && y && aligned16(xp) && aligned16(y) && (!residual || aligned16(residual)));
  GEO_CHECK();
  RYOLO_ARG_CHECK(dh >= 1 && dw >= 1 && (long long)batch * dh * dw < (1ll << 24));
  RYOLO_ARG_CHECK(xp_cstride >= c && xp_cstride % 8 == 0 && y_cstride >= c && y_cstride % 8 == 0);
  RYOLO_ARG_CHECK(!residual || (res_cstride >= c && res_cstride % 8 == 0));
  const Geo g = mk_geo(batch, h, w, c);
  const Geo gp = mk_geo(batch * dh * dw, (h + dh - 1) / dh, (w + dw - 1) / dw, c);
  const size_t items = n_items(g);
  dilate_merge_kernel<<<(unsigned)((items + 255) / 256), 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(xp), xp_cstride, gp, g, dh, dw, static_cast<const __nv_bfloat16*>(residual),
      res_cstride, accumulate, static_cast<__nv_bfloat16*>(y), y_cstride);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_maxpool2x2(const void* x, int x_cstride, int batch, int in_h, int in_w, int c, int stride, void* y,
                                int y_cstride, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(x && y && batch > 0 && in_h > 0 && in_w > 0 && c > 0 && c % 8 == 0);
  RYOLO_ARG_CHECK(stride == 1 || (stride == 2 && in_h % 2 == 0 && in_w % 2 == 0));
  const Geo g = mk_geo(batch, stride == 2 ? in_h / 2 : in_h, stride == 2 ? in_w / 2 : in_w, c);
  const size_t items = n_items(g);
  maxpool2x2_kernel<<<(unsigned)((items + 255) / 256), 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), x_cstride, in_h,
                                                                        in_w, g, stride, static_cast<__nv_bfloat16*>(y),
                                                                        y_cstride);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_im2col_first(const float* img, int batch, int h, int w, void* dst, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(img && dst && batch > 0 && h > 0 && w > 0);
  const size_t npix = (size_t)batch * h * w;
  im2col_first_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, stream>>>(img, batch, h, w, static_cast<__nv_bfloat16*>(dst));
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}
