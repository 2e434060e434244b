// Elementwise kernels of the parity-precision path (see conv_parity.cu): everything between two convolutions in fp32,
// reductions in fp64 (PyTorch's CPU BatchNorm / PReLU-gradient reductions accumulate in double: at::acc_type<float,false>).
//
// Tensors:  z / gradient buffers  fp32 padded NHWC [B, H+2, W+2, cs] (zero halo);
//           GEMM operands         "split" bf16 padded NHWC: plane 0 at channel 0 of the view, plane k `k*lo` channels
//                                 further (nplanes = 2 or 3; plane k = bf16 of the remainder left by planes < k).
// Reference semantics: nn.BatchNorm2d(momentum 0.1, eps 1e-5) -> nn.PReLU(1) (model/models.py:62-65), shortcut add
// (:281-282), nn.Upsample nearest x2 (:93-94) and their autograd (train.py:278-282); eval mode uses the running
// statistics through the same scale/shift form (utils/torch_utils.py:45-69 folds the same numbers into the conv).
// Simple memory-bound kernels (thread = 8 channels of one pixel); this path exists for the tolerance, not for speed.
#include <cuda_bf16.h>

#include "common.cuh"

namespace ryolo {

struct PGeo {
  int batch, h, w, c;    // interior size, channels (multiple of 8)
};

__device__ __forceinline__ size_t ppad_off(int b, int y, int x, int h, int w, int cs) {
  return (((size_t)b * (h + 2) + y + 1) * (w + 2) + x + 1) * cs;
}
__device__ __forceinline__ void pload8(const float* __restrict__ p, float* o) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
}
__device__ __forceinline__ void pstore8(float* __restrict__ p, const float* o) {
  *reinterpret_cast<float4*>(p) = make_float4(o[0], o[1], o[2], o[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(o[4], o[5], o[6], o[7]);
}
// 8 fp32 -> np bf16 planes `ps` channels apart (plane k = bf16 of what planes < k left over)
__device__ __forceinline__ void split_store8(__nv_bfloat16* __restrict__ p0, int ps, int np, const float* f) {
  float r[8];
#pragma unroll
  for (int e = 0; e < 8; e++) r[e] = f[e];
  for (int k = 0; k < np; k++) {
    __nv_bfloat16 h[8];
#pragma unroll
    for (int e = 0; e < 8; e++) {
      h[e] = __float2bfloat16_rn(r[e]);
      r[e] -= __bfloat162float(h[e]);
    }
    *reinterpret_cast<uint4*>(p0 + (size_t)k * ps) = *reinterpret_cast<const uint4*>(h);
  }
}
__device__ __forceinline__ void split_load8(const __nv_bfloat16* __restrict__ p0, int ps, int np, float* f) {
#pragma unroll
  for (int e = 0; e < 8; e++) f[e] = 0.f;
  for (int k = np - 1; k >= 0; k--) {      // small planes first: the sum is exact in fp32 (24 bits in total)
    const uint4 v = *reinterpret_cast<const uint4*>(p0 + (size_t)k * ps);
    const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(&v);
#pragma unroll
    for (int e = 0; e < 8; e++) f[e] += __bfloat162float(h[e]);
  }
}
__device__ __forceinline__ void split_store1(__nv_bfloat16* __restrict__ p0, int ps, int np, float v) {
  for (int k = 0; k < np; k++) {
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    p0[(size_t)k * ps] = h;
    v -= __bfloat162float(h);
  }
}

// thread -> (pixel, channel group) with the channel group FIXED per thread (cgs divides the block size): per-thread
// partial sums stay in registers.  Pixels are walked with a grid stride.
constexpr int PXT = 256;
struct PWalk {
  int cg;
  size_t pix0, pstep, npix;
};
__device__ __forceinline__ PWalk pwalk(const PGeo& g) {
  PWalk wk;
  const int cgs = g.c >> 3;
  const int ppb = PXT / cgs;                       // pixels per block iteration
  wk.cg = threadIdx.x % cgs;
  wk.pix0 = (size_t)blockIdx.x * ppb + threadIdx.x / cgs;
  wk.pstep = (size_t)gridDim.x * ppb;
  wk.npix = (size_t)g.batch * g.h * g.w;
  if (threadIdx.x >= ppb * cgs) wk.pix0 = wk.npix;  // idle tail threads when cgs does not divide the block
  return wk;
}
__device__ __forceinline__ void pix_decode(const PGeo& g, size_t pix, int& b, int& y, int& x) {
  x = (int)(pix % g.w);
  y = (int)((pix / g.w) % g.h);
  b = (int)(pix / ((size_t)g.w * g.h));
}

// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(PXT) px_bn_stats_kernel(const float* __restrict__ z, int zcs, PGeo g,
                                                          double* __restrict__ sums /*[2c]*/) {
  const PWalk wk = pwalk(g);
  double s1[8], s2[8];
#pragma unroll
  for (int e = 0; e < 8; e++) s1[e] = s2[e] = 0.0;
  for (size_t pix = wk.pix0; pix < wk.npix; pix += wk.pstep) {
    int b, y, x;
    pix_decode(g, pix, b, y, x);
    float f[8];
    pload8(z + ppad_off(b, y, x, g.h, g.w, zcs) + wk.cg * 8, f);
#pragma unroll
    for (int e = 0; e < 8; e++) {
      s1[e] += (double)f[e];
      s2[e] += (double)f[e] * (double)f[e];
    }
  }
  if (wk.pix0 < wk.npix) {
#pragma unroll
    for (int e = 0; e < 8; e++) {
      atomicAdd(&sums[wk.cg * 8 + e], s1[e]);
      atomicAdd(&sums[g.c + wk.cg * 8 + e], s2[e]);
    }
  }
}

// mode 0 (training): batch statistics from `sums`, running statistics updated (momentum, unbiased variance).
// mode 1 (eval): statistics = running_mean / running_var, nothing written back.
__global__ void px_bn_finalize_kernel(const double* __restrict__ sums, int c, double count, float eps, float momentum,
                                      const float* __restrict__ gamma, const float* __restrict__ beta, int mode,
                                      float* __restrict__ mean_o, float* __restrict__ invstd_o, float* __restrict__ scale_o,
                                      float* __restrict__ shift_o, float* __restrict__ running_mean,
                                      float* __restrict__ running_var) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= c) return;
  float mean, var;
  if (mode == 0) {
    const double m = sums[ch] / count;
    double v = sums[c + ch] / count - m * m;
    if (v < 0.0) v = 0.0;
    mean = (float)m;
    var = (float)v;
    if (running_mean) {
      running_mean[ch] = (1.f - momentum) * running_mean[ch] + momentum * mean;
      running_var[ch] = (1.f - momentum) * running_var[ch] + momentum * (float)(v * (count / fmax(count - 1.0, 1.0)));
    }
  } else {
    mean = running_mean[ch];
    var = running_var[ch];
  }
  const float invstd = 1.0f / sqrtf(var + eps);
  const float sc = gamma[ch] * invstd;
  mean_o[ch] = mean;
  invstd_o[ch] = invstd;
  scale_o[ch] = sc;
  shift_o[ch] = beta[ch] - mean * sc;
}

// y = prelu(z*scale + shift) [+ residual]  ->  split planes (optionally 2x2 replicated)
__global__ void __launch_bounds__(PXT) px_bn_act_fwd_kernel(const float* __restrict__ z, int zcs, PGeo g,
                                                            const float* __restrict__ scale, const float* __restrict__ shift,
                                                            const float* __restrict__ slope_dev, int has_act,
                                                            const __nv_bfloat16* __restrict__ res, int rcs, int rlo,
                                                            __nv_bfloat16* __restrict__ y, int ycs, int ylo, int up, int np) {
  const PWalk wk = pwalk(g);
  if (wk.pix0 >= wk.npix) return;
  const float slope = has_act ? __ldg(slope_dev) : 0.f;
  float sc[8], sh[8];
  pload8(scale + wk.cg * 8, sc);
  pload8(shift + wk.cg * 8, sh);
  for (size_t pix = wk.pix0; pix < wk.npix; pix += wk.pstep) {
    int b, yy, x;
    pix_decode(g, pix, b, yy, x);
    float f[8];
    pload8(z + ppad_off(b, yy, x, g.h, g.w, zcs) + wk.cg * 8, f);
#pragma unroll
    for (int e = 0; e < 8; e++) {
      float u = __fadd_rn(__fmul_rn(f[e], sc[e]), sh[e]);   // x*alpha + beta, unfused like ATen's CPU kernel
      if (has_act) u = u > 0.f ? u : slope * u;
      f[e] = u;
    }
    if (res) {
      float r[8];
      split_load8(res + ppad_off(b, yy, x, g.h, g.w, rcs) + wk.cg * 8, rlo, np, r);
#pragma unroll
      for (int e = 0; e < 8; e++) f[e] += r[e];
    }
    if (!up) {
      split_store8(y + ppad_off(b, yy, x, g.h, g.w, ycs) + wk.cg * 8, ylo, np, f);
    } else {
#pragma unroll
      for (int ry = 0; ry < 2; ry++)
#pragma unroll
        for (int rx = 0; rx < 2; rx++)
          split_store8(y + ppad_off(b, 2 * yy + ry, 2 * x + rx, 2 * g.h, 2 * g.w, ycs) + wk.cg * 8, ylo, np, f);
    }
  }
}

__device__ __forceinline__ void px_load_dy(const float* __restrict__ dy, int dcs, const PGeo& g, int b, int y, int x, int cg,
                                           int up, float* d) {
  if (!up) {
    pload8(dy + ppad_off(b, y, x, g.h, g.w, dcs) + cg * 8, d);
  } else {
#pragma unroll
    for (int e = 0; e < 8; e++) d[e] = 0.f;
#pragma unroll
    for (int ry = 0; ry < 2; ry++)
#pragma unroll
      for (int rx = 0; rx < 2; rx++) {
        float t[8];
        pload8(dy + ppad_off(b, 2 * y + ry, 2 * x + rx, 2 * g.h, 2 * g.w, dcs) + cg * 8, t);
#pragma unroll
        for (int e = 0; e < 8; e++) d[e] += t[e];
      }
  }
}

__global__ void __launch_bounds__(PXT) px_bn_act_bwd_reduce_kernel(const float* __restrict__ dy, int dcs, int up,
                                                                   const float* __restrict__ z, int zcs, PGeo g,
                                                                   const float* __restrict__ scale,
                                                                   const float* __restrict__ shift,
                                                                   const float* __restrict__ mean,
                                                                   const float* __restrict__ invstd,
                                                                   const float* __restrict__ slope_dev, int has_act,
                                                                   double* __restrict__ sums /*[2c+1]*/) {
  const PWalk wk = pwalk(g);
  if (wk.pix0 >= wk.npix) return;
  const float slope = has_act ? __ldg(slope_dev) : 0.f;
  float sc[8], sh[8], mu[8], is[8];
  pload8(scale + wk.cg * 8, sc);
  pload8(shift + wk.cg * 8, sh);
  pload8(mean + wk.cg * 8, mu);
  pload8(invstd + wk.cg * 8, is);
  double a1[8], a2[8], asl = 0.0;
#pragma unroll
  for (int e = 0; e < 8; e++) a1[e] = a2[e] = 0.0;
  for (size_t pix = wk.pix0; pix < wk.npix; pix += wk.pstep) {
    int b, y, x;
    pix_decode(g, pix, b, y, x);
    float f[8], d[8];
    pload8(z + ppad_off(b, y, x, g.h, g.w, zcs) + wk.cg * 8, f);
    px_load_dy(dy, dcs, g, b, y, x, wk.cg, up, d);
#pragma unroll
    for (int e = 0; e < 8; e++) {
      const float u = __fadd_rn(__fmul_rn(f[e], sc[e]), sh[e]);
      float du = d[e];
      if (has_act && !(u > 0.f)) {
        asl += (double)d[e] * (double)u;
        du *= slope;
      }
      const float zh = (f[e] - mu[e]) * is[e];
      a1[e] += (double)du;
      a2[e] += (double)du * (double)zh;
    }
  }
#pragma unroll
  for (int e = 0; e < 8; e++) {
    atomicAdd(&sums[wk.cg * 8 + e], a1[e]);
    atomicAdd(&sums[g.c + wk.cg * 8 + e], a2[e]);
  }
  if (has_act) atomicAdd(&sums[2 * g.c], asl);
}

// dz = scale*(du - mean(du) - zhat*mean(du*zhat)) (training) or scale*du (eval statistics) -> split planes;
// shortcut gradient (+)= dy in fp32
__global__ void __launch_bounds__(PXT) px_bn_act_bwd_apply_kernel(const float* __restrict__ dy, int dcs, int up,
                                                                  const float* __restrict__ z, int zcs, PGeo g,
                                                                  const float* __restrict__ scale,
                                                                  const float* __restrict__ shift,
                                                                  const float* __restrict__ mean,
                                                                  const float* __restrict__ invstd,
                                                                  const float* __restrict__ slope_dev, int has_act,
                                                                  int batch_stats, const double* __restrict__ sums,
                                                                  double inv_n, __nv_bfloat16* __restrict__ dz, int dzcs,
                                                                  int dzlo, float* __restrict__ gres, int gcs, int gres_acc, int np) {
  const PWalk wk = pwalk(g);
  if (wk.pix0 >= wk.npix) return;
  const float slope = has_act ? __ldg(slope_dev) : 0.f;
  float sc[8], sh[8], mu[8], is[8], m1[8], m2[8];
  pload8(scale + wk.cg * 8, sc);
  pload8(shift + wk.cg * 8, sh);
  pload8(mean + wk.cg * 8, mu);
  pload8(invstd + wk.cg * 8, is);
#pragma unroll
  for (int e = 0; e < 8; e++) {
    m1[e] = (float)(sums[wk.cg * 8 + e] * inv_n);
    m2[e] = (float)(sums[g.c + wk.cg * 8 + e] * inv_n);
  }
  for (size_t pix = wk.pix0; pix < wk.npix; pix += wk.pstep) {
    int b, y, x;
    pix_decode(g, pix, b, y, x);
    float f[8], d[8];
    pload8(z + ppad_off(b, y, x, g.h, g.w, zcs) + wk.cg * 8, f);
    px_load_dy(dy, dcs, g, b, y, x, wk.cg, up, d);
    if (gres) {
      float* gp = gres + ppad_off(b, y, x, g.h, g.w, gcs) + wk.cg * 8;
      float o[8];
      if (gres_acc) {
        pload8(gp, o);
#pragma unroll
        for (int e = 0; e < 8; e++) o[e] += d[e];
      } else {
#pragma unroll
        for (int e = 0; e < 8; e++) o[e] = d[e];
      }
      pstore8(gp, o);
    }
    float out[8];
#pragma unroll
    for (int e = 0; e < 8; e++) {
      const float u = __fadd_rn(__fmul_rn(f[e], sc[e]), sh[e]);
      float du = d[e];
      if (has_act && !(u > 0.f)) du *= slope;
      out[e] = batch_stats ? sc[e] * (du - m1[e] - (f[e] - mu[e]) * is[e] * m2[e]) : sc[e] * du;
    }
    split_store8(dz + ppad_off(b, y, x, g.h, g.w, dzcs) + wk.cg * 8, dzlo, np, out);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// layout kernels
// im2col of the 3-channel image (column = c*9 + kh*3 + kw, 27 real of 64) -> split planes
__global__ void __launch_bounds__(256) px_im2col_first_kernel(const float* __restrict__ img, int batch, int h, int w,
                                                              __nv_bfloat16* __restrict__ dst, int dcs, int dlo, int np) {
  const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (size_t)batch * h * w) return;
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
  __nv_bfloat16* o = dst + ppad_off(b, y, x, h, w, dcs);
#pragma unroll
  for (int q = 0; q < 4; q++) split_store8(o + q * 8, dlo, np, v + q * 8);
}

// fp32 padded NHWC (+ per-channel bias) -> plain fp32 NCHW [B, c, h, w]: the linear YOLO heads
__global__ void __launch_bounds__(256) px_to_nchw_kernel(const float* __restrict__ z, int zcs, int batch, int c, int h, int w,
                                                         const float* __restrict__ bias, float* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)batch * c * h * w;
  if (i >= total) return;
  const int x = (int)(i % w);
  const int y = (int)((i / w) % h);
  const int ch = (int)((i / ((size_t)w * h)) % c);
  const int b = (int)(i / ((size_t)w * h * c));
  float v = z[ppad_off(b, y, x, h, w, zcs) + ch];
  if (bias) v += bias[ch];
  out[i] = v;
}

// head gradient fp32 [B, na, ny, nx, no] -> split planes, channel = a*no + k (the head conv's filter index)
__global__ void __launch_bounds__(256) px_head_grad_kernel(const float* __restrict__ g, int batch, int na, int no, int ny,
                                                           int nx, __nv_bfloat16* __restrict__ dst, int dcs, int dlo, int np) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)batch * na * ny * nx * no;
  if (i >= total) return;
  const int k = (int)(i % no);
  const int x = (int)((i / no) % nx);
  const int y = (int)((i / ((size_t)no * nx)) % ny);
  const int a = (int)((i / ((size_t)no * nx * ny)) % na);
  const int b = (int)(i / ((size_t)no * nx * ny * na));
  split_store1(dst + ppad_off(b, y, x, ny, nx, dcs) + a * no + k, dlo, np, g[i]);
}

// adjoint of space-to-depth in fp32: gx[b, 2Y+py, 2X+px, c] (+)= dxs[b, Y, X, (py*2+px)*C + c]
__global__ void __launch_bounds__(256) px_depth_to_space_kernel(const float* __restrict__ dxs, int scs, PGeo g /*of gx*/,
                                                                float* __restrict__ gx, int gcs, int accumulate) {
  const size_t item = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int cgs = g.c >> 3;
  const size_t npix = (size_t)g.batch * g.h * g.w;
  if (item >= npix * cgs) return;
  const int cg = (int)(item % cgs);
  int b, y, x;
  pix_decode(g, item / cgs, b, y, x);
  const int ph = (y & 1) * 2 + (x & 1);
  float d[8];
  pload8(dxs + ppad_off(b, y >> 1, x >> 1, g.h >> 1, g.w >> 1, scs) + ph * g.c + cg * 8, d);
  float* gp = gx + ppad_off(b, y, x, g.h, g.w, gcs) + cg * 8;
  if (accumulate) {
    float o[8];
    pload8(gp, o);
#pragma unroll
    for (int e = 0; e < 8; e++) d[e] += o[e];
  }
  pstore8(gp, d);
}

// split planes -> fp32 NCHW (tests: read an activation back) and fp32 NCHW -> split planes (tests: feed one)
__global__ void __launch_bounds__(256) px_split_from_nchw_kernel(const float* __restrict__ src, int batch, int c, int h, int w,
                                                                 __nv_bfloat16* __restrict__ dst, int dcs, int dlo, int np) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)batch * c * h * w;
  if (i >= total) return;
  const int x = (int)(i % w);
  const int y = (int)((i / w) % h);
  const int ch = (int)((i / ((size_t)w * h)) % c);
  const int b = (int)(i / ((size_t)w * h * c));
  split_store1(dst + ppad_off(b, y, x, h, w, dcs) + ch, dlo, np, src[i]);
}

static inline PGeo mk_pgeo(int batch, int h, int w, int c) {
  PGeo g;
  g.batch = batch; g.h = h; g.w = w; g.c = c;
  return g;
}
static inline unsigned walk_blocks(const PGeo& g) {
  const int cgs = g.c >> 3;
  const int ppb = PXT / cgs;
  const size_t npix = (size_t)g.batch * g.h * g.w;
  size_t blocks = (npix + ppb - 1) / ppb;
  const size_t cap = (size_t)device_sm_count() * 16;
  return (unsigned)(blocks < cap ? (blocks < 1 ? 1 : blocks) : cap);
}

}  // namespace ryolo

using namespace ryolo;

#define PGEO_CHECK() RYOLO_ARG_CHECK(batch > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0 && c <= 2048)

extern "C" int ryolo_px_bn_stats(const float* z, int z_cstride, int batch, int h, int w, int c, double* sums, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(z && sums);
  PGEO_CHECK();
  const PGeo g = mk_pgeo(batch, h, w, c);
  RYOLO_CUDA_TRY(cudaMemsetAsync(sums, 0, sizeof(double) * 2 * c, stream));
  px_bn_stats_kernel<<<walk_blocks(g), PXT, 0, stream>>>(z, z_cstride, g, sums);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_px_bn_finalize(const double* sums, int c, double count, float eps, float momentum, const float* gamma,
                                    const float* beta, int eval_mode, float* mean, float* invstd, float* scale,
                                    float* shift, float* running_mean, float* running_var, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(gamma && beta && mean && invstd && scale && shift && c > 0);
  RYOLO_ARG_CHECK(eval_mode ? (running_mean && running_var) : (sums && count > 0.0));
  RYOLO_ARG_CHECK((running_mean == nullptr) == (running_var == nullptr));
  px_bn_finalize_kernel<<<(c + 127) / 128, 128, 0, stream>>>(sums, c, count, eps, momentum, gamma, beta, eval_mode ? 1 : 0,
                                                             mean, invstd, scale, shift, running_mean, running_var);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_px_bn_act_fwd(const float* z, int z_cstride, int batch, int h, int w, int c, const float* scale,
                                   const float* shift, const float* slope_dev, const void* residual, int res_cstride,
                                   int res_lo, void* y, int y_cstride, int y_lo, int upsample2x, int nplanes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(z && scale && shift && y);
  PGEO_CHECK();
  RYOLO_ARG_CHECK(!(residual && upsample2x));
  RYOLO_ARG_CHECK(y_cstride % 8 == 0 && y_lo % 8 == 0 && (!residual || (res_cstride % 8 == 0 && res_lo % 8 == 0)));
  const PGeo g = mk_pgeo(batch, h, w, c);
  px_bn_act_fwd_kernel<<<walk_blocks(g), PXT, 0, stream>>>(z, z_cstride, g, scale, shift, slope_dev, slope_dev != nullptr,
                                                           static_cast<const __nv_bfloat16*>(residual), res_cstride, res_lo,
                                                           static_cast<__nv_bfloat16*>(y), y_cstride, y_lo, upsample2x, nplanes);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_px_bn_act_bwd(const float* dy, int dy_cstride, int upsample2x, const float* z, int z_cstride, int batch,
                                   int h, int w, int c, const float* scale, const float* shift, const float* mean,
                                   const float* invstd, const float* slope_dev, int batch_stats, double* sums, void* dz,
                                   int dz_cstride, int dz_lo, float* gres, int gres_cstride, int gres_accumulate,
                                   int nplanes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(dy && z && scale && shift && mean && invstd && sums && dz);
  PGEO_CHECK();
  RYOLO_ARG_CHECK(!(gres && upsample2x));
  const PGeo g = mk_pgeo(batch, h, w, c);
  RYOLO_CUDA_TRY(cudaMemsetAsync(sums, 0, sizeof(double) * (2 * c + 1), stream));
  const unsigned blocks = walk_blocks(g);
  px_bn_act_bwd_reduce_kernel<<<blocks, PXT, 0, stream>>>(dy, dy_cstride, upsample2x, z, z_cstride, g, scale, shift, mean, invstd,
                                                          slope_dev, slope_dev != nullptr, sums);
  RYOLO_LAUNCH_CHECK();
  px_bn_act_bwd_apply_kernel<<<blocks, PXT, 0, stream>>>(dy, dy_cstride, upsample2x, z, z_cstride, g, scale, shift, mean, invstd,
                                                         slope_dev, slope_dev != nullptr, batch_stats, sums,
                                                         1.0 / ((double)batch * h * w), static_cast<__nv_bfloat16*>(dz),
                                                         dz_cstride, dz_lo, gres, gres_cstride, gres_accumulate, nplanes);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_px_im2col_first(const float* img, int batch, int h, int w, void* dst, int dst_cstride, int dst_lo,
                                     int nplanes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(img && dst && batch > 0 && h > 0 && w > 0 && dst_cstride % 8 == 0 && dst_lo % 8 == 0 && dst_lo >= 32);
  const size_t npix = (size_t)batch * h * w;
  px_im2col_first_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, stream>>>(img, batch, h, w, static_cast<__nv_bfloat16*>(dst),
                                                                            dst_cstride, dst_lo, nplanes);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_px_to_nchw(const float* z, int z_cstride, int batch, int c, int h, int w, const float* bias, float* out,
                                void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(z && out && batch > 0 && c > 0 && h > 0 && w > 0 && z_cstride >= c);
  const size_t total = (size_t)batch * c * h * w;
  px_to_nchw_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(z, z_cstride, batch, c, h, w, bias, out);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_px_head_grad(const float* g, int batch, int na, int no, int ny, int nx, void* dst, int dst_cstride,
                                  int dst_lo, int nplanes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(g && dst && batch > 0 && na > 0 && no > 0 && ny > 0 && nx > 0 && dst_lo >= na * no);
  const size_t total = (size_t)batch * na * no * ny * nx;
  px_head_grad_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(g, batch, na, no, ny, nx,
                                                                          static_cast<__nv_bfloat16*>(dst), dst_cstride, dst_lo, nplanes);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_px_depth_to_space(const float* dxs, int dxs_cstride, int batch, int h, int w, int c, float* gx,
                                       int gx_cstride, int accumulate, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(dxs && gx);
  PGEO_CHECK();
  RYOLO_ARG_CHECK(h % 2 == 0 && w % 2 == 0 && dxs_cstride >= 4 * c);
  const PGeo g = mk_pgeo(batch, h, w, c);
  const size_t items = (size_t)batch * h * w * (c >> 3);
  px_depth_to_space_kernel<<<(unsigned)((items + 255) / 256), 256, 0, stream>>>(dxs, dxs_cstride, g, gx, gx_cstride, accumulate);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_px_split_from_nchw(const float* src, int batch, int c, int h, int w, void* dst, int dst_cstride,
                                        int dst_lo, int nplanes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(src && dst && batch > 0 && c > 0 && h > 0 && w > 0 && dst_lo >= c);
  const size_t total = (size_t)batch * c * h * w;
  px_split_from_nchw_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(src, batch, c, h, w,
                                                                                static_cast<__nv_bfloat16*>(dst), dst_cstride,
                                                                                dst_lo, nplanes);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}
