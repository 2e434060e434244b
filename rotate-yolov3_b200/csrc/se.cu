// Squeeze-and-excitation block of the reference's *_se.cfg graphs (model/models.py:16-31 SELayer; built for `[se]` blocks at
// models.py:88-90; cfg/ICDAR/yolov3_608_se.cfg, cfg/HRSC+/yolov3_512_se.cfg): per image and channel
//     s = sigmoid(W2 . relu(W1 . mean_{h,w} x)),   x <- x * s
// on a padded-NHWC bf16 activation, in place (the scaled tensor is what every later block reads).  Eval path:
// three small memory-bound kernels -- channel means (fp32 sums of the bf16 tensor), the two bias-free linear layers of
// one image in one CTA, and the channel-wise rescale.
//
// Training / routed-input path (ryolo_se_fwd / ryolo_se_bwd): out of place, u = x * s into a buffer of its own so that the
// unscaled x stays readable by the shortcut three blocks later (`from=-4`) and by concat routes, and deterministic: every
// reduction (channel sums, dot products, batch sums of the weight gradients) runs in a fixed order with no float atomics.
// An image's spatial sums are split into se_nsplit(h, w, c) contiguous pixel spans that depend on the image shape only,
// so each image's numbers are the same bits in any batch.
#include <cuda_bf16.h>

#include "common.cuh"

namespace ryolo {

__device__ __forceinline__ size_t se_pad_off(int b, int y, int x, int h, int w, int cs) {
  return (((size_t)b * (h + 2) + y + 1) * (w + 2) + x + 1) * cs;
}

// sums[b, c] += sum over a span of interior rows; grid (row spans, batch); thread = 8-channel group x pixel stride
__global__ void __launch_bounds__(256) se_pool_kernel(const __nv_bfloat16* __restrict__ x, int cs, int h, int w, int c,
                                                      int rows_per_block, float* __restrict__ sums) {
  const int b = blockIdx.y;
  const int cgs = c >> 3;
  const int cg = threadIdx.x % cgs, p0 = threadIdx.x / cgs, pstep = 256 / cgs;
  if (p0 >= pstep) return;
  const int y0 = blockIdx.x * rows_per_block, y1 = min(h, y0 + rows_per_block);
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; e++) acc[e] = 0.f;
  for (int y = y0; y < y1; y++) {
    const __nv_bfloat16* row = x + se_pad_off(b, y, 0, h, w, cs) + cg * 8;
    for (int xx = p0; xx < w; xx += pstep) {
      const uint4 v = *reinterpret_cast<const uint4*>(row + (size_t)xx * cs);
      const __nv_bfloat162* hp = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
      for (int e = 0; e < 4; e++) {
        const float2 f = __bfloat1622float2(hp[e]);
        acc[2 * e] += f.x;
        acc[2 * e + 1] += f.y;
      }
    }
  }
#pragma unroll
  for (int e = 0; e < 8; e++) atomicAdd(&sums[(size_t)b * c + cg * 8 + e], acc[e]);
}

// one CTA per image: hidden = relu(W1 [cr, c] . mean), s = sigmoid(W2 [c, cr] . hidden)
__global__ void __launch_bounds__(256) se_fc_kernel(const float* __restrict__ sums, float inv_hw, const float* __restrict__ w1,
                                                    const float* __restrict__ w2, int c, int cr, float* __restrict__ scale) {
  extern __shared__ float se_sm[];     // [c] means, [cr] hidden
  float* mean = se_sm;
  float* hid = se_sm + c;
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < c; i += 256) mean[i] = sums[(size_t)b * c + i] * inv_hw;
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j = warp; j < cr; j += 8) {
    float a = 0.f;
    for (int i = lane; i < c; i += 32) a = fmaf(w1[(size_t)j * c + i], mean[i], a);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) hid[j] = fmaxf(a, 0.f);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < c; i += 256) {
    float a = 0.f;
    for (int j = 0; j < cr; j++) a = fmaf(w2[(size_t)i * cr + j], hid[j], a);
    scale[(size_t)b * c + i] = 1.f / (1.f + expf(-a));
  }
}

__global__ void __launch_bounds__(256) se_scale_kernel(__nv_bfloat16* __restrict__ x, int cs, int batch, int h, int w, int c,
                                                       const float* __restrict__ scale) {
  const size_t item = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int cgs = c >> 3;
  const size_t npix = (size_t)batch * h * w;
  if (item >= npix * cgs) return;
  const int cg = (int)(item % cgs);
  const size_t pix = item / cgs;
  const int xx = (int)(pix % w), y = (int)((pix / w) % h), b = (int)(pix / ((size_t)w * h));
  __nv_bfloat16* p = x + se_pad_off(b, y, xx, h, w, cs) + cg * 8;
  uint4 v = *reinterpret_cast<const uint4*>(p);
  __nv_bfloat162* hp = reinterpret_cast<__nv_bfloat162*>(&v);
  const float* s = scale + (size_t)b * c + cg * 8;
#pragma unroll
  for (int e = 0; e < 4; e++) {
    const float2 f = __bfloat1622float2(hp[e]);
    hp[e] = __floats2bfloat162_rn(f.x * s[2 * e], f.y * s[2 * e + 1]);
  }
  *reinterpret_cast<uint4*>(p) = v;
}


// ---------------------------------------------------------------------------------------------------------------------
// Training path.  Pixel spans: ~4096 16-byte items per CTA, at most 128 spans per image.
inline int se_nsplit(int h, int w, int c) {
  const long long items = (long long)h * w * (c >> 3);
  const long long n = (items + 4095) / 4096;
  return (int)(n < 1 ? 1 : (n > 128 ? 128 : n));
}

// part[b, span, c] = sum over the span's pixels of a (kDot: of a * g; bf16 products are exact in fp32).  Thread =
// (8-channel group, pixel lane): it adds every lanes-th pixel of the span in order; the lanes of a channel are then added
// in lane order.
template <bool kDot>
__global__ void __launch_bounds__(256) se_partial_kernel(const __nv_bfloat16* __restrict__ a, int acs,
                                                         const __nv_bfloat16* __restrict__ g, int gcs, int h, int w, int c,
                                                         int span, float* __restrict__ part) {
  __shared__ float red[2048];
  const int b = blockIdx.y, sp = blockIdx.x, nsplit = gridDim.x;
  const int cgs = c >> 3, lanes = 256 / cgs;
  const int cg = threadIdx.x % cgs, lane = threadIdx.x / cgs;
  const int p0 = sp * span, p1 = min(h * w, p0 + span);
  if (lane < lanes) {
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; e++) acc[e] = 0.f;
    for (int p = p0 + lane; p < p1; p += lanes) {
      const int y = p / w, xx = p - y * w;
      const uint4 va = *reinterpret_cast<const uint4*>(a + se_pad_off(b, y, xx, h, w, acs) + cg * 8);
      const __nv_bfloat162* ha = reinterpret_cast<const __nv_bfloat162*>(&va);
      if (kDot) {
        const uint4 vg = *reinterpret_cast<const uint4*>(g + se_pad_off(b, y, xx, h, w, gcs) + cg * 8);
        const __nv_bfloat162* hg = reinterpret_cast<const __nv_bfloat162*>(&vg);
#pragma unroll
        for (int e = 0; e < 4; e++) {
          const float2 fa = __bfloat1622float2(ha[e]), fg = __bfloat1622float2(hg[e]);
          acc[2 * e] = fmaf(fa.x, fg.x, acc[2 * e]);
          acc[2 * e + 1] = fmaf(fa.y, fg.y, acc[2 * e + 1]);
        }
      } else {
#pragma unroll
        for (int e = 0; e < 4; e++) {
          const float2 fa = __bfloat1622float2(ha[e]);
          acc[2 * e] += fa.x;
          acc[2 * e + 1] += fa.y;
        }
      }
    }
#pragma unroll
    for (int e = 0; e < 8; e++) red[lane * c + cg * 8 + e] = acc[e];
  }
  __syncthreads();
  for (int ch = threadIdx.x; ch < c; ch += 256) {
    float s = 0.f;
    for (int l = 0; l < lanes; l++) s += red[l * c + ch];
    part[((size_t)b * nsplit + sp) * c + ch] = s;
  }
}

// one CTA per image: m = (sum of the spans in span order) / hw, p = W1 m (warp per hidden unit: lane-strided partial dot
// products, then a 5-level butterfly), s = sigmoid(W2 relu(p)) (thread per channel, hidden units in order)
__global__ void __launch_bounds__(256) se_fc_fwd_kernel(const float* __restrict__ part, int nsplit, int hw,
                                                        const float* __restrict__ w1, const float* __restrict__ w2, int c,
                                                        int cr, float* __restrict__ m, float* __restrict__ p,
                                                        float* __restrict__ s) {
  extern __shared__ float se_sm[];     // [c] means, [cr] hidden
  float* mean = se_sm;
  float* hid = se_sm + c;
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < c; i += 256) {
    float acc = 0.f;
    for (int sp = 0; sp < nsplit; sp++) acc += part[((size_t)b * nsplit + sp) * c + i];
    const float mv = acc / (float)hw;
    mean[i] = mv;
    m[(size_t)b * c + i] = mv;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j = warp; j < cr; j += 8) {
    float a = 0.f;
    for (int i = lane; i < c; i += 32) a = fmaf(w1[(size_t)j * c + i], mean[i], a);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) {
      p[(size_t)b * cr + j] = a;
      hid[j] = a > 0.f ? a : 0.f;
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < c; i += 256) {
    float a = 0.f;
    for (int j = 0; j < cr; j++) a = fmaf(w2[(size_t)i * cr + j], hid[j], a);
    s[(size_t)b * c + i] = 1.f / (1.f + expf(-a));
  }
}

// u = bf16(x * s) on the interior (u's halo is never written); one thread per 8-channel group and pixel
__global__ void __launch_bounds__(256) se_scale_out_kernel(const __nv_bfloat16* __restrict__ x, int xcs,
                                                           __nv_bfloat16* __restrict__ u, int ucs, int items, FastDiv fcgs,
                                                           FastDiv fw, FastDiv fh, int c, const float* __restrict__ s) {
  const int item = blockIdx.x * blockDim.x + threadIdx.x;
  if (item >= items) return;
  int pix, cg, row, xx, b, y;
  fast_divmod(item, fcgs, pix, cg);
  fast_divmod(pix, fw, row, xx);
  fast_divmod(row, fh, b, y);
  const int h = fh.d, w = fw.d;
  uint4 v = *reinterpret_cast<const uint4*>(x + se_pad_off(b, y, xx, h, w, xcs) + cg * 8);
  __nv_bfloat162* hp = reinterpret_cast<__nv_bfloat162*>(&v);
  const float4 s0 = *reinterpret_cast<const float4*>(s + (size_t)b * c + cg * 8);
  const float4 s1 = *reinterpret_cast<const float4*>(s + (size_t)b * c + cg * 8 + 4);
  const float sv[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
#pragma unroll
  for (int e = 0; e < 4; e++) {
    const float2 f = __bfloat1622float2(hp[e]);
    hp[e] = __floats2bfloat162_rn(f.x * sv[2 * e], f.y * sv[2 * e + 1]);
  }
  *reinterpret_cast<uint4*>(u + se_pad_off(b, y, xx, h, w, ucs) + cg * 8) = v;
}

// one CTA per image: ds = sum of the spans in span order, da = ds s (1 - s), dhid = (W2^T da) [p > 0], dm = W1^T dhid,
// dmh = dm / hw (the per-pixel share that the apply kernel adds)
__global__ void __launch_bounds__(256) se_fc_bwd_kernel(const float* __restrict__ part, int nsplit, int hw,
                                                        const float* __restrict__ w1, const float* __restrict__ w2, int c,
                                                        int cr, const float* __restrict__ p, const float* __restrict__ s,
                                                        float* __restrict__ ds, float* __restrict__ da_out,
                                                        float* __restrict__ dhid_out, float* __restrict__ dm,
                                                        float* __restrict__ dmh) {
  extern __shared__ float se_sm[];     // [c] da, [cr] dhid
  float* da = se_sm;
  float* dh = se_sm + c;
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < c; i += 256) {
    float acc = 0.f;
    for (int sp = 0; sp < nsplit; sp++) acc += part[((size_t)b * nsplit + sp) * c + i];
    ds[(size_t)b * c + i] = acc;
    const float sv = s[(size_t)b * c + i];
    const float d = acc * (sv * (1.f - sv));
    da[i] = d;
    da_out[(size_t)b * c + i] = d;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j = warp; j < cr; j += 8) {
    float a = 0.f;
    for (int i = lane; i < c; i += 32) a = fmaf(w2[(size_t)i * cr + j], da[i], a);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) {
      const float d = p[(size_t)b * cr + j] > 0.f ? a : 0.f;     // relu'(0) = 0, like torch
      dh[j] = d;
      dhid_out[(size_t)b * cr + j] = d;
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < c; i += 256) {
    float a = 0.f;
    for (int j = 0; j < cr; j++) a = fmaf(w1[(size_t)j * c + i], dh[j], a);
    dm[(size_t)b * c + i] = a;
    dmh[(size_t)b * c + i] = a / (float)hw;
  }
}

// weight gradients, one thread per element, images added in order 0..batch-1:
// gw2[i, j] = sum_b da[b, i] relu(p[b, j]),  gw1[j, i] = sum_b dhid[b, j] m[b, i]
__global__ void __launch_bounds__(256) se_wgrad_kernel(const float* __restrict__ da, const float* __restrict__ dhid,
                                                       const float* __restrict__ p, const float* __restrict__ m, int batch,
                                                       int c, int cr, float* __restrict__ gw1, float* __restrict__ gw2) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = c * cr;
  if (e >= 2 * n) return;
  float acc = 0.f;
  if (e < n) {
    const int i = e / cr, j = e - i * cr;
    for (int b = 0; b < batch; b++) {
      const float pv = p[(size_t)b * cr + j];
      acc = fmaf(da[(size_t)b * c + i], pv > 0.f ? pv : 0.f, acc);
    }
    gw2[e] = acc;
  } else {
    const int f = e - n, j = f / c, i = f - j * c;
    for (int b = 0; b < batch; b++) acc = fmaf(dhid[(size_t)b * cr + j], m[(size_t)b * c + i], acc);
    gw1[f] = acc;
  }
}

// gx = bf16([gx +] gu s + dmh), fp32 arithmetic, one rounding
__global__ void __launch_bounds__(256) se_apply_kernel(const __nv_bfloat16* __restrict__ gu, int gucs,
                                                       __nv_bfloat16* __restrict__ gx, int gxcs, int accumulate, int items,
                                                       FastDiv fcgs, FastDiv fw, FastDiv fh, int c,
                                                       const float* __restrict__ s, const float* __restrict__ dmh) {
  const int item = blockIdx.x * blockDim.x + threadIdx.x;
  if (item >= items) return;
  int pix, cg, row, xx, b, y;
  fast_divmod(item, fcgs, pix, cg);
  fast_divmod(pix, fw, row, xx);
  fast_divmod(row, fh, b, y);
  const int h = fh.d, w = fw.d;
  const uint4 vg = *reinterpret_cast<const uint4*>(gu + se_pad_off(b, y, xx, h, w, gucs) + cg * 8);
  const __nv_bfloat162* hg = reinterpret_cast<const __nv_bfloat162*>(&vg);
  __nv_bfloat16* po = gx + se_pad_off(b, y, xx, h, w, gxcs) + cg * 8;
  uint4 vo = make_uint4(0u, 0u, 0u, 0u);
  if (accumulate) vo = *reinterpret_cast<const uint4*>(po);
  __nv_bfloat162* ho = reinterpret_cast<__nv_bfloat162*>(&vo);
  const size_t so = (size_t)b * c + cg * 8;
  const float4 s0 = *reinterpret_cast<const float4*>(s + so), s1 = *reinterpret_cast<const float4*>(s + so + 4);
  const float4 d0 = *reinterpret_cast<const float4*>(dmh + so), d1 = *reinterpret_cast<const float4*>(dmh + so + 4);
  const float sv[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
  const float dv[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
#pragma unroll
  for (int e = 0; e < 4; e++) {
    const float2 fg = __bfloat1622float2(hg[e]);
    float lo = fmaf(fg.x, sv[2 * e], dv[2 * e]), hi = fmaf(fg.y, sv[2 * e + 1], dv[2 * e + 1]);
    if (accumulate) {
      const float2 fo = __bfloat1622float2(ho[e]);
      lo += fo.x;
      hi += fo.y;
    }
    ho[e] = __floats2bfloat162_rn(lo, hi);
  }
  *reinterpret_cast<uint4*>(po) = vo;
}

struct SeWs {
  float *part, *da, *dhid, *dmh;
};
inline size_t se_ws_carve(void* base, int batch, int h, int w, int c, int reduced, SeWs* out) {
  Carver cv(base);
  SeWs ws;
  ws.part = cv.take<float>((size_t)batch * se_nsplit(h, w, c) * c);
  ws.da = cv.take<float>((size_t)batch * c);
  ws.dhid = cv.take<float>((size_t)batch * reduced);
  ws.dmh = cv.take<float>((size_t)batch * c);
  if (out) *out = ws;
  return cv.off;
}
}  // namespace ryolo

using namespace ryolo;

extern "C" int ryolo_se_block(void* x, int x_cstride, int batch, int h, int w, int c, const float* w1, const float* w2,
                              int reduced, float* sums_scratch, float* scale_scratch, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(x && w1 && w2 && sums_scratch && scale_scratch && batch > 0 && h > 0 && w > 0);
  RYOLO_ARG_CHECK(c > 0 && c % 8 == 0 && c <= 2048 && 256 % (c >> 3) == 0 && reduced > 0 && reduced <= c && batch <= 65535);
  RYOLO_ARG_CHECK(x_cstride >= c && x_cstride % 8 == 0);
  RYOLO_CUDA_TRY(cudaMemsetAsync(sums_scratch, 0, sizeof(float) * (size_t)batch * c, stream));
  const int rpb = h > 64 ? (h + 63) / 64 : 1;
  dim3 gp((h + rpb - 1) / rpb, batch);
  se_pool_kernel<<<gp, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), x_cstride, h, w, c, rpb, sums_scratch);
  RYOLO_LAUNCH_CHECK();
  se_fc_kernel<<<batch, 256, (size_t)(c + reduced) * sizeof(float), stream>>>(sums_scratch, 1.0f / ((float)h * w), w1, w2, c,
                                                                             reduced, scale_scratch);
  RYOLO_LAUNCH_CHECK();
  const size_t items = (size_t)batch * h * w * (c >> 3);
  se_scale_kernel<<<(unsigned)((items + 255) / 256), 256, 0, stream>>>(static_cast<__nv_bfloat16*>(x), x_cstride, batch, h, w, c,
                                                                      scale_scratch);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

#define SE_SHAPE_CHECK()                                                                                                  \
  RYOLO_ARG_CHECK(batch > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0 && c <= 2048 && reduced > 0 && reduced <= c);     \
  RYOLO_ARG_CHECK(batch <= 65535 && (long long)batch * h * w * (c >> 3) < (1ll << 31))

extern "C" size_t ryolo_se_workspace_bytes(int batch, int h, int w, int c, int reduced) {
  if (batch <= 0 || h <= 0 || w <= 0 || c <= 0 || reduced <= 0) return 0;
  return se_ws_carve(nullptr, batch, h, w, c, reduced, nullptr) + 256;
}

static bool se_aligned(const void* p) { return ((uintptr_t)p & 15) == 0; }

extern "C" int ryolo_se_fwd(const void* x, int x_cstride, void* u, int u_cstride, int batch, int h, int w, int c,
                            const float* w1, const float* w2, int reduced, float* m, float* p, float* s, void* workspace,
                            size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(x && u && w1 && w2 && m && p && s && workspace);
  SE_SHAPE_CHECK();
  RYOLO_ARG_CHECK(x_cstride >= c && x_cstride % 8 == 0 && u_cstride >= c && u_cstride % 8 == 0 && se_aligned(x) &&
                  se_aligned(u) && se_aligned(s));
  RYOLO_ARG_CHECK(workspace_bytes >= ryolo_se_workspace_bytes(batch, h, w, c, reduced));
  SeWs ws;
  se_ws_carve(reinterpret_cast<void*>(align_up((uintptr_t)workspace, 256)), batch, h, w, c, reduced, &ws);
  const int nsplit = se_nsplit(h, w, c), span = (h * w + nsplit - 1) / nsplit;
  se_partial_kernel<false><<<dim3(nsplit, batch), 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), x_cstride, nullptr,
                                                                   0, h, w, c, span, ws.part);
  RYOLO_LAUNCH_CHECK();
  se_fc_fwd_kernel<<<batch, 256, (size_t)(c + reduced) * sizeof(float), stream>>>(ws.part, nsplit, h * w, w1, w2, c, reduced,
                                                                                 m, p, s);
  RYOLO_LAUNCH_CHECK();
  const int items = batch * h * w * (c >> 3);
  se_scale_out_kernel<<<(items + 255) / 256, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), x_cstride,
                                                               static_cast<__nv_bfloat16*>(u), u_cstride, items,
                                                               make_fastdiv(c >> 3), make_fastdiv(w), make_fastdiv(h), c, s);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_se_bwd(const void* gu, int gu_cstride, const void* x, int x_cstride, void* gx, int gx_cstride,
                            int accumulate, int batch, int h, int w, int c, const float* w1, const float* w2, int reduced,
                            const float* m, const float* p, const float* s, float* ds, float* dm, float* gw1, float* gw2,
                            void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(gu && x && gx && w1 && w2 && m && p && s && ds && dm && gw1 && gw2 && workspace);
  SE_SHAPE_CHECK();
  RYOLO_ARG_CHECK(gu_cstride >= c && gu_cstride % 8 == 0 && x_cstride >= c && x_cstride % 8 == 0 && gx_cstride >= c &&
                  gx_cstride % 8 == 0 && se_aligned(gu) && se_aligned(x) && se_aligned(gx) && se_aligned(s));
  RYOLO_ARG_CHECK(workspace_bytes >= ryolo_se_workspace_bytes(batch, h, w, c, reduced));
  SeWs ws;
  se_ws_carve(reinterpret_cast<void*>(align_up((uintptr_t)workspace, 256)), batch, h, w, c, reduced, &ws);
  const int nsplit = se_nsplit(h, w, c), span = (h * w + nsplit - 1) / nsplit;
  se_partial_kernel<true><<<dim3(nsplit, batch), 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(gu), gu_cstride,
                                                                  static_cast<const __nv_bfloat16*>(x), x_cstride, h, w, c,
                                                                  span, ws.part);
  RYOLO_LAUNCH_CHECK();
  se_fc_bwd_kernel<<<batch, 256, (size_t)(c + reduced) * sizeof(float), stream>>>(ws.part, nsplit, h * w, w1, w2, c, reduced,
                                                                                 p, s, ds, ws.da, ws.dhid, dm, ws.dmh);
  RYOLO_LAUNCH_CHECK();
  se_wgrad_kernel<<<(2 * c * reduced + 255) / 256, 256, 0, stream>>>(ws.da, ws.dhid, p, m, batch, c, reduced, gw1, gw2);
  RYOLO_LAUNCH_CHECK();
  const int items = batch * h * w * (c >> 3);
  se_apply_kernel<<<(items + 255) / 256, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(gu), gu_cstride,
                                                           static_cast<__nv_bfloat16*>(gx), gx_cstride, accumulate, items,
                                                           make_fastdiv(c >> 3), make_fastdiv(w), make_fastdiv(h), c, s,
                                                           ws.dmh);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}
