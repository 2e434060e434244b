// Training augmentation of letterboxed uint8 HWC BGR images (utils/augment.py, utils/datasets.py:470-500), byte for
// byte what the reference computes on the host with cv2 and numpy:
//
//   ryolo_augment_warp    random_affine's cv2.warpAffine(INTER_AREA, which warpAffine runs as INTER_LINEAR, border
//                         128): cv2's fixed-point remap.  Per output row y, X0 = rint((m1 * y + m2) * 1024) + 16 and
//                         per column adelta = rint(m0 * x * 1024) (doubles, each product and sum rounded on its own:
//                         explicit __dmul_rn / __dadd_rn, no FMA); X = (X0 + adelta) >> 5 holds the source pixel in
//                         its high bits and a 5-bit fraction in its low 5; the four taps carry 15-bit weights
//                         (32 - ay)(32 - ax) * 32, ..., taps outside the image read 128, and (sum + 2^14) >> 15.
//                         The same launch writes each row's maximum, which Gamma needs over the whole image.
//   ryolo_augment_finish  Gamma: uint8(pow(v / M, gm) * M) in float64 through a 256-entry table per image (M the
//                         image maximum from the row maxima; M = 0 leaves 0).  HSV: cv2's 8-bit BGR2HSV (12-bit
//                         fixed-point divisions), S and V times the float32 factor, clipped at 255 and truncated
//                         as numpy's assignment into uint8 does, and cv2's 8-bit HSV2BGR, float32 inside.  cv2 runs
//                         HSV2BGR as vector code over blocks of 32 pixels of a row (AVX2: 4 x 8 float lanes), with
//                         the products 1 - s * h fused and the result truncated, and the rest of the row as scalar
//                         code that rounds instead; the column of a pixel before the flips picks the path.  Then the
//                         flips as index remaps, BGR->RGB and /255 (IEEE division; fp16 rounds that quotient once).
//
// One CTA per output row of one job (grid.y = job); consecutive threads take consecutive pixels of the row.
#include <cuda_fp16.h>

#include "common.cuh"

namespace ryolo {

constexpr int kAugThreads = 256;   // the finish kernel fills its 256-entry tables with one thread per entry
constexpr int kHsvVecPixels = 32;  // pixels per vector iteration of cv2's HSV2BGR_b (AVX2 dispatch)

template <typename T>
__device__ __forceinline__ T aug_cast(float v);
template <>
__device__ __forceinline__ float aug_cast<float>(float v) { return v; }
template <>
__device__ __forceinline__ __half aug_cast<__half>(float v) { return __float2half_rn(v); }

__device__ __forceinline__ int block_max(int v, int* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  v = 0;
  for (int i = 0; i < kAugThreads / 32; i++) v = max(v, red[i]);
  return v;
}

__global__ void __launch_bounds__(kAugThreads)
    augment_warp_kernel(const ryolo_warp_job* __restrict__ jobs, uint8_t* __restrict__ rowmax, int h, int w) {
  __shared__ int red[kAugThreads / 32];
  const ryolo_warp_job& jb = jobs[blockIdx.y];
  const int y = blockIdx.x;
  int mx = 0;
  if (jb.warp) {
    const double m0 = jb.m[0], m1 = jb.m[1], m2 = jb.m[2], m3 = jb.m[3], m4 = jb.m[4], m5 = jb.m[5];
    const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m1, (double)y), m2), 1024.0)) + 16;
    const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m4, (double)y), m5), 1024.0)) + 16;
    uint8_t* o = jb.dst + (size_t)y * w * 3;
    for (int x = threadIdx.x; x < w; x += kAugThreads) {
      const int X = (X0 + __double2int_rn(__dmul_rn(__dmul_rn(m0, (double)x), 1024.0))) >> 5;
      const int Y = (Y0 + __double2int_rn(__dmul_rn(__dmul_rn(m3, (double)x), 1024.0))) >> 5;
      const int sx = min(max(X >> 5, -32768), 32767), sy = min(max(Y >> 5, -32768), 32767);   // saturate_cast<short>
      const int ax = X & 31, ay = Y & 31;
      const int wt[4] = {(32 - ay) * (32 - ax) * 32, (32 - ay) * ax * 32, ay * (32 - ax) * 32, ay * ax * 32};
      int acc[3] = {0, 0, 0};
#pragma unroll
      for (int t = 0; t < 4; t++) {
        const int tx = sx + (t & 1), ty = sy + (t >> 1);
        const bool in = tx >= 0 && tx < w && ty >= 0 && ty < h;
        const uint8_t* p = jb.src + (long long)ty * jb.src_stride + 3LL * tx;
#pragma unroll
        for (int c = 0; c < 3; c++) acc[c] += (in ? (int)__ldg(p + c) : 128) * wt[t];
      }
#pragma unroll
      for (int c = 0; c < 3; c++) {
        const int v = (acc[c] + (1 << 14)) >> 15;
        o[3 * x + c] = (uint8_t)v;
        mx = max(mx, v);
      }
    }
  } else {
    const uint8_t* r = jb.src + (long long)y * jb.src_stride;
    for (int i = threadIdx.x; i < 3 * w; i += kAugThreads) mx = max(mx, (int)__ldg(r + i));
  }
  mx = block_max(mx, red);
  if (threadIdx.x == 0) rowmax[(size_t)jb.image * h + y] = (uint8_t)mx;
}

// cv2's 8-bit BGR2HSV (hrange 180): h in [0, 180), s, v in [0, 255]
__device__ __forceinline__ void bgr2hsv(int b, int g, int r, const int* sdiv, const int* hdiv, int& h, int& s,
                                        int& v) {
  v = max(max(b, g), r);
  const int vmin = min(min(b, g), r);
  const int diff = v - vmin;
  s = (diff * sdiv[v] + (1 << 11)) >> 12;
  int hh = v == r ? g - b : (v == g ? b - r + 2 * diff : r - g + 4 * diff);
  hh = (hh * hdiv[diff] + (1 << 11)) >> 12;
  h = hh < 0 ? hh + 180 : hh;
}

// cv2's 8-bit HSV2BGR (hrange 180), vector form (vec: fused 1 - s * h, truncation) or scalar tail (rounding)
__device__ __forceinline__ void hsv2bgr(int h, int s, int v, bool vec, int bgr[3]) {
  const float sf = __fmul_rn((float)s, __fdiv_rn(1.f, 255.f));
  const float vf = __fmul_rn((float)v, __fdiv_rn(1.f, 255.f));
  const float hh = __fmul_rn((float)h, __fdiv_rn(6.f, 180.f));
  const float pre = truncf(hh);
  const float fr = __fsub_rn(hh, pre);
  const int sector = (int)__fsub_rn(pre, __fmul_rn(truncf(__fmul_rn(pre, __fdiv_rn(1.f, 6.f))), 6.f));
  const float t0 = vf;
  const float t1 = __fmul_rn(vf, __fsub_rn(1.f, sf));
  const float t2 = __fmul_rn(vf, __fmaf_rn(-sf, fr, 1.f));
  const float t3 = __fmul_rn(vf, __fmaf_rn(-sf, __fsub_rn(1.f, fr), 1.f));
  float c[3];                                                // B, G, R by sector
  switch (sector) {
    case 0: c[0] = t1, c[1] = t3, c[2] = t0; break;
    case 1: c[0] = t1, c[1] = t0, c[2] = t2; break;
    case 2: c[0] = t3, c[1] = t0, c[2] = t1; break;
    case 3: c[0] = t0, c[1] = t2, c[2] = t1; break;
    case 4: c[0] = t0, c[1] = t1, c[2] = t3; break;
    default: c[0] = t2, c[1] = t1, c[2] = t0; break;
  }
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const float o = __fmul_rn(c[k], 255.f);
    const int q = vec ? (int)truncf(o) : __float2int_rn(o);
    bgr[k] = q < 0 ? 0 : (q > 255 ? 255 : q);
  }
}

template <typename T>
__global__ void __launch_bounds__(kAugThreads)
    augment_finish_kernel(const ryolo_finish_job* __restrict__ jobs, const uint8_t* __restrict__ rowmax,
                          T* __restrict__ out, int h, int w) {
  __shared__ int gtab[256], sdiv[256], hdiv[256];
  __shared__ int red[kAugThreads / 32];
  const ryolo_finish_job& jb = jobs[blockIdx.y];
  const int b = blockIdx.y, y = blockIdx.x, t = threadIdx.x;
  const int flags = jb.flags;
  if (flags & RYOLO_AUG_GAMMA) {
    int m = 0;
    for (int i = t; i < h; i += kAugThreads) m = max(m, (int)__ldg(rowmax + (size_t)b * h + i));
    m = block_max(m, red);
    const double dm = (double)m;
    gtab[t] = (m == 0 || t > m) ? 0 : (int)__dmul_rn(pow(__ddiv_rn((double)t, dm), jb.gamma), dm);
  }
  if (flags & RYOLO_AUG_HSV) {
    sdiv[t] = t ? __double2int_rn(__ddiv_rn((double)(255 << 12), (double)t)) : 0;
    hdiv[t] = t ? __double2int_rn(__ddiv_rn((double)(180 << 12), __dmul_rn(6.0, (double)t))) : 0;
  }
  __syncthreads();
  const size_t plane = (size_t)h * w;
  T* o = out + (size_t)b * 3 * plane + (size_t)y * w;
  const int sy = (flags & RYOLO_AUG_VFLIP) ? h - 1 - y : y;
  const uint8_t* row = jb.src + (long long)sy * jb.src_stride;
  const int vec_end = w / kHsvVecPixels * kHsvVecPixels;
  for (int x = t; x < w; x += kAugThreads) {
    const int sx = (flags & RYOLO_AUG_HFLIP) ? w - 1 - x : x;
    int px[3] = {__ldg(row + 3 * sx), __ldg(row + 3 * sx + 1), __ldg(row + 3 * sx + 2)};    // B, G, R
    if (flags & RYOLO_AUG_GAMMA) px[0] = gtab[px[0]], px[1] = gtab[px[1]], px[2] = gtab[px[2]];
    if (flags & RYOLO_AUG_HSV) {
      int hh, ss, vv;
      bgr2hsv(px[0], px[1], px[2], sdiv, hdiv, hh, ss, vv);
      ss = (int)fminf(__fmul_rn((float)ss, jb.hsv_s), 255.f);
      vv = (int)fminf(__fmul_rn((float)vv, jb.hsv_v), 255.f);
      hsv2bgr(hh, ss, vv, sx < vec_end, px);
    }
    o[x] = aug_cast<T>(__fdiv_rn((float)px[2], 255.f));
    o[plane + x] = aug_cast<T>(__fdiv_rn((float)px[1], 255.f));
    o[2 * plane + x] = aug_cast<T>(__fdiv_rn((float)px[0], 255.f));
  }
}

}  // namespace ryolo

using namespace ryolo;

extern "C" int ryolo_augment_warp(const ryolo_warp_job* jobs_dev, int njobs, uint8_t* rowmax, int h, int w,
                                  void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(jobs_dev && rowmax && njobs > 0 && njobs <= 65535 && h > 0 && w > 0);
  augment_warp_kernel<<<dim3(h, njobs), kAugThreads, 0, stream>>>(jobs_dev, rowmax, h, w);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_augment_finish(const ryolo_finish_job* jobs_dev, int njobs, const uint8_t* rowmax, void* out,
                                    int h, int w, int out_dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(jobs_dev && rowmax && out && njobs > 0 && njobs <= 65535 && h > 0 && w > 0);
  RYOLO_ARG_CHECK(out_dtype == RYOLO_DT_F32 || out_dtype == RYOLO_DT_F16);
  const dim3 grid(h, njobs);
  if (out_dtype == RYOLO_DT_F32) {
    augment_finish_kernel<float><<<grid, kAugThreads, 0, stream>>>(jobs_dev, rowmax, static_cast<float*>(out), h, w);
  } else {
    augment_finish_kernel<__half><<<grid, kAugThreads, 0, stream>>>(jobs_dev, rowmax, static_cast<__half*>(out), h,
                                                                     w);
  }
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}
