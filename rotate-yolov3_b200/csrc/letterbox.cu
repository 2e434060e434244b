// Letterboxes a batch of uint8 HWC BGR images of any sizes into the reference's network input [B, 3, H, W]: cv2's
// INTER_AREA resize (utils/datasets.py:536), a grey 128 border (:544), BGR->RGB, CHW and /255 (:112-117, :498-500).
// The result is byte for byte the reference's, so every path restates cv2's arithmetic in cv2's order:
//
//   RYOLO_LB_AREA      per source row of the output pixel's y taps, in order, buf = sum_i S * wx[i] (float32, tap
//                      order), then sum += wy[j] * buf (float32); rint and saturate.  No FMA: cv2's x86 build rounds
//                      each product, so every product and sum here is an explicit __fmul_rn / __fadd_rn.
//   RYOLO_LB_AREA_INT  integer sum of the kx x ky block; (sum + 2) >> 2 for 2x2 (cv2's SIMD path), otherwise
//                      rint(sum * float(1 / (kx * ky))).
//   RYOLO_LB_LINEAR    h_r = S[r][x0] * a0 + S[r][x1] * a1 (int, 11-bit weights) for the two rows, then
//                      ((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2 (cv2's fixed-point vertical pass).
//
// The value v in [0, 255] becomes v / 255.f by IEEE division (numpy's float32 `/= 255.0`), and for fp16 that float32
// quotient rounded to half (numpy's float16 `/=` computes in float32 and rounds once to half).
//
// RYOLO_DT_U8 writes the letterboxed uint8 image itself, [B, H, W, 3] BGR with border 128, for the training
// augmentation that runs on it (csrc/augment.cu); the float outputs are untouched by that mode.
//
// One CTA per output row of one job (grid.y = job).  Consecutive threads take consecutive output pixels, so a warp
// reads one contiguous span of each source row it needs and writes 32 consecutive elements of each output plane.
#include <cuda_fp16.h>

#include "common.cuh"

namespace ryolo {

constexpr int kLbThreads = 256;

template <typename T>
__device__ __forceinline__ T lb_cast(float v);
template <>
__device__ __forceinline__ float lb_cast<float>(float v) { return v; }
template <>
__device__ __forceinline__ __half lb_cast<__half>(float v) { return __float2half_rn(v); }

__device__ __forceinline__ int sat_u8(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

// one output pixel of a resize job: the three BGR channel values in [0, 255]
__device__ __forceinline__ void area_px(const ryolo_letterbox_job& jb, const int* __restrict__ tab, int yy, int xx,
                                        int v[3]) {
  const int* ye = tab + jb.ytab + 3 * yy;
  const int* xe = tab + jb.xtab + 3 * xx;
  const int ys = __ldg(ye), yn = __ldg(ye + 1), xs = __ldg(xe), xn = __ldg(xe + 1);
  const float* yw = reinterpret_cast<const float*>(tab + jb.ytab + __ldg(ye + 2));
  const float* xw = reinterpret_cast<const float*>(tab + jb.xtab + __ldg(xe + 2));
  float s0 = 0.f, s1 = 0.f, s2 = 0.f;
  for (int j = 0; j < yn; j++) {
    const uint8_t* row = jb.src + (long long)(ys + j) * jb.src_stride + 3LL * xs;
    float b0 = 0.f, b1 = 0.f, b2 = 0.f;
    for (int i = 0; i < xn; i++) {
      const float w = __ldg(xw + i);
      b0 = __fadd_rn(b0, __fmul_rn((float)__ldg(row + 3 * i), w));
      b1 = __fadd_rn(b1, __fmul_rn((float)__ldg(row + 3 * i + 1), w));
      b2 = __fadd_rn(b2, __fmul_rn((float)__ldg(row + 3 * i + 2), w));
    }
    const float beta = __ldg(yw + j);
    s0 = __fadd_rn(s0, __fmul_rn(beta, b0));
    s1 = __fadd_rn(s1, __fmul_rn(beta, b1));
    s2 = __fadd_rn(s2, __fmul_rn(beta, b2));
  }
  v[0] = sat_u8(__float2int_rn(s0));
  v[1] = sat_u8(__float2int_rn(s1));
  v[2] = sat_u8(__float2int_rn(s2));
}

__device__ __forceinline__ void area_int_px(const ryolo_letterbox_job& jb, int yy, int xx, int v[3]) {
  const uint8_t* base = jb.src + (long long)yy * jb.ky * jb.src_stride + 3LL * xx * jb.kx;
  int s0 = 0, s1 = 0, s2 = 0;
  for (int j = 0; j < jb.ky; j++) {
    const uint8_t* row = base + (long long)j * jb.src_stride;
    for (int i = 0; i < jb.kx; i++) {
      s0 += __ldg(row + 3 * i);
      s1 += __ldg(row + 3 * i + 1);
      s2 += __ldg(row + 3 * i + 2);
    }
  }
  if (jb.kx == 2 && jb.ky == 2) {
    v[0] = (s0 + 2) >> 2, v[1] = (s1 + 2) >> 2, v[2] = (s2 + 2) >> 2;
  } else {
    const float inv = __fdiv_rn(1.f, (float)(jb.kx * jb.ky));
    v[0] = sat_u8(__float2int_rn(__fmul_rn((float)s0, inv)));
    v[1] = sat_u8(__float2int_rn(__fmul_rn((float)s1, inv)));
    v[2] = sat_u8(__float2int_rn(__fmul_rn((float)s2, inv)));
  }
}

__device__ __forceinline__ void linear_px(const ryolo_letterbox_job& jb, const int* __restrict__ tab, int yy, int xx,
                                          int v[3]) {
  const int* ye = tab + jb.ytab + 3 * yy;
  const int* xe = tab + jb.xtab + 3 * xx;
  const int y0 = __ldg(ye), y1 = min(y0 + 1, jb.src_h - 1), x0 = __ldg(xe), x1 = min(x0 + 1, jb.src_w - 1);
  const int* yw = tab + jb.ytab + __ldg(ye + 2);
  const int* xw = tab + jb.xtab + __ldg(xe + 2);
  const int a0 = __ldg(xw), a1 = __ldg(xw + 1), b0 = __ldg(yw), b1 = __ldg(yw + 1);
  const uint8_t* r0 = jb.src + (long long)y0 * jb.src_stride;
  const uint8_t* r1 = jb.src + (long long)y1 * jb.src_stride;
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const int h0 = __ldg(r0 + 3 * x0 + c) * a0 + __ldg(r0 + 3 * x1 + c) * a1;
    const int h1 = __ldg(r1 + 3 * x0 + c) * a0 + __ldg(r1 + 3 * x1 + c) * a1;
    v[c] = sat_u8((((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2);
  }
}

template <typename T>
__global__ void __launch_bounds__(kLbThreads)
    letterbox_kernel(const ryolo_letterbox_job* __restrict__ jobs, const int* __restrict__ tab, T* __restrict__ out,
                     int out_h, int out_w) {
  const ryolo_letterbox_job jb = jobs[blockIdx.y];
  const int y = blockIdx.x;
  const size_t plane = (size_t)out_h * out_w;
  T* o = out + (size_t)blockIdx.y * 3 * plane + (size_t)y * out_w;
  const T grey = lb_cast<T>(__fdiv_rn(128.f, 255.f));
  const int yy = y - jb.top;
  const bool row_in = yy >= 0 && yy < jb.dst_h;
  for (int x = threadIdx.x; x < out_w; x += kLbThreads) {
    const int xx = x - jb.left;
    if (!row_in || xx < 0 || xx >= jb.dst_w) {
      o[x] = grey, o[plane + x] = grey, o[2 * plane + x] = grey;
      continue;
    }
    int v[3];                                                // B, G, R
    if (jb.kind == RYOLO_LB_AREA) {
      area_px(jb, tab, yy, xx, v);
    } else if (jb.kind == RYOLO_LB_AREA_INT) {
      area_int_px(jb, yy, xx, v);
    } else {
      linear_px(jb, tab, yy, xx, v);
    }
    o[x] = lb_cast<T>(__fdiv_rn((float)v[2], 255.f));
    o[plane + x] = lb_cast<T>(__fdiv_rn((float)v[1], 255.f));
    o[2 * plane + x] = lb_cast<T>(__fdiv_rn((float)v[0], 255.f));
  }
}

// the same pixels into a uint8 HWC BGR image per job: out [njobs, out_h, out_w, 3], border 128
__global__ void __launch_bounds__(kLbThreads)
    letterbox_u8_kernel(const ryolo_letterbox_job* __restrict__ jobs, const int* __restrict__ tab,
                        uint8_t* __restrict__ out, int out_h, int out_w) {
  const ryolo_letterbox_job jb = jobs[blockIdx.y];
  const int y = blockIdx.x;
  uint8_t* o = out + ((size_t)blockIdx.y * out_h + y) * out_w * 3;
  const int yy = y - jb.top;
  const bool row_in = yy >= 0 && yy < jb.dst_h;
  for (int x = threadIdx.x; x < out_w; x += kLbThreads) {
    const int xx = x - jb.left;
    int v[3] = {128, 128, 128};
    if (row_in && xx >= 0 && xx < jb.dst_w) {
      if (jb.kind == RYOLO_LB_AREA) {
        area_px(jb, tab, yy, xx, v);
      } else if (jb.kind == RYOLO_LB_AREA_INT) {
        area_int_px(jb, yy, xx, v);
      } else {
        linear_px(jb, tab, yy, xx, v);
      }
    }
    o[3 * x] = (uint8_t)v[0], o[3 * x + 1] = (uint8_t)v[1], o[3 * x + 2] = (uint8_t)v[2];
  }
}

}  // namespace ryolo

using namespace ryolo;

extern "C" int ryolo_letterbox(const ryolo_letterbox_job* jobs_dev, int njobs, const int32_t* tables_dev, void* out,
                               int out_h, int out_w, int out_dtype, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(jobs_dev && tables_dev && out && njobs > 0 && njobs <= 65535 && out_h > 0 && out_w > 0);
  RYOLO_ARG_CHECK(out_dtype == RYOLO_DT_F32 || out_dtype == RYOLO_DT_F16 || out_dtype == RYOLO_DT_U8);
  const dim3 grid(out_h, njobs);
  if (out_dtype == RYOLO_DT_U8) {
    letterbox_u8_kernel<<<grid, kLbThreads, 0, stream>>>(jobs_dev, tables_dev, static_cast<uint8_t*>(out), out_h,
                                                         out_w);
  } else if (out_dtype == RYOLO_DT_F32) {
    letterbox_kernel<float><<<grid, kLbThreads, 0, stream>>>(jobs_dev, tables_dev, static_cast<float*>(out), out_h,
                                                              out_w);
  } else {
    letterbox_kernel<__half><<<grid, kLbThreads, 0, stream>>>(jobs_dev, tables_dev, static_cast<__half*>(out), out_h,
                                                               out_w);
  }
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}
