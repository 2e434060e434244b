// Cross-scale merge of multi-scale detection (reference multi_detect, detect.py:81-101): per image, the kept rows of
// every scale's class-aware NMS, mapped back to original-image pixels as scale_coords(...).round() maps them
// (utils/utils.py:181-189), concatenated in scale order.  The second NMS runs on the result with the existing selection
// and class-aware NMS launches.
#include "common.cuh"

namespace ryolo {

struct MergeScales {
  const float* dets[RYOLO_MERGE_MAX_SCALES];
  const int64_t* keep[RYOLO_MERGE_MAX_SCALES];
  const int32_t* num[RYOLO_MERGE_MAX_SCALES];
};

// grid = (row chunks, batch): a thread owns output rows j of image b.  Row j belongs to the scale whose prefix of kept
// counts brackets it; the prefix is taken per thread from the `scales` counts of the image (no host read, no scan pass).
__global__ void __launch_bounds__(256) merge_scales_kernel(const MergeScales a, int scales, int batch, int cap,
                                                           const float* __restrict__ table, float* __restrict__ out) {
  const int b = blockIdx.y;
  const long long rows = (long long)scales * cap;
  for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < rows; j += (long long)gridDim.x * blockDim.x) {
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    long long off = 0;
#pragma unroll
    for (int s = 0; s < RYOLO_MERGE_MAX_SCALES; s++) {
      if (s >= scales) break;
      const int n = min(max(a.num[s][b], 0), cap);
      if (j < off + n) {
        const long long r = a.keep[s][(long long)b * cap + (j - off)];
        if (r >= 0 && r < cap) {
          const float* src = a.dets[s] + ((long long)b * cap + r) * 8;
          const float* t = table + ((long long)s * batch + b) * 3;
          const float padx = t[0], pady = t[1], gain = t[2];
          // scale_coords in fp32: x -= padx, y -= pady, then x, y, w, h /= gain (IEEE division); .round() half to even
          v[0] = rintf(__fdiv_rn(__fsub_rn(src[0], padx), gain));
          v[1] = rintf(__fdiv_rn(__fsub_rn(src[1], pady), gain));
          v[2] = rintf(__fdiv_rn(src[2], gain));
          v[3] = rintf(__fdiv_rn(src[3], gain));
#pragma unroll
          for (int k = 4; k < 8; k++) v[k] = src[k];
        }
        break;
      }
      off += n;
    }
    float* dst = out + ((long long)b * rows + j) * 8;
#pragma unroll
    for (int k = 0; k < 8; k++) dst[k] = v[k];
  }
}

}  // namespace ryolo

extern "C" int ryolo_merge_scales(const float* const* dets_host, const int64_t* const* keep_host,
                                  const int32_t* const* num_keep_host, int scales, int batch, int cap,
                                  const float* table, float* out, void* stream_) {
  using namespace ryolo;
  RYOLO_ARG_CHECK(dets_host && keep_host && num_keep_host && table && out);
  RYOLO_ARG_CHECK(scales >= 1 && scales <= RYOLO_MERGE_MAX_SCALES);
  RYOLO_ARG_CHECK(batch >= 1 && batch <= 65535 && cap >= 1);
  MergeScales a;
  memset(&a, 0, sizeof(a));
  for (int s = 0; s < scales; s++) {
    RYOLO_ARG_CHECK(dets_host[s] && keep_host[s] && num_keep_host[s]);
    a.dets[s] = dets_host[s];
    a.keep[s] = keep_host[s];
    a.num[s] = num_keep_host[s];
  }
  const long long rows = (long long)scales * cap;
  const long long chunks = (rows + 255) / 256;
  const dim3 grid((unsigned)(chunks < 1024 ? chunks : 1024), (unsigned)batch);
  merge_scales_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream_)>>>(a, scales, batch, cap, table, out);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}
