// libryolo.so: error/launch bookkeeping, the non_max_suppression candidate filter and the YOLO head decode.
#include <stdarg.h>

#include "common.cuh"
#include "filter.cuh"

namespace ryolo {

std::atomic<uint64_t> g_launches{0};
std::atomic<int> g_reserved_sms{0};

char* err_buf() {
  static thread_local char buf[512] = {0};
  return buf;
}
void set_err(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(err_buf(), 512, fmt, ap);
  va_end(ap);
}

// ------------------------------------------------------------------------------------------------
// non_max_suppression candidate filter (reference utils/nms/nms.py:34-40,55)
// ------------------------------------------------------------------------------------------------
constexpr int FT = 256;  // rows per block

// pass 1: in-place conf update + per-block survivor counts
__global__ void __launch_bounds__(FT) nms_filter_count_kernel(float* __restrict__ pred, int p, int nc, float conf_thres,
                                                             float min_wh, int* __restrict__ block_counts) {
  const int i = blockIdx.x * FT + threadIdx.x;
  bool keep = false;
  if (i < p) {
    float* row = pred + (size_t)i * (6 + nc);
    float best; int bi; bool fin;
    class_max(row, nc, &best, &bi, &fin);
    const float conf = row[5] * best;  // pred[:, 5] *= class_conf, in place (nms.py:35)
    row[5] = conf;
    keep = keep_row(row, conf, fin, conf_thres, min_wh);
  }
  const int cnt = __syncthreads_count(keep);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = cnt;
}

// pass 2: exclusive scan of the block counts (single CTA), total -> num_out
__global__ void __launch_bounds__(1024) nms_filter_scan_kernel(int* __restrict__ block_counts, int nblocks,
                                                               int* __restrict__ num_out) {
  __shared__ int s_warp[32];
  __shared__ int s_carry;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_carry = 0;
  __syncthreads();
  for (int start = 0; start < nblocks; start += 1024) {
    const int i = start + tid;
    const int v = i < nblocks ? block_counts[i] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int w = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += y;
      }
      s_warp[lane] = w;
    }
    __syncthreads();
    const int carry = s_carry;
    const int incl = x + (warp ? s_warp[warp - 1] : 0) + carry;
    if (i < nblocks) block_counts[i] = incl - v;  // exclusive
    __syncthreads();
    if (tid == 1023) s_carry = incl;
    __syncthreads();
  }
  if (tid == 0) *num_out = s_carry;
}

// pass 3: stable write of the survivors
__global__ void __launch_bounds__(FT) nms_filter_write_kernel(const float* __restrict__ pred, int p, int nc,
                                                             float conf_thres, float min_wh,
                                                             const int* __restrict__ block_offsets,
                                                             float* __restrict__ out, int capacity) {
  __shared__ int s_warp[FT / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int i = blockIdx.x * FT + tid;
  bool keep = false;
  float cc = 0.f, ci = 0.f;
  const float* row = pred + (size_t)i * (6 + nc);
  if (i < p) {  // pass 1 already stored conf in row[5]
    float best; int bi; bool fin;
    class_max(row, nc, &best, &bi, &fin);
    cc = best; ci = (float)bi;
    keep = keep_row(row, row[5], fin, conf_thres, min_wh);
  }
  const unsigned bal = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) s_warp[warp] = __popc(bal);
  __syncthreads();
  int prefix = 0;
  for (int w = 0; w < warp; w++) prefix += s_warp[w];
  if (keep) {
    const int dst = block_offsets[blockIdx.x] + prefix + __popc(bal & ((1u << lane) - 1u));
    if (dst < capacity) {
      float* o = out + (size_t)dst * 8;
      o[0] = row[0]; o[1] = row[1]; o[2] = row[2]; o[3] = row[3]; o[4] = row[4];
      o[5] = row[5]; o[6] = cc; o[7] = ci;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// YOLO head decode (reference model/models.py:198-227)
// ------------------------------------------------------------------------------------------------
// One thread decodes one (b, anchor, y, x) cell.  The head tensor is NCHW (plane-strided, coalesced reads across x);
// the two outputs are row-major [.., no] -- a CTA's 256 cells form ONE contiguous range of 256*no floats in each, so
// the rows are staged in shared memory and written back with fully coalesced stores (the direct per-thread row store
// touches every 32-B sector of the range `no` times with 4 useful bytes each).
template <bool STAGED>
__global__ void __launch_bounds__(256) yolo_decode_kernel(const float* __restrict__ p, int bs, int na, int nc, int ny,
                                                          int nx, const float* __restrict__ anchors, float stride,
                                                          float ctx, int arc_default, float* __restrict__ io,
                                                          int rows_total, int row_offset, float* __restrict__ p_out) {
  constexpr int NO_MAX = 8;
  __shared__ float s_io[STAGED ? 256 * NO_MAX : 1];
  __shared__ float s_p[STAGED ? 256 * NO_MAX : 1];
  const int no = nc + 6;
  const int per_img = na * ny * nx;
  const int b = blockIdx.y;
  const int cell0 = blockIdx.x * 256;
  const int cell = cell0 + threadIdx.x;              // within the image: (a, y, x)
  const bool live = cell < per_img;
  const size_t plane = (size_t)ny * nx;
  float* io_base = io + ((size_t)b * rows_total + row_offset + cell0) * no;
  float* p_base = p_out ? p_out + ((size_t)b * per_img + cell0) * no : nullptr;
  if (live) {
    const int x = cell % nx;
    const int y = (cell / nx) % ny;
    const int a = cell / (nx * ny);
    const float* src = p + ((size_t)b * na * no + (size_t)a * no) * plane + (size_t)y * nx + x;
    float* dst = STAGED ? s_io + threadIdx.x * no : io_base + (size_t)threadIdx.x * no;
    float* pd = STAGED ? s_p + threadIdx.x * no : (p_base ? p_base + (size_t)threadIdx.x * no : nullptr);
    // anchor_vec = anchors / stride (model_utils.py:30-31), theta untouched
    const float aw = anchors[a * 3 + 0] / stride, ah = anchors[a * 3 + 1] / stride, at = anchors[a * 3 + 2];
    const float t0 = src[0], t1 = src[plane], t2 = src[2 * plane], t3 = src[3 * plane], t4 = src[4 * plane];
    if (pd) { pd[0] = t0; pd[1] = t1; pd[2] = t2; pd[3] = t3; pd[4] = t4; }
    float bx = (1.f / (1.f + expf(-t0)) + (float)x) * stride;   // (sigmoid + grid) * stride
    float by = (1.f / (1.f + expf(-t1)) + (float)y) * stride;
    float bw = (expf(t2) * aw) * stride;
    float bh = (expf(t3) * ah) * stride;
    const float th = atanf(t4) + at;
    bh = bh / ctx;                    // io[..., 3] /= context_factor
    bw = bw - bh * (ctx - 1.f);       // io[..., 2] -= io[..., 3] * (context_factor - 1)
    dst[0] = bx; dst[1] = by; dst[2] = bw; dst[3] = bh; dst[4] = th;
    for (int k = 5; k < no; k++) {
      const float v = src[(size_t)k * plane];
      if (pd) pd[k] = v;
      float o = arc_default ? 1.f / (1.f + expf(-v)) : v;
      if (nc == 1 && k == 6) o = 1.f;  // models.py:220-221
      dst[k] = o;
    }
  }
  if (STAGED) {
    __syncthreads();
    const int nval = min(256, per_img - cell0) * no;
    for (int e = threadIdx.x; e < nval; e += 256) {
      io_base[e] = s_io[e];
      if (p_base) p_base[e] = s_p[e];
    }
  }
}

}  // namespace ryolo

using namespace ryolo;

extern "C" int ryolo_abi_version(void) { return 2; }
extern "C" const char* ryolo_last_error(void) { return err_buf(); }
extern "C" uint64_t ryolo_launch_count(void) { return g_launches.load(); }

extern "C" int ryolo_set_reserved_sms(int n) {
  if (n < 0 || n > 64) return RYOLO_E_ARG;
  ryolo::g_reserved_sms.store(n, std::memory_order_relaxed);
  return RYOLO_OK;
}

extern "C" size_t ryolo_nms_filter_workspace_bytes(int p) {
  const int nblocks = (p > 0 ? p : 0) / FT + 1;
  return align_up((size_t)nblocks * sizeof(int), 256) + 256;
}

extern "C" int ryolo_nms_filter(float* pred, int p, int nc, float conf_thres, float min_wh, float* out, int capacity,
                                int32_t* num_out, void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(p >= 0 && nc >= 1 && capacity >= 0 && num_out != nullptr);
  if (p == 0) {
    RYOLO_CUDA_TRY(cudaMemsetAsync(num_out, 0, sizeof(int32_t), stream));
    return RYOLO_OK;
  }
  RYOLO_ARG_CHECK(pred && out && workspace);
  if (workspace_bytes < ryolo_nms_filter_workspace_bytes(p)) {
    set_err("ryolo_nms_filter: workspace too small");
    return RYOLO_E_WORKSPACE;
  }
  const int nblocks = (p + FT - 1) / FT;
  int* counts = static_cast<int*>(workspace);
  nms_filter_count_kernel<<<nblocks, FT, 0, stream>>>(pred, p, nc, conf_thres, min_wh, counts);
  RYOLO_LAUNCH_CHECK();
  nms_filter_scan_kernel<<<1, 1024, 0, stream>>>(counts, nblocks, num_out);
  RYOLO_LAUNCH_CHECK();
  nms_filter_write_kernel<<<nblocks, FT, 0, stream>>>(pred, p, nc, conf_thres, min_wh, counts, out, capacity);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_yolo_decode(const float* p, int bs, int na, int nc, int ny, int nx, const float* anchors,
                                 float stride, float context_factor, int arc_default, float* io_out, int io_rows_total,
                                 int row_offset, float* p_out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(bs >= 0 && na > 0 && nc >= 1 && ny > 0 && nx > 0);
  RYOLO_ARG_CHECK(p && anchors && io_out);
  RYOLO_ARG_CHECK(row_offset >= 0 && row_offset + na * ny * nx <= io_rows_total);
  const size_t total = (size_t)bs * na * ny * nx;
  if (total == 0) return RYOLO_OK;
  RYOLO_ARG_CHECK(bs <= 65535 && (size_t)na * ny * nx < (1u << 30));
  dim3 grid((unsigned)((na * ny * nx + 255) / 256), (unsigned)bs);
  if (nc + 6 <= 8)
    yolo_decode_kernel<true><<<grid, 256, 0, stream>>>(p, bs, na, nc, ny, nx, anchors, stride, context_factor, arc_default,
                                                       io_out, io_rows_total, row_offset, p_out);
  else
    yolo_decode_kernel<false><<<grid, 256, 0, stream>>>(p, bs, na, nc, ny, nx, anchors, stride, context_factor, arc_default,
                                                        io_out, io_rows_total, row_offset, p_out);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}
