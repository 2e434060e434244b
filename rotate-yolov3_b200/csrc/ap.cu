// ap_per_class (reference utils/utils.py:200-265) over every detection row of an evaluation, on the device.
//   1. one stable radix sort of all rows by (class ascending, confidence descending): within a class the rows come in
//      the order of a stable sort by confidence -- ties keep their row order (np.argsort(-conf) leaves it unspecified);
//   2. per sorted row: its true-positive flag, and the first / last row of each class;
//   3. an exclusive scan of the flags numbers the true positives, which are then listed by position;
//   4. one thread per class: precision, recall, AP and F1 from its true positives (ap.cuh), sums in row order.
// Integer sums and a fixed summation order: the results repeat bit for bit, whatever the launch configuration.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "ap.cuh"
#include "common.cuh"

namespace ryolo {

using u64 = unsigned long long;

__device__ __forceinline__ unsigned ap_desc_conf_bits(float v) {
  const unsigned u = __float_as_uint(v == 0.f ? 0.f : v);            // -0 ties with +0
  return (u & 0x80000000u) ? u : ~(u | 0x80000000u);                  // ~(order-preserving bits)
}

// rows at or past *n_rows, and rows whose class is not an integer in [0, nc), sort into bucket nc after every class
__global__ void __launch_bounds__(256) ap_keys_kernel(const float* __restrict__ conf, const float* __restrict__ pcls,
                                                      const int* __restrict__ n_rows, int n_cap, int nc,
                                                      u64* __restrict__ keys, int* __restrict__ vals) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_cap) return;
  unsigned cls = (unsigned)nc, bits = 0u;
  if (k < *n_rows) {
    const float c = pcls[k];
    if (c >= 0.f && c < (float)nc && c == floorf(c)) cls = (unsigned)c;
    bits = ap_desc_conf_bits(conf[k]);
  }
  keys[k] = ((u64)cls << 32) | bits;
  vals[k] = k;
}

__global__ void __launch_bounds__(256) ap_flags_kernel(const u64* __restrict__ keys, const int* __restrict__ order,
                                                       const unsigned char* __restrict__ correct, int n_cap, int nc,
                                                       int* __restrict__ tp, int* __restrict__ lo, int* __restrict__ hi) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_cap) return;
  const unsigned cls = (unsigned)(keys[k] >> 32);
  const bool live = cls < (unsigned)nc;
  tp[k] = live && correct[order[k]] ? 1 : 0;
  if (!live) return;
  if (k == 0 || (unsigned)(keys[k - 1] >> 32) != cls) lo[cls] = k;
  if (k == n_cap - 1 || (unsigned)(keys[k + 1] >> 32) != cls) hi[cls] = k + 1;
}

__global__ void __launch_bounds__(256) ap_list_kernel(const int* __restrict__ tp, const int* __restrict__ rank, int n_cap,
                                                      int* __restrict__ tp_pos) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n_cap && tp[k]) tp_pos[rank[k]] = k;
}

__global__ void __launch_bounds__(128) ap_class_kernel(const int* __restrict__ tp, const int* __restrict__ rank,
                                                       const int* __restrict__ tp_pos, const int* __restrict__ lo,
                                                       const int* __restrict__ hi, const int* __restrict__ n_gt, int nc,
                                                       double* __restrict__ env, double* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nc) return;
  ApClass s = {0.0, 0.0, 0.0, 0.0};
  const int n_p = hi[c] - lo[c];
  if (n_gt[c] > 0) {
    int r0 = 0, ntp = 0;
    if (n_p > 0) {
      r0 = rank[lo[c]];
      ntp = rank[hi[c] - 1] + tp[hi[c] - 1] - r0;
    }
    s = ap_class_stats(tp_pos + r0, lo[c], ntp, n_p, n_gt[c], env + r0);
  }
  out[c * 4 + 0] = s.p;
  out[c * 4 + 1] = s.r;
  out[c * 4 + 2] = s.ap;
  out[c * 4 + 3] = s.f1;
}

struct ApPlan {
  u64* keys[2];
  int *vals[2], *tp, *rank, *tp_pos, *lo, *hi;
  double* env;
  void* cub_temp;
  size_t cub_bytes, total;
  int end_bit;
};

static int plan_ap(int n_cap, int nc, void* ws, ApPlan* p, cudaStream_t stream) {
  p->end_bit = 32;
  while (p->end_bit < 64 && ((u64)nc >> (p->end_bit - 32)) != 0) p->end_bit++;   // classes 0..nc fit
  size_t sort_bytes = 0, scan_bytes = 0;
  cub::DoubleBuffer<u64> k(nullptr, nullptr);
  cub::DoubleBuffer<int> v(nullptr, nullptr);
  RYOLO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, k, v, n_cap, 0, p->end_bit, stream));
  RYOLO_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const int*)nullptr, (int*)nullptr, n_cap, stream));
  p->cub_bytes = sort_bytes > scan_bytes ? sort_bytes : scan_bytes;
  const size_t n = n_cap > 0 ? (size_t)n_cap : 1;
  Carver c(ws);
  p->keys[0] = c.take<u64>(n);
  p->keys[1] = c.take<u64>(n);
  p->vals[0] = c.take<int>(n);
  p->vals[1] = c.take<int>(n);
  p->tp = c.take<int>(n);
  p->rank = c.take<int>(n);
  p->tp_pos = c.take<int>(n);
  p->env = c.take<double>(n);
  p->lo = c.take<int>(2 * (size_t)nc);
  p->hi = p->lo + nc;
  p->cub_temp = c.take<unsigned char>(p->cub_bytes);
  p->total = align_up(c.off, 256);
  return RYOLO_OK;
}

}  // namespace ryolo

using namespace ryolo;

extern "C" int ryolo_ap_per_class(const unsigned char* correct, const float* conf, const float* pcls, const int32_t* n_rows,
                                  int n_cap, const int32_t* n_gt, int nc, double* out, void* workspace,
                                  size_t* workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(n_cap >= 0 && nc >= 1 && nc < (1 << 24) && workspace_bytes != nullptr);
  ApPlan p;
  if (workspace == nullptr) {
    const int st = plan_ap(n_cap, nc, nullptr, &p, stream);
    *workspace_bytes = p.total;
    return st;
  }
  RYOLO_ARG_CHECK(n_rows && n_gt && out && (n_cap == 0 || (correct && conf && pcls)));
  RYOLO_ARG_CHECK((reinterpret_cast<uintptr_t>(workspace) & 255) == 0);
  const int st = plan_ap(n_cap, nc, workspace, &p, stream);
  if (st != RYOLO_OK) return st;
  if (p.total > *workspace_bytes) {
    set_err("ryolo_ap_per_class: workspace %zu B < required %zu B", *workspace_bytes, p.total);
    return RYOLO_E_WORKSPACE;
  }
  RYOLO_CUDA_TRY(cudaMemsetAsync(p.lo, 0, 2 * (size_t)nc * sizeof(int), stream));
  const int T = 256, blocks = (n_cap + T - 1) / T;
  if (n_cap > 0) {
    ap_keys_kernel<<<blocks, T, 0, stream>>>(conf, pcls, n_rows, n_cap, nc, p.keys[0], p.vals[0]);
    RYOLO_LAUNCH_CHECK();
    cub::DoubleBuffer<u64> dk(p.keys[0], p.keys[1]);
    cub::DoubleBuffer<int> dv(p.vals[0], p.vals[1]);
    size_t tmp = p.cub_bytes;
    RYOLO_CUDA_TRY(cub::DeviceRadixSort::SortPairs(p.cub_temp, tmp, dk, dv, n_cap, 0, p.end_bit, stream));
    count_launch(4);  // radix sort passes (library kernels, counted as a lower bound)
    ap_flags_kernel<<<blocks, T, 0, stream>>>(dk.Current(), dv.Current(), correct, n_cap, nc, p.tp, p.lo, p.hi);
    RYOLO_LAUNCH_CHECK();
    tmp = p.cub_bytes;
    RYOLO_CUDA_TRY(cub::DeviceScan::ExclusiveSum(p.cub_temp, tmp, p.tp, p.rank, n_cap, stream));
    count_launch(1);
    ap_list_kernel<<<blocks, T, 0, stream>>>(p.tp, p.rank, n_cap, p.tp_pos);
    RYOLO_LAUNCH_CHECK();
  }
  ap_class_kernel<<<(nc + 127) / 128, 128, 0, stream>>>(p.tp, p.rank, p.tp_pos, p.lo, p.hi, n_gt, nc, p.env, out);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}
