// Greedy prediction <-> ground-truth matching of the mAP evaluation on the device (reference test.py:134-151: a Python
// loop over the predictions of an image, one skew_bbox_iou call -- i.e. one GPU round trip -- per prediction).
// Input: the rotated-IoU matrix of the image (ryolo_riou_pairwise, [P, T]), prediction / target classes; output:
// correct[P] in {0, 1}.  The assignment is sequential in the confidence order by definition (a target can be claimed
// once), but each step is only an argmax over the T targets of the prediction's class: one warp walks the predictions,
// lanes stride over the targets, (value, index) warp reduction with the FIRST maximum winning like torch.max.
//
// ryolo_match_batched does the same for every image of a batch straight from detect_postprocess_classes' output, with
// no host read: targets grouped by image (count, scan, stable placement), a segmented sort of each image's kept rows
// into test.py's order, one launch for the same-image IoU pairs (riou.cu), and one warp per image for the walk.
#include <cub/device/device_segmented_radix_sort.cuh>

#include "common.cuh"

namespace ryolo {

// the walk of one image, run by one warp (threadIdx.x = lane)
__device__ __forceinline__ void match_walk(const float* __restrict__ iou, int p, int t, int iou_stride,
                                           const float* __restrict__ pcls, int pcls_stride,
                                           const float* __restrict__ tcls, float thr,
                                           unsigned char* __restrict__ claimed, unsigned char* __restrict__ correct) {
  const int lane = threadIdx.x;
  for (int j = lane; j < t; j += 32) claimed[j] = 0;
  for (int i = lane; i < p; i += 32) correct[i] = 0;
  __syncwarp();
  int n_claimed = 0;
  for (int i = 0; i < p && n_claimed < t; i++) {          // "break if all targets already located" (test.py:137-139)
    const float c = pcls[(size_t)i * pcls_stride];
    float best = -1.f;                                     // IoU >= 0; -1 = no target of this class
    int bi = 0x7fffffff;
    for (int j = lane; j < t; j += 32) {
      if (tcls[j] == c) {
        const float v = iou[(size_t)i * iou_stride + j];
        if (v > best) { best = v; bi = j; }               // strict: keeps the first maximum of this lane's stride
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    // "continue if predicted class not among image classes" = no target of this class: best stays -1
    if (best > thr && bi != 0x7fffffff && !claimed[bi]) {
      if (lane == 0) {
        claimed[bi] = 1;
        correct[i] = 1;
      }
      n_claimed++;
    }
    __syncwarp();
  }
}

__global__ void __launch_bounds__(32) match_kernel(const float* __restrict__ iou, int p, int t, int iou_stride,
                                                   const float* __restrict__ pcls, int pcls_stride,
                                                   const float* __restrict__ tcls, float thr,
                                                   unsigned char* __restrict__ claimed /*[t] scratch*/,
                                                   unsigned char* __restrict__ correct) {
  match_walk(iou, p, t, iou_stride, pcls, pcls_stride, tcls, thr, claimed, correct);
}

// riou.cu
int launch_riou_image_pairs(const float* pbox, int cap, const int* num_keep, const float* tbox, const int* timg,
                            const int* tstart, int batch, int nt, float* iou, cudaStream_t stream);

using u64 = unsigned long long;
constexpr int kMatchMaxBatch = 4096;
constexpr int kGroupThreads = 1024;

// One CTA.  Targets of image b are the rows with targets[k, 0] == b (test.py: targets[targets[:, 0] == si]); rows of any
// other image index belong to no image.  Warp w counts the targets of images w, w + 32, ... (ballots over all rows),
// thread 0 scans the counts, then the same warps place each image's targets in row order: grouped row g holds a target
// of image timg[g], scaled to pixels like test.py:131-133.  Thread 0 also gives each image its first output row
// (*count, then the images' kept counts in batch order) and advances *count.
__global__ void __launch_bounds__(kGroupThreads) match_group_kernel(const float* __restrict__ targets, int nt, int batch,
                                                                    const int* __restrict__ num_keep, float width,
                                                                    float height, int* __restrict__ tstart,
                                                                    int* __restrict__ timg, float* __restrict__ tbox,
                                                                    float* __restrict__ tcls, int* __restrict__ roff,
                                                                    int* __restrict__ count, int* __restrict__ hist,
                                                                    int nc) {
  __shared__ int first[kMatchMaxBatch];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned below = (1u << lane) - 1u;
  for (int b = warp; b < batch; b += kGroupThreads / 32) {
    int c = 0;
    for (int k0 = 0; k0 < nt; k0 += 32) {
      const int k = k0 + lane;
      c += __popc(__ballot_sync(0xffffffffu, k < nt && targets[(size_t)k * 7] == (float)b));
    }
    if (lane == 0) first[b] = c;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int b = 0; b < batch; b++) {
      const int c = first[b];
      tstart[b] = s;
      first[b] = s;
      s += c;
    }
    tstart[batch] = s;
    int r = *count;
    for (int b = 0; b < batch; b++) {
      roff[b] = r;
      r += num_keep[b];
    }
    *count = r;
  }
  __syncthreads();
  for (int b = warp; b < batch; b += kGroupThreads / 32) {
    int pos = first[b];
    for (int k0 = 0; k0 < nt; k0 += 32) {
      const int k = k0 + lane;
      const float* row = targets + (size_t)k * 7;
      const bool mine = k < nt && row[0] == (float)b;
      const unsigned m = __ballot_sync(0xffffffffu, mine);
      if (mine) {
        const int g = pos + __popc(m & below);
        timg[g] = b;
        tbox[(size_t)g * 5 + 0] = __fmul_rn(row[2], width);
        tbox[(size_t)g * 5 + 1] = __fmul_rn(row[3], height);
        tbox[(size_t)g * 5 + 2] = __fmul_rn(row[4], width);
        tbox[(size_t)g * 5 + 3] = __fmul_rn(row[5], height);
        tbox[(size_t)g * 5 + 4] = row[6];
        const float c = row[1];
        tcls[g] = c;
        if (hist != nullptr) atomicAdd(&hist[c >= 0.f && c < (float)nc && c == floorf(c) ? (int)c : nc], 1);
      }
      pos += __popc(m);
    }
  }
}

// ascending sort key of image b's kept row i: (confidence descending, class ascending); the stable sort keeps row order
// within ties -- the order nms.detections_per_image produces
__device__ __forceinline__ unsigned desc_conf_bits(float v) {
  const unsigned u = __float_as_uint(v == 0.f ? 0.f : v);            // -0 ties with +0
  return (u & 0x80000000u) ? u : ~(u | 0x80000000u);                  // ~(order-preserving bits)
}

__global__ void __launch_bounds__(256) match_keys_kernel(const float* __restrict__ dets8, const long long* __restrict__ keep,
                                                         const int* __restrict__ num_keep, int cap, u64* __restrict__ keys,
                                                         int* __restrict__ vals, int* __restrict__ seg_begin,
                                                         int* __restrict__ seg_end) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = num_keep[b];
  if (i == 0) {
    seg_begin[b] = b * cap;
    seg_end[b] = b * cap + n;
  }
  if (i >= n) return;
  const size_t base = (size_t)b * cap;
  const float* d = dets8 + (base + (size_t)keep[base + i]) * 8;
  keys[base + i] = ((u64)desc_conf_bits(d[5]) << 32) | (u64)(unsigned)d[7];
  vals[base + i] = i;
}

// image b's kept rows in sorted order: boxes to pbox (the IoU rows), confidence and class to the output at roff[b]
__global__ void __launch_bounds__(256) match_gather_kernel(const float* __restrict__ dets8, const long long* __restrict__ keep,
                                                           const int* __restrict__ num_keep, int cap,
                                                           const int* __restrict__ order, const int* __restrict__ roff,
                                                           float* __restrict__ pbox, float* __restrict__ conf,
                                                           float* __restrict__ pcls) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= num_keep[b]) return;
  const size_t base = (size_t)b * cap;
  const float* d = dets8 + (base + (size_t)keep[base + order[base + i]]) * 8;
#pragma unroll
  for (int k = 0; k < 5; k++) pbox[(base + i) * 5 + k] = d[k];
  conf[roff[b] + i] = d[5];
  pcls[roff[b] + i] = d[7];
}

__global__ void __launch_bounds__(32) match_batched_kernel(const float* __restrict__ iou, int cap,
                                                           const int* __restrict__ num_keep, const int* __restrict__ tstart,
                                                           const int* __restrict__ roff, const float* __restrict__ pcls,
                                                           const float* __restrict__ tcls, float thr,
                                                           unsigned char* __restrict__ claimed,
                                                           unsigned char* __restrict__ correct) {
  const int b = blockIdx.x, t0 = tstart[b], t = tstart[b + 1] - t0, r0 = roff[b];
  match_walk(iou + (size_t)cap * t0, num_keep[b], t, t, pcls + r0, 1, tcls + t0, thr, claimed + t0, correct + r0);
}

struct MatchPlan {
  int *tstart, *roff, *timg, *seg_begin, *seg_end, *vals[2];
  float *tbox, *tcls, *pbox;
  unsigned char* claimed;
  u64* keys[2];
  void* cub_temp;
  size_t cub_bytes, total;
};

static int plan_match(int batch, int cap, int nt, void* ws, MatchPlan* p, cudaStream_t stream) {
  const size_t items = (size_t)batch * cap;
  p->cub_bytes = 0;
  cub::DoubleBuffer<u64> k(nullptr, nullptr);
  cub::DoubleBuffer<int> v(nullptr, nullptr);
  RYOLO_CUDA_TRY(cub::DeviceSegmentedRadixSort::SortPairs(nullptr, p->cub_bytes, k, v, (int)items, batch,
                                                          (const int*)nullptr, (const int*)nullptr, 0, 64, stream));
  Carver c(ws);
  p->tstart = c.take<int>(batch + 1);
  p->roff = c.take<int>(batch);
  p->seg_begin = c.take<int>(batch);
  p->seg_end = c.take<int>(batch);
  p->timg = c.take<int>(nt);
  p->tbox = c.take<float>((size_t)nt * 5);
  p->tcls = c.take<float>(nt);
  p->claimed = c.take<unsigned char>(nt);
  p->keys[0] = c.take<u64>(items);
  p->keys[1] = c.take<u64>(items);
  p->vals[0] = c.take<int>(items);
  p->vals[1] = c.take<int>(items);
  p->pbox = c.take<float>(items * 5);
  p->cub_temp = c.take<unsigned char>(p->cub_bytes);
  p->total = align_up(c.off, 256);
  return RYOLO_OK;
}

}  // namespace ryolo

using namespace ryolo;

extern "C" int ryolo_match_detections(const float* iou, int p, int t, int iou_stride, const float* pcls, int pcls_stride,
                                      const float* tcls, float iou_thres, unsigned char* claimed_scratch,
                                      unsigned char* correct, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(p >= 0 && t >= 0 && correct != nullptr);
  if (p == 0) return RYOLO_OK;
  if (t == 0) {
    RYOLO_CUDA_TRY(cudaMemsetAsync(correct, 0, (size_t)p, stream));
    return RYOLO_OK;
  }
  RYOLO_ARG_CHECK(iou && pcls && tcls && claimed_scratch && iou_stride >= t && pcls_stride >= 1);
  match_kernel<<<1, 32, 0, stream>>>(iou, p, t, iou_stride, pcls, pcls_stride, tcls, iou_thres, claimed_scratch, correct);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_match_batched(const float* dets8, const int64_t* keep, const int32_t* num_keep, int batch, int cap,
                                   const float* targets, int nt, int height, int width, float iou_thres,
                                   unsigned char* correct, float* conf, float* pcls, int32_t* count, int32_t* class_hist,
                                   int nc, float* iou_scratch, void* workspace, size_t* workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(batch >= 1 && batch <= kMatchMaxBatch && cap >= 1 && nt >= 0 && workspace_bytes != nullptr);
  RYOLO_ARG_CHECK((long long)batch * cap < (1ll << 31) && (long long)cap * nt < (1ll << 40));
  MatchPlan p;
  if (workspace == nullptr) {
    const int st = plan_match(batch, cap, nt, nullptr, &p, stream);
    *workspace_bytes = p.total;
    return st;
  }
  RYOLO_ARG_CHECK(dets8 && keep && num_keep && correct && conf && pcls && count && height > 0 && width > 0);
  RYOLO_ARG_CHECK(nt == 0 || (targets && iou_scratch));
  RYOLO_ARG_CHECK(class_hist == nullptr || nc >= 1);
  RYOLO_ARG_CHECK((reinterpret_cast<uintptr_t>(workspace) & 255) == 0);
  const int st = plan_match(batch, cap, nt, workspace, &p, stream);
  if (st != RYOLO_OK) return st;
  if (p.total > *workspace_bytes) {
    set_err("ryolo_match_batched: workspace %zu B < required %zu B", *workspace_bytes, p.total);
    return RYOLO_E_WORKSPACE;
  }
  match_group_kernel<<<1, kGroupThreads, 0, stream>>>(targets, nt, batch, num_keep, (float)width, (float)height, p.tstart,
                                                      p.timg, p.tbox, p.tcls, p.roff, count, class_hist, nc);
  RYOLO_LAUNCH_CHECK();
  const dim3 grid((cap + 255) / 256, batch);
  match_keys_kernel<<<grid, 256, 0, stream>>>(dets8, reinterpret_cast<const long long*>(keep), num_keep, cap, p.keys[0],
                                              p.vals[0], p.seg_begin, p.seg_end);
  RYOLO_LAUNCH_CHECK();
  cub::DoubleBuffer<u64> dk(p.keys[0], p.keys[1]);
  cub::DoubleBuffer<int> dv(p.vals[0], p.vals[1]);
  size_t tmp = p.cub_bytes;
  // stable per-image sort; rows beyond an image's kept count are never read
  RYOLO_CUDA_TRY(cub::DeviceSegmentedRadixSort::SortPairs(p.cub_temp, tmp, dk, dv, batch * cap, batch, p.seg_begin,
                                                          p.seg_end, 0, 64, stream));
  count_launch(8);  // radix sort passes (library kernels, counted as a lower bound)
  match_gather_kernel<<<grid, 256, 0, stream>>>(dets8, reinterpret_cast<const long long*>(keep), num_keep, cap, dv.Current(),
                                                p.roff, p.pbox, conf, pcls);
  RYOLO_LAUNCH_CHECK();
  const int rc = launch_riou_image_pairs(p.pbox, cap, num_keep, p.tbox, p.timg, p.tstart, batch, nt, iou_scratch, stream);
  if (rc != RYOLO_OK) return rc;
  match_batched_kernel<<<batch, 32, 0, stream>>>(iou_scratch, cap, num_keep, p.tstart, p.roff, pcls, p.tcls, iou_thres,
                                                 p.claimed, correct);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}
