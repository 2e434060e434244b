// Rotated NMS for sm_90a: device sort -> per-box geometry -> upper-triangle suppression mask
// (conservative filter + pinned-arithmetic exact overlap on the survivors) -> on-device greedy scan
// -> ascending compaction of the kept ORIGINAL indices.  No host round trip anywhere.
//
// Replaces r_nms / nms_cuda of the reference (utils/nms/src/rotate_polygon_nms.cpp:7-16,
// utils/nms/src/rotate_polygon_nms_kernel.cu:323-384).  Differences in *how* (never in the result):
//   * only tiles with column-block >= row-block are evaluated (the reference evaluates all N^2
//     pairs because its early exit is commented out, :267, yet its host scan reads only those, :371-374);
//   * 2 sincos per BOX instead of per PAIR (prep kernel), identical values;
//   * a conservative separating-axis pre-filter rejects pairs whose exact result is provably
//     "0 candidate points -> area 0 -> IoU 0" (DESIGN.md, "filter soundness"); survivors are compacted
//     through a shared-memory queue so the ~1k-instruction exact path runs with full warps;
//   * the 50 MB mask never leaves HBM: the greedy scan runs on the device.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_segmented_radix_sort.cuh>
#include <cub/util_type.cuh>

#include <type_traits>

#include "common.cuh"
#include "rbox_exact.cuh"

namespace ryolo {

typedef unsigned long long u64;

constexpr int TB = 64;            // boxes per tile side == bits per mask word (reference threadsPerBlock, :20)
constexpr int CH = 8;             // column blocks handled per CTA
constexpr int MASK_THREADS = 256;
constexpr int SCAN_THREADS = 1024;
constexpr int kRowChunkBlocks = 16;   // row blocks per lazy-mask chunk (1024 boxes)

// field indices of the SoA geometry array geom[f * n_pad + i]
enum {
  F_PX = 0, F_PY = 4, F_ABX = 8, F_ABY = 9, F_ADX = 10, F_ADY = 11, F_ABAB = 12, F_ADAD = 13,
  F_W = 14, F_H = 15, F_AREA = 16, F_CX = 17, F_CY = 18, F_RAD = 19, F_UX = 20, F_UY = 21,
  F_HW = 22, F_HH = 23
};

// Segments: S independent NMS problems (one per image; the CLASSES kernels run one NMS per class inside it) in ONE set
// of launches.  Segment s owns rows
// [s*cap, s*cap + count_s) of dets; count_s comes from device memory (the candidate selection never visits the host) or
// from the host (the single-problem r_nms entry point); at most `limit` boxes (the best-scored) enter the NMS.
struct SegArgs {
  const int* n_dev;   // [S] candidate counts, or nullptr: every segment has n_host boxes
  int n_host;
  int limit;          // boxes entering NMS per segment = min(count, limit)
  int cap;            // rows per segment of dets / keys / order / keep_out
  int n_pad;          // cap rounded up to the tile size: stride of the geometry arrays / keep flags / mask rows
  int cbs;            // n_pad / 64: words per mask row, entries of remv / keptw per segment
};
__device__ __forceinline__ int seg_count(const SegArgs& a, int seg) {
  const int n = a.n_dev ? a.n_dev[seg] : a.n_host;
  return n < 0 ? 0 : (n < a.cap ? n : a.cap);
}
__device__ __forceinline__ int seg_n(const SegArgs& a, int seg) {
  const int n = seg_count(a, seg);
  return n < a.limit ? n : a.limit;
}

__global__ void rnms_keys_kernel(const float* __restrict__ dets, SegArgs sa, float* __restrict__ keys,
                                 int* __restrict__ vals, int* __restrict__ seg_begin, int* __restrict__ seg_end) {
  const int seg = blockIdx.y;
  const int n = seg_count(sa, seg);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0 && seg_begin) {
    seg_begin[seg] = seg * sa.cap;
    seg_end[seg] = seg * sa.cap + n;
  }
  if (i < n) {
    keys[(size_t)seg * sa.cap + i] = dets[((size_t)seg * sa.cap + i) * 6 + 5];
    vals[(size_t)seg * sa.cap + i] = i;
  }
}

// Class-aware form (CLASSES): dets rows are (x, y, w, h, theta, score, class_conf, class).  A segment is one image with
// its boxes of every class, sorted by (class asc, score desc, row asc); the mask only sets bits of same-class pairs, so
// the greedy scan over that order is exactly one NMS per class.  A box's "group" encodes its class so that it is
// non-increasing along the sort order: 2^24 - class for a class id that is an integer in [0, 2^24) with a score > 0,
// else 0 -- such a box sorts last and neither suppresses nor is suppressed.
constexpr float kClassLimit = 16777216.f;   // 2^24: class ids below it are exact in fp32
__device__ __forceinline__ int class_group(float score, float cls) {
  return (score > 0.f && cls >= 0.f && cls < kClassLimit && cls == floorf(cls)) ? (int)(kClassLimit - cls) : 0;
}

__global__ void rnms_class_keys_kernel(const float* __restrict__ dets, SegArgs sa, u64* __restrict__ keys,
                                       int* __restrict__ vals, int* __restrict__ seg_begin, int* __restrict__ seg_end) {
  const int seg = blockIdx.y;
  const int n = seg_count(sa, seg);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) {
    seg_begin[seg] = seg * sa.cap;
    seg_end[seg] = seg * sa.cap + n;
  }
  if (i < n) {
    const float* d = dets + ((size_t)seg * sa.cap + i) * 8;
    const float score = d[5];
    const int grp = class_group(score, d[7]);
    keys[(size_t)seg * sa.cap + i] = grp ? ((u64)grp << 32) | __float_as_uint(score) : 0ull;
    vals[(size_t)seg * sa.cap + i] = i;
  }
}

// One thread per score-sorted box: gather, pinned corner arithmetic, filter data.  CLASSES: 8-column rows, and the
// box's group goes to grp[seg * n_pad + i] (0 for padding).
template <bool CLASSES>
__global__ void rnms_prep_kernel(const float* __restrict__ dets, const int* __restrict__ order_in, SegArgs sa,
                                 float* __restrict__ sorted_boxes, int* __restrict__ order_out,
                                 float* __restrict__ geom, unsigned char* __restrict__ keep_flag, int* __restrict__ grp) {
  constexpr int DW = CLASSES ? 8 : 6;
  const int seg = blockIdx.y;
  const int n = seg_n(sa, seg), n_pad = sa.n_pad;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pad) return;
  if constexpr (CLASSES) {
    const int src = i < n ? order_in[(size_t)seg * sa.cap + i] : 0;
    const float* d = dets + ((size_t)seg * sa.cap + src) * 8;
    grp[(size_t)seg * n_pad + i] = i < n ? class_group(d[5], d[7]) : 0;
  }
  dets += (size_t)seg * sa.cap * DW;
  order_in += (size_t)seg * sa.cap;
  sorted_boxes += (size_t)seg * sa.cap * 6;
  order_out += (size_t)seg * sa.cap;
  geom += (size_t)seg * kGeomFields * n_pad;
  keep_flag += (size_t)seg * n_pad;
  keep_flag[i] = 0;                       // flags are indexed by ORIGINAL row (< count <= cap <= n_pad)
  float g[kGeomFields];
#pragma unroll
  for (int f = 0; f < kGeomFields; f++) g[f] = 0.f;
  if (i < n) {
    const int src = order_in[i];
    order_out[i] = src;
    float b[6];
#pragma unroll
    for (int k = 0; k < 6; k++) {
      b[k] = dets[(size_t)src * DW + k];
      sorted_boxes[(size_t)i * 6 + k] = b[k];
    }
    const float cx = b[0], cy = b[1], w = b[2], h = b[3], ang = b[4];
    float px[4], py[4], c, s;
    exact_corners(cx, cy, w, h, ang, px, py, &c, &s);
#pragma unroll
    for (int k = 0; k < 4; k++) {
      g[F_PX + k] = px[k];
      g[F_PY + k] = py[k];
    }
    // in_rect invariants (:143-155): ab = P1 - P0, ad = P3 - P0
    const float abx = __fsub_rn(px[1], px[0]), aby = __fsub_rn(py[1], py[0]);
    const float adx = __fsub_rn(px[3], px[0]), ady = __fsub_rn(py[3], py[0]);
    g[F_ABX] = abx; g[F_ABY] = aby; g[F_ADX] = adx; g[F_ADY] = ady;
    g[F_ABAB] = __fmaf_rn(abx, abx, __fmul_rn(aby, aby));
    g[F_ADAD] = __fmaf_rn(adx, adx, __fmul_rn(ady, ady));
    g[F_W] = w; g[F_H] = h;
    g[F_AREA] = __fmul_rn(w, h);
    // conservative filter data: only for well-conditioned boxes, else "never reject"
    const float mag = fabsf(cx) + fabsf(cy) + fmaxf(fabsf(w), fabsf(h));
    const bool ok = isfinite(cx) && isfinite(cy) && isfinite(w) && isfinite(h) && isfinite(ang) && w > 0.f &&
                    h > 0.f && fminf(w, h) >= 2.5e-4f * mag;
    const float inf = __int_as_float(0x7f800000);
    const float pad = 2e-3f * 0.5f * (w + h) + 1e-5f * mag;
    g[F_CX] = cx; g[F_CY] = cy;
    g[F_UX] = c; g[F_UY] = s;
    g[F_HW] = ok ? 0.5f * w + pad : inf;
    g[F_HH] = ok ? 0.5f * h + pad : inf;
    g[F_RAD] = ok ? 0.5f * sqrtf(w * w + h * h) * 1.002f + pad : inf;
  }
#pragma unroll
  for (int f = 0; f < kGeomFields; f++) geom[(size_t)f * n_pad + i] = g[f];
}

struct TileGeom {  // accessor over a shared-memory SoA tile [kGeomFields][TB]
  const float* t;
  int i;
  __device__ __forceinline__ float f(int field) const { return t[field * TB + i]; }
  __device__ __forceinline__ float px(int k) const { return f(F_PX + k); }
  __device__ __forceinline__ float py(int k) const { return f(F_PY + k); }
  __device__ __forceinline__ float abx() const { return f(F_ABX); }
  __device__ __forceinline__ float aby() const { return f(F_ABY); }
  __device__ __forceinline__ float adx() const { return f(F_ADX); }
  __device__ __forceinline__ float ady() const { return f(F_ADY); }
  __device__ __forceinline__ float abab() const { return f(F_ABAB); }
  __device__ __forceinline__ float adad() const { return f(F_ADAD); }
};

struct MaskSmem {
  float row[kGeomFields * TB];
  float col[kGeomFields * TB];
  float scratch[3 * kMaxPts * MASK_THREADS];
  u64 mask[TB * CH];
  unsigned short queue[TB * TB];    // stage A1 survivors (bounding circles)
  unsigned short queue2[TB * TB];   // stage A2 survivors (separating axes) = exact-path work list
  int cnt, cnt2;
};
struct MaskSmemClasses : MaskSmem {
  int grp_row[TB];
  int grp_col[TB];
};

// Conservative "provably no intersection" test.  true => the exact path would find 0 candidate
// points (so IoU == 0 exactly); false => unknown, run the exact path.  NaN/inf anywhere => false.
__device__ __forceinline__ bool surely_disjoint(float rcx, float rcy, float rrad, float rux, float ruy, float rhw,
                                                float rhh, float ccx, float ccy, float crad, float cux, float cuy,
                                                float chw, float chh) {
  const float dx = ccx - rcx, dy = ccy - rcy;
  const float R = rrad + crad;
  if (dx * dx + dy * dy > R * R) return true;
  const float C = fabsf(rux * cux + ruy * cuy);
  const float S = fabsf(rux * cuy - ruy * cux);
  if (fabsf(dx * rux + dy * ruy) > rhw + chw * C + chh * S) return true;
  if (fabsf(dy * rux - dx * ruy) > rhh + chw * S + chh * C) return true;
  if (fabsf(dx * cux + dy * cuy) > chw + rhw * C + rhh * S) return true;
  if (fabsf(dy * cux - dx * cuy) > chh + rhw * S + rhh * C) return true;
  return false;
}

// `remv` (optional): suppression state at launch time (bit set = box already suppressed by a kept box of an earlier
// row chunk).  Rows and columns that are already suppressed are skipped: their mask bits can never influence the
// greedy scan (a suppressed row is never kept, so its mask row is never read; a suppressed column stays suppressed).
// CLASSES: only same-group pairs are candidates, and the column loop stops at the first later tile whose first group is
// below the row tile's last group (groups never increase along the rows, so no later tile can hold a same-class pair);
// the words it does not evaluate are written as zeros.
template <bool CLASSES>
__global__ void __launch_bounds__(MASK_THREADS, 3) rnms_mask_kernel(const float* __restrict__ geom, SegArgs sa, float thr,
                                                                 int use_filter, u64* __restrict__ mask, int rb_begin,
                                                                 const u64* __restrict__ remv, const int* __restrict__ grp) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  MaskSmem& sm = *reinterpret_cast<MaskSmem*>(smem_raw);
  int* grp_row = nullptr;
  int* grp_col = nullptr;
  if constexpr (CLASSES) {
    grp_row = reinterpret_cast<MaskSmemClasses*>(smem_raw)->grp_row;
    grp_col = reinterpret_cast<MaskSmemClasses*>(smem_raw)->grp_col;
  }
  const int seg = blockIdx.z;
  const int n = seg_n(sa, seg), n_pad = sa.n_pad, cbs = sa.cbs;
  const int col_blocks = (n + TB - 1) / TB;          // of THIS segment
  const int rb = rb_begin + blockIdx.y;
  const int cb0 = rb + blockIdx.x * CH;
  if (rb >= col_blocks || cb0 >= col_blocks) return;
  geom += (size_t)seg * kGeomFields * n_pad;
  mask += (size_t)seg * n_pad * cbs;
  if (remv) remv += (size_t)seg * cbs;
  const u64 row_dead = remv ? remv[rb] : 0ull;
  if (row_dead == ~0ull) return;   // every row of this block is already suppressed: nothing it could contribute
  const int ncols = min(CH, col_blocks - cb0);
  const int tid = threadIdx.x;

  for (int e = tid; e < kGeomFields * TB; e += MASK_THREADS) {
    const int f = e / TB, i = e % TB;
    sm.row[e] = geom[(size_t)f * n_pad + rb * TB + i];
  }
  for (int e = tid; e < TB * CH; e += MASK_THREADS) sm.mask[e] = 0ull;
  int grp_last = 0;   // group of the row tile's last box
  if constexpr (CLASSES) {
    grp += (size_t)seg * n_pad;
    for (int e = tid; e < TB; e += MASK_THREADS) grp_row[e] = grp[rb * TB + e];
    grp_last = grp[min(n, (rb + 1) * TB) - 1];
  }

  const int r = tid & (TB - 1);
  const int g = tid >> 6;  // 4 groups of 16 columns
  const int lane = tid & 31;

  for (int cc = 0; cc < ncols; cc++) {
    const int cbi = cb0 + cc;
    if constexpr (CLASSES) {
      const int grp_first = grp[cbi * TB];
      if (cbi > rb && (grp_first == 0 || grp_first < grp_last)) break;   // uniform for the CTA
    }
    const u64 col_dead = remv ? remv[cbi] : 0ull;
    if (col_dead == ~0ull) continue;   // uniform for the CTA: whole column tile already suppressed
    __syncthreads();  // previous tile fully consumed (also covers the row-tile load on cc == 0)
    for (int e = tid; e < kGeomFields * TB; e += MASK_THREADS) {
      const int f = e / TB, i = e % TB;
      sm.col[e] = geom[(size_t)f * n_pad + cbi * TB + i];
    }
    if constexpr (CLASSES) {
      for (int e = tid; e < TB; e += MASK_THREADS) grp_col[e] = grp[cbi * TB + e];
    }
    if (tid == 0) { sm.cnt = 0; sm.cnt2 = 0; }
    __syncthreads();

    // ---- stage A1: bounding circles, 16 pairs per thread, ONE compaction per thread ----
    {
      const float rcx = sm.row[F_CX * TB + r], rcy = sm.row[F_CY * TB + r], rrad = sm.row[F_RAD * TB + r];
      const bool row_ok = rb * TB + r < n && !((row_dead >> r) & 1ull);
      unsigned pass = 0;
      if (row_ok) {
#pragma unroll
        for (int k = 0; k < 16; k++) {
          const int c = g * 16 + k;   // same column for the whole warp: shared-memory broadcast
          bool cand = (cbi * TB + c < n) && (cbi > rb || c > r) && !((col_dead >> c) & 1ull);
          if constexpr (CLASSES) cand = cand && grp_col[c] == grp_row[r] && grp_row[r] != 0;
          if (use_filter) {
            const float dx = sm.col[F_CX * TB + c] - rcx, dy = sm.col[F_CY * TB + c] - rcy;
            const float R = rrad + sm.col[F_RAD * TB + c];
            cand = cand && !(dx * dx + dy * dy > R * R);
          }
          pass |= (cand ? 1u : 0u) << k;
        }
      }
      const int cnt = __popc(pass);
      int incl = cnt;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
      }
      int base = 0;
      if (lane == 31) base = atomicAdd(&sm.cnt, incl);
      base = __shfl_sync(0xffffffffu, base, 31) + incl - cnt;
      while (pass) {
        const int k = __ffs(pass) - 1;
        pass &= pass - 1;
        sm.queue[base++] = (unsigned short)((r << 6) | (g * 16 + k));
      }
    }
    __syncthreads();
    // ---- stage A2: separating axes on the circle survivors, converged warps ----
    {
      const int cnt1 = sm.cnt;
      for (int q0 = 0; q0 < cnt1; q0 += MASK_THREADS) {
        const int q = q0 + tid;
        bool keep = false;
        int e = 0;
        if (q < cnt1) {
          e = sm.queue[q];
          const int qr = e >> 6, qc = e & 63;
          keep = !use_filter ||
                 !surely_disjoint(sm.row[F_CX * TB + qr], sm.row[F_CY * TB + qr], sm.row[F_RAD * TB + qr],
                                  sm.row[F_UX * TB + qr], sm.row[F_UY * TB + qr], sm.row[F_HW * TB + qr],
                                  sm.row[F_HH * TB + qr], sm.col[F_CX * TB + qc], sm.col[F_CY * TB + qc],
                                  sm.col[F_RAD * TB + qc], sm.col[F_UX * TB + qc], sm.col[F_UY * TB + qc],
                                  sm.col[F_HW * TB + qc], sm.col[F_HH * TB + qc]);
        }
        const unsigned mk = __ballot_sync(0xffffffffu, keep);
        if (mk) {
          int base = 0;
          if (lane == 0) base = atomicAdd(&sm.cnt2, __popc(mk));
          base = __shfl_sync(0xffffffffu, base, 0);
          if (keep) sm.queue2[base + __popc(mk & ((1u << lane) - 1u))] = (unsigned short)e;
        }
      }
    }
    __syncthreads();

    // ---- stage B: exact overlap on the survivors, one pair per thread ----
    {
      const int cnt = sm.cnt2;
      PtScratch sc;
      sc.x = sm.scratch + tid;
      sc.y = sm.scratch + kMaxPts * MASK_THREADS + tid;
      sc.k = sm.scratch + 2 * kMaxPts * MASK_THREADS + tid;
      sc.stride = MASK_THREADS;
      for (int q = tid; q < cnt; q += MASK_THREADS) {
        const int e = sm.queue2[q];
        const int qr = e >> 6, qc = e & 63;
        TileGeom g1{sm.row, qr}, g2{sm.col, qc};
        const float inter = exact_inter_area(g1, g2, sc);
        const float iou = exact_iou_from_inter(g1.f(F_AREA), g2.f(F_W), g2.f(F_H), inter);
        if (iou > thr) atomicOr(&sm.mask[qr * CH + cc], 1ull << qc);
      }
    }
  }
  __syncthreads();
  for (int e = tid; e < TB * ncols; e += MASK_THREADS) {
    const int rr = e / ncols, cc = e % ncols;
    const int row = rb * TB + rr;
    if (row < n) mask[(size_t)row * cbs + cb0 + cc] = sm.mask[rr * CH + cc];
  }
}

// Greedy scan (reference host loop :358-376) + original-index compaction (:380-383), one CTA, software-pipelined:
//   warp 0 is the serial critical path.  For block b it needs remv[b] = OR of the mask word b of every box kept so far.
//   Contributions of blocks <= b-2 are accumulated into shared remv[] by the helper warps one iteration behind;
//   the contribution of block b-1 comes from registers: warp 0 prefetches, one block ahead, the diagonal words
//   (64 rows x word b) and the next-column words (64 rows x word b+1) of the block, so no global-memory latency sits
//   on the chain -- only ~kept(b) iterations of {find-first-set, 64-bit shuffle, OR}.
//   Helper warps (1..31), after the per-block barrier, OR the rows kept in block b into remv[j], j >= b+2, one warp
//   per 32 consecutive columns (coalesced 256-byte row segments, up to 8 loads in flight per lane), while warp 0 is
//   already resolving block b+1.
__device__ __forceinline__ u64 shfl_u64(u64 v, int src) {
  const unsigned lo = __shfl_sync(0xffffffffu, (unsigned)v, src);
  const unsigned hi = __shfl_sync(0xffffffffu, (unsigned)(v >> 32), src);
  return ((u64)hi << 32) | lo;
}

// Processes row blocks [b_begin, b_end) of the greedy scan; the suppression state `remv_g` and the kept bits `keptw_g`
// live in global memory between launches (row chunks alternate with mask launches that skip what is already
// suppressed).  The last launch (`final`) also compacts the kept ORIGINAL indices.
__global__ void __launch_bounds__(SCAN_THREADS) rnms_scan_kernel(const u64* __restrict__ mask, SegArgs sa,
                                                                 const int* __restrict__ order,
                                                                 unsigned char* __restrict__ keep_flag,
                                                                 long long* __restrict__ keep_out,
                                                                 int* __restrict__ num_keep, int b_begin, int b_end,
                                                                 u64* __restrict__ remv_g, u64* __restrict__ keptw_g,
                                                                 int final) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int seg = blockIdx.x;                      // one scan CTA per segment, all segments concurrently
  const int n = seg_n(sa, seg), n_raw = seg_count(sa, seg), cbs = sa.cbs;
  const int col_blocks = (n + TB - 1) / TB;        // of THIS segment
  b_begin = min(b_begin, col_blocks);
  b_end = min(b_end, col_blocks);
  mask += (size_t)seg * sa.n_pad * cbs;
  order += (size_t)seg * sa.cap;
  keep_flag += (size_t)seg * sa.n_pad;
  keep_out += (size_t)seg * sa.cap;
  num_keep += seg;
  remv_g += (size_t)seg * cbs;
  keptw_g += (size_t)seg * cbs;
  u64* remv = reinterpret_cast<u64*>(smem_raw);   // [cbs]
  u64* keptw = remv + cbs;                         // [cbs] kept bits per block
  __shared__ int s_warp_sums[SCAN_THREADS / 32];
  __shared__ int s_base;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int j = tid; j < col_blocks; j += SCAN_THREADS) {
    remv[j] = remv_g[j];
    keptw[j] = keptw_g[j];
  }
  __syncthreads();

  auto ld = [&](int row, int word) -> u64 {
    return (row < n && word < col_blocks) ? mask[(size_t)row * cbs + word] : 0ull;
  };
  u64 dg0 = 0, dg1 = 0, nx0 = 0, nx1 = 0, ext = 0;
  if (warp == 0) {
    const int r0 = b_begin * TB + lane;
    dg0 = ld(r0, b_begin); dg1 = ld(r0 + 32, b_begin);
    nx0 = ld(r0, b_begin + 1); nx1 = ld(r0 + 32, b_begin + 1);
  }
  for (int b = b_begin; b < b_end; b++) {
    if (warp == 0) {
      const int r1 = (b + 1) * TB + lane;
      const u64 pd0 = ld(r1, b + 1), pd1 = ld(r1 + 32, b + 1);   // consumed next iteration
      const u64 pn0 = ld(r1, b + 2), pn1 = ld(r1 + 32, b + 2);
      const int nvalid = min(TB, n - b * TB);
      const u64 valid = nvalid >= 64 ? ~0ull : ((1ull << nvalid) - 1ull);
      u64 rm = remv[b] | ext;
      u64 kept = 0ull;
      u64 avail = ~rm & valid;
      while (avail) {
        const int i = __ffsll((long long)avail) - 1;
        kept |= 1ull << i;
        rm |= shfl_u64(i < 32 ? dg0 : dg1, i & 31);
        avail = ~rm & valid & ~((2ull << i) - 1ull);
      }
      // contribution of this block's kept rows to column b+1, from the prefetched registers
      const u64 x = (((kept >> lane) & 1ull) ? nx0 : 0ull) | (((kept >> (lane + 32)) & 1ull) ? nx1 : 0ull);
      const unsigned xlo = __reduce_or_sync(0xffffffffu, (unsigned)x);
      const unsigned xhi = __reduce_or_sync(0xffffffffu, (unsigned)(x >> 32));
      ext = ((u64)xhi << 32) | xlo;
      if (lane == 0) keptw[b] = kept;
      dg0 = pd0; dg1 = pd1; nx0 = pn0; nx1 = pn1;
    }
    __syncthreads();
    if (warp >= 1) {
      const u64 kept = keptw[b];
      const int first = b + 2;
      for (int j0 = first + (warp - 1) * 32; j0 < col_blocks; j0 += (SCAN_THREADS / 32 - 1) * 32) {
        const int j = j0 + lane;
        if (j < col_blocks) {
          u64 acc = 0ull;
          u64 bits = kept;
          const u64* base = mask + (size_t)b * TB * cbs + j;
          while (bits) {
            u64 v[8];
#pragma unroll
            for (int u = 0; u < 8; u++) {
              v[u] = 0ull;
              if (bits) {
                const int i = __ffsll((long long)bits) - 1;
                bits &= bits - 1;
                v[u] = base[(size_t)i * cbs];
              }
            }
            acc |= ((v[0] | v[1]) | (v[2] | v[3])) | ((v[4] | v[5]) | (v[6] | v[7]));
          }
          remv[j] |= acc;   // column j is owned by exactly one lane of one warp
        }
      }
    }
  }
  __syncthreads();
  if (tid == 0 && b_end < col_blocks) remv[b_end] |= ext;   // last block's contribution to the next chunk's first column
  __syncthreads();
  if (!final) {
    for (int j = tid; j < col_blocks; j += SCAN_THREADS) {
      remv_g[j] = remv[j];
      keptw_g[j] = keptw[j];
    }
    return;
  }
  // flag kept boxes by ORIGINAL index
  for (int i = tid; i < n; i += SCAN_THREADS)
    if ((keptw[i >> 6] >> (i & 63)) & 1ull) keep_flag[order[i]] = 1;
  if (tid == 0) s_base = 0;
  __syncthreads();
  // compaction over ORIGINAL indices (all count rows of the segment, not only the `limit` that entered NMS), ascending
  for (int start = 0; start < n_raw; start += SCAN_THREADS) {
    const int i = start + tid;
    const int flag = (i < n_raw) ? (int)keep_flag[i] : 0;
    const unsigned bal = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) s_warp_sums[warp] = __popc(bal);
    __syncthreads();
    int prefix = 0;
    for (int w = 0; w < warp; w++) prefix += s_warp_sums[w];
    const int base = s_base;
    if (flag) keep_out[base + prefix + __popc(bal & ((1u << lane) - 1u))] = (long long)i;
    __syncthreads();
    if (tid == SCAN_THREADS - 1) s_base = base + prefix + __popc(bal);
    __syncthreads();
  }
  if (tid == 0) *num_keep = s_base;
}

struct RnmsPlan {
  int segs, cap, n_pad, cbs;
  size_t cub_bytes;
  float* sorted_boxes;
  int* order;
  float* keys[2];
  u64* keys64[2];    // class-aware form: (group << 32 | score bits) sort keys instead of keys[]
  int* grp;          // class-aware form: [segs][n_pad] group of each sorted box
  int* vals[2];
  float* geom;
  u64* mask;
  unsigned char* keep_flag;
  u64* remv_g;
  u64* keptw_g;
  int* seg_begin;
  int* seg_end;
  void* cub_temp;
  size_t total;
};

constexpr int kClassKeyBits = 57;   // group (<= 2^24, 25 bits) << 32 | score bits

template <typename K>
static size_t cub_temp_bytes(int items, int segs, int end_bit) {
  size_t bytes = 0, bytes2 = 0;
  cub::DoubleBuffer<K> k(nullptr, nullptr);
  cub::DoubleBuffer<int> v(nullptr, nullptr);
  cudaError_t e = cub::DeviceRadixSort::SortPairsDescending(nullptr, bytes, k, v, items, 0, end_bit, (cudaStream_t)0);
  if (e != cudaSuccess) {
    cudaGetLastError();  // clear (no device in this process: size-only query)
    bytes = 0;
  }
  e = cub::DeviceSegmentedRadixSort::SortPairsDescending(nullptr, bytes2, k, v, items, segs, (const int*)nullptr,
                                                         (const int*)nullptr, 0, end_bit, (cudaStream_t)0);
  if (e != cudaSuccess) {
    cudaGetLastError();
    bytes2 = 0;
  }
  if (bytes2 > bytes) bytes = bytes2;
  // conservative floor so that a size computed on a GPU-less host still fits the real query
  const size_t floor_bytes = (size_t)1 << 20;
  return bytes > floor_bytes ? bytes : floor_bytes + (size_t)16 * (size_t)(items > 0 ? items : 0);
}

static void plan_rnms(int segs, int cap, void* ws, RnmsPlan* p, bool classes = false) {
  p->segs = segs;
  p->cap = cap;
  p->n_pad = (cap + TB - 1) / TB * TB;
  p->cbs = p->n_pad / TB;
  const size_t items = (size_t)segs * cap;
  p->cub_bytes = classes ? cub_temp_bytes<u64>((int)items, segs, kClassKeyBits)
                         : cub_temp_bytes<float>((int)items, segs, 32);
  Carver c(ws);
  p->sorted_boxes = c.take<float>(items * 6);
  p->order = c.take<int>(items);
  p->keys[0] = p->keys[1] = nullptr;
  p->keys64[0] = p->keys64[1] = nullptr;
  p->grp = nullptr;
  if (classes) {
    p->keys64[0] = c.take<u64>(items);
    p->keys64[1] = c.take<u64>(items);
    p->grp = c.take<int>((size_t)segs * p->n_pad);
  } else {
    p->keys[0] = c.take<float>(items);
    p->keys[1] = c.take<float>(items);
  }
  p->vals[0] = c.take<int>(items);
  p->vals[1] = c.take<int>(items);
  p->geom = c.take<float>((size_t)segs * kGeomFields * p->n_pad);
  p->mask = c.take<u64>((size_t)segs * p->n_pad * p->cbs);
  p->keep_flag = c.take<unsigned char>((size_t)segs * p->n_pad);
  p->remv_g = c.take<u64>(2 * (size_t)segs * p->cbs);
  p->keptw_g = p->remv_g + (size_t)segs * p->cbs;
  p->seg_begin = c.take<int>(2 * (size_t)segs);
  p->seg_end = p->seg_begin + segs;
  p->cub_temp = c.take<unsigned char>(p->cub_bytes);
  p->total = align_up(c.off, 256);
}

}  // namespace ryolo

using namespace ryolo;

extern "C" size_t ryolo_rnms_workspace_bytes(int n) {
  if (n <= 0) return 256;
  RnmsPlan p;
  plan_rnms(1, n, nullptr, &p);
  return p.total;
}
extern "C" size_t ryolo_rnms_batched_workspace_bytes(int segments, int cap) {
  if (segments <= 0 || cap <= 0) return 256;
  RnmsPlan p;
  plan_rnms(segments, cap, nullptr, &p);
  return p.total;
}

template <bool CLASSES>
static int rnms_mask_and_scan(const RnmsPlan& p, const SegArgs& sa, float thr, bool full_mask, int64_t* keep_out,
                              int32_t* num_keep, cudaStream_t stream) {
  using MaskSmemT = typename std::conditional<CLASSES, MaskSmemClasses, MaskSmem>::type;
  RYOLO_SMEM_OPT_IN(rnms_mask_kernel<CLASSES>, sizeof(MaskSmemT));
  const size_t smem = (size_t)p.cbs * sizeof(u64) * 2;
  if (smem > 200 * 1024) {
    set_err("ryolo_rnms: cap=%d too large for the single-CTA scan (col_blocks=%d)", p.cap, p.cbs);
    return RYOLO_E_UNSUPPORTED;
  }
  if (smem > 40 * 1024)
    RYOLO_CUDA_TRY(cudaFuncSetAttribute(rnms_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  RYOLO_CUDA_TRY(cudaMemsetAsync(p.remv_g, 0, 2 * (size_t)p.segs * p.cbs * sizeof(u64), stream));
  // Row chunks of `chunk` blocks: mask(chunk rows x all later columns, skipping what earlier chunks suppressed),
  // then scan(chunk) -- for ALL segments at once (grid z / one scan CTA per segment).  full_mask computes every
  // upper-triangle tile in one launch like the reference.
  const int chunk = full_mask ? p.cbs : kRowChunkBlocks;
  for (int b0 = 0; b0 < p.cbs; b0 += chunk) {
    const int b1 = b0 + chunk < p.cbs ? b0 + chunk : p.cbs;
    dim3 grid((p.cbs - b0 + CH - 1) / CH, b1 - b0, p.segs);
    rnms_mask_kernel<CLASSES><<<grid, MASK_THREADS, sizeof(MaskSmemT), stream>>>(
        p.geom, sa, thr, thr >= 0.f ? 1 : 0, p.mask, b0, full_mask ? nullptr : p.remv_g, p.grp);
    RYOLO_LAUNCH_CHECK();
    rnms_scan_kernel<<<p.segs, SCAN_THREADS, smem, stream>>>(p.mask, sa, p.order, p.keep_flag,
                                                             reinterpret_cast<long long*>(keep_out), num_keep, b0, b1,
                                                             p.remv_g, p.keptw_g, b1 == p.cbs ? 1 : 0);
    RYOLO_LAUNCH_CHECK();
  }
  return RYOLO_OK;
}

static int rnms_impl(const float* dets, int segs, int cap, const int32_t* n_dev, int n_host, int limit, float thr,
                     int64_t* keep_out, int32_t* num_keep, void* workspace, size_t workspace_bytes, void* stream_,
                     bool full_mask, bool classes = false) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(dets != nullptr && keep_out != nullptr && workspace != nullptr && num_keep != nullptr);
  RYOLO_ARG_CHECK(segs > 0 && segs <= 65535 && cap > 0 && limit > 0);
  RYOLO_ARG_CHECK((long long)segs * cap < (1ll << 31));
  RYOLO_ARG_CHECK((reinterpret_cast<uintptr_t>(workspace) & 255) == 0);
  RnmsPlan p;
  plan_rnms(segs, cap, workspace, &p, classes);
  if (p.total > workspace_bytes) {
    set_err("ryolo_rnms: workspace %zu B < required %zu B", workspace_bytes, p.total);
    return RYOLO_E_WORKSPACE;
  }
  SegArgs sa;
  sa.n_dev = n_dev;
  sa.n_host = n_host;
  sa.limit = limit;
  sa.cap = cap;
  sa.n_pad = p.n_pad;
  sa.cbs = p.cbs;
  const int T = 256;
  const bool segmented = segs > 1 || n_dev != nullptr;
  cub::DoubleBuffer<float> dk(p.keys[0], p.keys[1]);
  cub::DoubleBuffer<int> dv(p.vals[0], p.vals[1]);
  size_t need = 0;
  const int items = segs * cap;
  if (classes) {
    // stable per-segment sort by (group desc = class asc, score desc); rows beyond a segment's count are never read
    rnms_class_keys_kernel<<<dim3((cap + T - 1) / T, segs), T, 0, stream>>>(dets, sa, p.keys64[0], p.vals[0],
                                                                           p.seg_begin, p.seg_end);
    RYOLO_LAUNCH_CHECK();
    cub::DoubleBuffer<u64> dk64(p.keys64[0], p.keys64[1]);
    RYOLO_CUDA_TRY(cub::DeviceSegmentedRadixSort::SortPairsDescending(nullptr, need, dk64, dv, items, segs, p.seg_begin,
                                                                      p.seg_end, 0, kClassKeyBits, stream));
    if (need > p.cub_bytes) {
      set_err("ryolo_rnms: sort scratch %zu B > planned %zu B", need, p.cub_bytes);
      return RYOLO_E_WORKSPACE;
    }
    size_t tmp = p.cub_bytes;
    RYOLO_CUDA_TRY(cub::DeviceSegmentedRadixSort::SortPairsDescending(p.cub_temp, tmp, dk64, dv, items, segs,
                                                                      p.seg_begin, p.seg_end, 0, kClassKeyBits, stream));
    count_launch(4);
    rnms_prep_kernel<true><<<dim3((p.n_pad + T - 1) / T, segs), T, 0, stream>>>(
        dets, dv.Current(), sa, p.sorted_boxes, p.order, p.geom, p.keep_flag, p.grp);
    RYOLO_LAUNCH_CHECK();
    return rnms_mask_and_scan<true>(p, sa, thr, full_mask, keep_out, num_keep, stream);
  }
  rnms_keys_kernel<<<dim3((cap + T - 1) / T, segs), T, 0, stream>>>(dets, sa, p.keys[0], p.vals[0],
                                                                   segmented ? p.seg_begin : nullptr, p.seg_end);
  RYOLO_LAUNCH_CHECK();
  if (!segmented) {
    RYOLO_CUDA_TRY(cub::DeviceRadixSort::SortPairsDescending(nullptr, need, dk, dv, n_host, 0, 32, stream));
  } else {
    RYOLO_CUDA_TRY(cub::DeviceSegmentedRadixSort::SortPairsDescending(nullptr, need, dk, dv, items, segs, p.seg_begin,
                                                                      p.seg_end, 0, 32, stream));
  }
  if (need > p.cub_bytes) {
    set_err("ryolo_rnms: sort scratch %zu B > planned %zu B", need, p.cub_bytes);
    return RYOLO_E_WORKSPACE;
  }
  size_t tmp = p.cub_bytes;
  if (!segmented) {
    RYOLO_CUDA_TRY(cub::DeviceRadixSort::SortPairsDescending(p.cub_temp, tmp, dk, dv, n_host, 0, 32, stream));
  } else {
    // stable per-segment sort by score, descending; rows beyond a segment's count are never read
    RYOLO_CUDA_TRY(cub::DeviceSegmentedRadixSort::SortPairsDescending(p.cub_temp, tmp, dk, dv, items, segs, p.seg_begin,
                                                                      p.seg_end, 0, 32, stream));
  }
  count_launch(4);  // radix sort passes (library kernels, counted as a lower bound)
  rnms_prep_kernel<false><<<dim3((p.n_pad + T - 1) / T, segs), T, 0, stream>>>(
      dets, dv.Current(), sa, p.sorted_boxes, p.order, p.geom, p.keep_flag, nullptr);
  RYOLO_LAUNCH_CHECK();
  return rnms_mask_and_scan<false>(p, sa, thr, full_mask, keep_out, num_keep, stream);
}

static int rnms_single(const float* dets, int n, float thr, int64_t* keep_out, int32_t* num_keep, void* workspace,
                       size_t workspace_bytes, void* stream_, bool full_mask) {
  RYOLO_ARG_CHECK(n >= 0);
  RYOLO_ARG_CHECK(num_keep != nullptr);
  if (n == 0) {
    RYOLO_CUDA_TRY(cudaMemsetAsync(num_keep, 0, sizeof(int32_t), static_cast<cudaStream_t>(stream_)));
    return RYOLO_OK;
  }
  return rnms_impl(dets, 1, n, nullptr, n, n, thr, keep_out, num_keep, workspace, workspace_bytes, stream_, full_mask);
}

extern "C" int ryolo_rnms(const float* dets, int n, float thr, int64_t* keep_out, int32_t* num_keep, void* workspace,
                          size_t workspace_bytes, void* stream_) {
  return rnms_single(dets, n, thr, keep_out, num_keep, workspace, workspace_bytes, stream_, false);
}
extern "C" int ryolo_rnms_full_mask(const float* dets, int n, float thr, int64_t* keep_out, int32_t* num_keep,
                                    void* workspace, size_t workspace_bytes, void* stream_) {
  return rnms_single(dets, n, thr, keep_out, num_keep, workspace, workspace_bytes, stream_, true);
}

extern "C" int ryolo_rnms_batched(const float* dets, int segments, int cap, const int32_t* n_dev, int limit, float thr,
                                  int64_t* keep_out, int32_t* num_keep, void* workspace, size_t workspace_bytes,
                                  void* stream_) {
  RYOLO_ARG_CHECK(n_dev != nullptr);
  return rnms_impl(dets, segments, cap, n_dev, 0, limit, thr, keep_out, num_keep, workspace, workspace_bytes, stream_, false);
}

extern "C" size_t ryolo_rnms_batched_classes_workspace_bytes(int segments, int cap) {
  if (segments <= 0 || cap <= 0) return 256;
  RnmsPlan p;
  plan_rnms(segments, cap, nullptr, &p, true);
  return p.total;
}

extern "C" int ryolo_rnms_batched_classes(const float* dets8, int segments, int cap, const int32_t* n_dev, float thr,
                                          int64_t* keep_out, int32_t* num_keep, void* workspace, size_t workspace_bytes,
                                          void* stream_) {
  RYOLO_ARG_CHECK(n_dev != nullptr);
  return rnms_impl(dets8, segments, cap, n_dev, 0, cap, thr, keep_out, num_keep, workspace, workspace_bytes, stream_,
                   false, true);
}

extern "C" int ryolo_rnms_debug_views(void* workspace, int n, const float** sorted_boxes, const int32_t** order,
                                      const unsigned long long** mask) {
  RYOLO_ARG_CHECK(workspace != nullptr && n > 0);
  RnmsPlan p;
  plan_rnms(1, n, workspace, &p);
  if (sorted_boxes) *sorted_boxes = p.sorted_boxes;
  if (order) *order = p.order;
  if (mask) *mask = p.mask;
  return RYOLO_OK;
}
