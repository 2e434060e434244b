// Batched candidate selection for detection (detect.py:204-213 -> non_max_suppression, utils/nms/nms.py:28-56) without
// host round trips: for every image of a decoded batch io [B, P, 6+nc], the `limit` most confident rows that pass the
// reference's candidate filter (conf = obj * max class conf > conf_thres, w, h > min_wh, all finite; nms.py:34-40) are
// gathered as NMS input [B, cap, 6] = (x, y, w, h, theta, conf), together with their count -- on the device.
//
// The reference has no cap (trained weights leave a few hundred candidates); a random-init network puts ~half of the
// 545 832 proposals above any threshold, and RNMS is quadratic, so detect caps the candidates per image (SURVEY.md 8d
// config 5).  The selection is exact: the top-`limit` rows by conf, ties resolved by lowest row index, for every
// distribution of conf (no histogram-bin surplus, whatever the number of rows sharing a value).
//   1. conf_thres >= 0, so every passing conf is a positive finite float and its fp32 bit pattern orders like the value.
//      One pass over io stores key = bits(conf) per row (0 = filtered out) and histograms bits 30..19 of the keys.
//   2. Radix select in three digits (bits 30..19, 18..7, 6..0), one 4096-bin histogram pass over the keys per digit,
//      each restricted to the keys that share the digits found so far -> v = the limit-th largest key, `above` = the
//      number of keys > v (< limit) and need = limit - above.  At most `limit` passing rows: v = 0, need = 0.
//   3. Ordered two-pass compaction (block counts -> scan -> write) of the rows with key > v and of the first `need`
//      rows with key == v: two block counts per 256 rows (above / tied), both scanned, so the output position of a row
//      is above_before + min(tied_before, need).  Deterministic, input order, exactly min(limit, #passing) rows.
// The batched RNMS then sorts the candidates by score (stable): the same order as a stable top-`limit` sort.
#include "common.cuh"
#include "filter.cuh"

namespace ryolo {

constexpr int SEL_BINS = 4096;
constexpr int SEL_T = 256;
constexpr int SEL_ROWS_PER_CTA = 8192;
constexpr int SEL_PASSES = 3;
__constant__ int c_sel_shift[SEL_PASSES] = {19, 7, 0};   // digit of pass d: bits [shift, shift + bits) of the key
__constant__ int c_sel_bits[SEL_PASSES] = {12, 12, 7};

struct SelState {
  unsigned prefix;   // the key digits found so far; after the last pass: v, the limit-th largest key
  int k;             // rank (1-based, from the top) of the wanted key among the keys that share `prefix`; after the
                     // last pass: need, the number of rows with key == v to take
  int done;          // at most `limit` rows pass: all of them are selected (v = 0, need = 0)
};

__device__ __forceinline__ unsigned sel_key(const float* __restrict__ row, int nc, float conf_thres, float min_wh) {
  float best; int bi; bool fin;
  class_max(row, nc, &best, &bi, &fin);
  const float conf = row[5] * best;
  return keep_row(row, conf, fin, conf_thres, min_wh) ? __float_as_uint(conf) : 0u;
}

// warp-aggregated shared-memory histogram update (many rows share one bin: dense or quantised confidences)
__device__ __forceinline__ void sel_hist_add(int* s_h, bool valid, int bin) {
  const unsigned same = __match_any_sync(0xffffffffu, valid ? bin : -1);
  if (valid && (threadIdx.x & 31) == __ffs(same) - 1) atomicAdd(&s_h[bin], __popc(same));
}

__device__ __forceinline__ void sel_hist_flush(const int* s_h, int* __restrict__ hist) {
  __syncthreads();
  for (int i = threadIdx.x; i < SEL_BINS; i += SEL_T)
    if (s_h[i]) atomicAdd(&hist[i], s_h[i]);
}

// pass 0: keys of all rows + histogram of their top digit
__global__ void __launch_bounds__(SEL_T) sel_key_hist_kernel(const float* __restrict__ io, int p, int nc,
                                                             float conf_thres, float min_wh,
                                                             unsigned* __restrict__ keys /*[B][p]*/,
                                                             int* __restrict__ hist /*[B][SEL_BINS]*/) {
  __shared__ int s_h[SEL_BINS];
  for (int i = threadIdx.x; i < SEL_BINS; i += SEL_T) s_h[i] = 0;
  __syncthreads();
  const int b = blockIdx.y;
  const int r0 = blockIdx.x * SEL_ROWS_PER_CTA;
  const int r1 = min(p, r0 + SEL_ROWS_PER_CTA);
  const float* base = io + (size_t)b * p * (6 + nc);
  for (int r = r0 + (int)threadIdx.x; r - (int)threadIdx.x < r1; r += SEL_T) {   // warp-uniform trip count
    unsigned key = 0;
    if (r < r1) {
      key = sel_key(base + (size_t)r * (6 + nc), nc, conf_thres, min_wh);
      keys[(size_t)b * p + r] = key;
    }
    sel_hist_add(s_h, key != 0, (int)(key >> 19));
  }
  sel_hist_flush(s_h, hist + (size_t)b * SEL_BINS);
}

// passes 1, 2: histogram of the next digit over the keys that share the digits found so far
__global__ void __launch_bounds__(SEL_T) sel_digit_hist_kernel(const unsigned* __restrict__ keys, int p, int pass,
                                                               const SelState* __restrict__ st,
                                                               int* __restrict__ hist) {
  __shared__ int s_h[SEL_BINS];
  const int b = blockIdx.y;
  if (st[b].done) return;
  const unsigned prefix = st[b].prefix;
  const int shift = c_sel_shift[pass], top = shift + c_sel_bits[pass];
  const unsigned dmask = (1u << c_sel_bits[pass]) - 1u;
  for (int i = threadIdx.x; i < SEL_BINS; i += SEL_T) s_h[i] = 0;
  __syncthreads();
  const int r0 = blockIdx.x * SEL_ROWS_PER_CTA;
  const int r1 = min(p, r0 + SEL_ROWS_PER_CTA);
  const unsigned* kb = keys + (size_t)b * p;
  for (int r = r0 + (int)threadIdx.x; r - (int)threadIdx.x < r1; r += SEL_T) {
    const unsigned key = r < r1 ? kb[r] : 0u;
    sel_hist_add(s_h, key != 0 && (key >> top) == prefix, (int)((key >> shift) & dmask));
  }
  sel_hist_flush(s_h, hist + (size_t)b * SEL_BINS);
}

// one CTA per image: suffix sums over the bins from the top; the bin whose suffix count first reaches k holds the wanted
// key -> append its digit to the prefix; its rank within that bin = k - (keys in the bins above it)
__global__ void __launch_bounds__(1024) sel_radix_kernel(const int* __restrict__ hist, int pass, int limit,
                                                         SelState* __restrict__ st) {
  __shared__ int s_part[1024];
  const int b = blockIdx.x, tid = threadIdx.x;
  if (pass > 0 && st[b].done) return;
  const unsigned prefix = pass ? st[b].prefix : 0u;
  const int k = pass ? st[b].k : limit;
  constexpr int PER = SEL_BINS / 1024;
  const int* h = hist + (size_t)b * SEL_BINS;
  int loc[PER];
  int sum = 0;
#pragma unroll
  for (int j = 0; j < PER; j++) {      // thread tid owns bins [tid*PER, tid*PER + PER)
    loc[j] = h[tid * PER + j];
    sum += loc[j];
  }
  s_part[tid] = sum;
  __syncthreads();
  // inclusive suffix scan over threads
  for (int o = 1; o < 1024; o <<= 1) {
    const int v = tid + o < 1024 ? s_part[tid + o] : 0;
    __syncthreads();
    s_part[tid] += v;
    __syncthreads();
  }
  if (pass == 0 && s_part[0] <= limit) {   // at most `limit` rows pass the filter: take them all
    if (tid == 0) st[b] = SelState{0u, 0, 1};
    return;
  }
  int above = tid + 1 < 1024 ? s_part[tid + 1] : 0;   // keys in bins above this thread's range
#pragma unroll
  for (int j = PER - 1; j >= 0; j--) {
    const int incl = above + loc[j];
    if (above < k && incl >= k)                        // exactly one (thread, j) satisfies this
      st[b] = SelState{(prefix << c_sel_bits[pass]) | (unsigned)(tid * PER + j), k - above, 0};
    above = incl;
  }
}

// per 256-row block: number of keys > v and number of keys == v, at [b][0][blk] and [b][1][blk]
__global__ void __launch_bounds__(SEL_T) sel_count_kernel(const unsigned* __restrict__ keys, int p,
                                                          const SelState* __restrict__ st,
                                                          int* __restrict__ block_counts, int nblocks) {
  const int b = blockIdx.y;
  const int i = blockIdx.x * SEL_T + threadIdx.x;
  const unsigned v = st[b].prefix;
  const unsigned key = i < p ? keys[(size_t)b * p + i] : 0u;
  const int n_above = __syncthreads_count(i < p && key > v);
  const int n_tied = __syncthreads_count(i < p && key == v);
  if (threadIdx.x == 0) {
    block_counts[((size_t)b * 2 + 0) * nblocks + blockIdx.x] = n_above;
    block_counts[((size_t)b * 2 + 1) * nblocks + blockIdx.x] = n_tied;
  }
}

// exclusive scan of one row of block counts (one CTA per row), its total -> totals[row]
__global__ void __launch_bounds__(1024) sel_scan_kernel(int* __restrict__ block_counts, int nblocks,
                                                        int* __restrict__ totals) {
  __shared__ int s_warp[32];
  __shared__ int s_carry;
  int* bc = block_counts + (size_t)blockIdx.x * nblocks;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_carry = 0;
  __syncthreads();
  for (int start = 0; start < nblocks; start += 1024) {
    const int i = start + tid;
    const int v = i < nblocks ? bc[i] : 0;
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
    if (i < nblocks) bc[i] = incl - v;
    __syncthreads();
    if (tid == 1023) s_carry = incl;
    __syncthreads();
  }
  if (tid == 0) totals[blockIdx.x] = s_carry;
}

// rows of this block before this thread's row that satisfy pred
__device__ __forceinline__ int sel_block_prefix(int* s_warp, bool pred) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned bal = __ballot_sync(0xffffffffu, pred);
  if (lane == 0) s_warp[warp] = __popc(bal);
  __syncthreads();
  int prefix = 0;
  for (int w = 0; w < warp; w++) prefix += s_warp[w];
  return prefix + __popc(bal & ((1u << lane) - 1u));
}

// CLASSES: 8-column rows (x, y, w, h, theta, conf, class_conf, class) like the reference's torch.cat((pred[:, :6],
// class_conf, class_pred.float())) (nms.py:51)
template <bool CLASSES>
__global__ void __launch_bounds__(SEL_T) sel_write_kernel(const float* __restrict__ io, int p, int nc,
                                                          const unsigned* __restrict__ keys,
                                                          const SelState* __restrict__ st,
                                                          const int* __restrict__ block_offsets,
                                                          const int* __restrict__ totals, int nblocks,
                                                          float* __restrict__ dets, int cap, int* __restrict__ n_out) {
  __shared__ int s_warp[2][SEL_T / 32];
  const int b = blockIdx.y;
  const int i = blockIdx.x * SEL_T + threadIdx.x;
  const unsigned v = st[b].prefix;
  const int need = st[b].done ? 0 : st[b].k;
  const unsigned key = i < p ? keys[(size_t)b * p + i] : 0u;
  const bool is_above = i < p && key > v, is_tied = i < p && key == v;
  const int above_before = block_offsets[((size_t)b * 2 + 0) * nblocks + blockIdx.x] +
                           sel_block_prefix(s_warp[0], is_above);
  const int tied_before = block_offsets[((size_t)b * 2 + 1) * nblocks + blockIdx.x] +
                          sel_block_prefix(s_warp[1], is_tied);
  if (is_above || (is_tied && tied_before < need)) {
    const float* row = io + ((size_t)b * p + i) * (6 + nc);
    constexpr int DW = CLASSES ? 8 : 6;
    float* o = dets + ((size_t)b * cap + above_before + min(tied_before, need)) * DW;
    o[0] = row[0]; o[1] = row[1]; o[2] = row[2]; o[3] = row[3]; o[4] = row[4]; o[5] = __uint_as_float(key);
    if constexpr (CLASSES) {
      float best; int bi; bool fin;
      class_max(row, nc, &best, &bi, &fin);
      o[6] = best; o[7] = (float)bi;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) n_out[b] = totals[b * 2 + 0] + min(totals[b * 2 + 1], need);
}

}  // namespace ryolo

using namespace ryolo;

extern "C" size_t ryolo_detect_select_workspace_bytes(int batch, int p) {
  if (batch <= 0 || p <= 0) return 256;
  const size_t nblocks = (size_t)(p + SEL_T - 1) / SEL_T;
  return SEL_PASSES * align_up((size_t)batch * SEL_BINS * sizeof(int), 256) +
         align_up((size_t)batch * sizeof(SelState), 256) + align_up((size_t)batch * p * sizeof(unsigned), 256) +
         align_up((size_t)batch * 2 * nblocks * sizeof(int), 256) + align_up((size_t)batch * 2 * sizeof(int), 256) +
         256;
}

template <bool CLASSES>
static int detect_select_impl(const float* io, int batch, int p, int nc, float conf_thres, float min_wh, int limit,
                              float* dets_out, int cap, int32_t* n_out, void* workspace, size_t workspace_bytes,
                              void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(io && dets_out && n_out && workspace && batch > 0 && p > 0 && nc >= 1 && limit > 0 && cap >= limit);
  RYOLO_ARG_CHECK(batch <= 65535);
  RYOLO_ARG_CHECK(conf_thres >= 0.f);   // also rejects NaN; a positive conf's bit pattern orders like its value
  if (workspace_bytes < ryolo_detect_select_workspace_bytes(batch, p)) {
    set_err("ryolo_detect_select: workspace too small");
    return RYOLO_E_WORKSPACE;
  }
  const int nblocks = (p + SEL_T - 1) / SEL_T;
  Carver c(workspace);
  int* hist = c.take<int>((size_t)SEL_PASSES * batch * SEL_BINS);
  SelState* st = c.take<SelState>(batch);
  unsigned* keys = c.take<unsigned>((size_t)batch * p);
  int* counts = c.take<int>((size_t)batch * 2 * nblocks);
  int* totals = c.take<int>((size_t)batch * 2);
  RYOLO_CUDA_TRY(cudaMemsetAsync(hist, 0, (size_t)SEL_PASSES * batch * SEL_BINS * sizeof(int), stream));
  dim3 gh((p + SEL_ROWS_PER_CTA - 1) / SEL_ROWS_PER_CTA, batch);
  sel_key_hist_kernel<<<gh, SEL_T, 0, stream>>>(io, p, nc, conf_thres, min_wh, keys, hist);
  RYOLO_LAUNCH_CHECK();
  sel_radix_kernel<<<batch, 1024, 0, stream>>>(hist, 0, limit, st);
  RYOLO_LAUNCH_CHECK();
  for (int pass = 1; pass < SEL_PASSES; pass++) {
    int* h = hist + (size_t)pass * batch * SEL_BINS;
    sel_digit_hist_kernel<<<gh, SEL_T, 0, stream>>>(keys, p, pass, st, h);
    RYOLO_LAUNCH_CHECK();
    sel_radix_kernel<<<batch, 1024, 0, stream>>>(h, pass, limit, st);
    RYOLO_LAUNCH_CHECK();
  }
  dim3 gc(nblocks, batch);
  sel_count_kernel<<<gc, SEL_T, 0, stream>>>(keys, p, st, counts, nblocks);
  RYOLO_LAUNCH_CHECK();
  sel_scan_kernel<<<batch * 2, 1024, 0, stream>>>(counts, nblocks, totals);
  RYOLO_LAUNCH_CHECK();
  sel_write_kernel<CLASSES><<<gc, SEL_T, 0, stream>>>(io, p, nc, keys, st, counts, totals, nblocks, dets_out, cap,
                                                      n_out);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_detect_select(const float* io, int batch, int p, int nc, float conf_thres, float min_wh, int limit,
                                   float* dets_out, int cap, int32_t* n_out, void* workspace, size_t workspace_bytes,
                                   void* stream_) {
  return detect_select_impl<false>(io, batch, p, nc, conf_thres, min_wh, limit, dets_out, cap, n_out, workspace,
                                   workspace_bytes, stream_);
}

extern "C" int ryolo_detect_select_classes(const float* io, int batch, int p, int nc, float conf_thres, float min_wh,
                                           int limit, float* dets_out, int cap, int32_t* n_out, void* workspace,
                                           size_t workspace_bytes, void* stream_) {
  RYOLO_ARG_CHECK(nc <= (1 << 24));   // class ids in [0, 2^24): exact in fp32 and a valid class of the batched NMS
  return detect_select_impl<true>(io, batch, p, nc, conf_thres, min_wh, limit, dets_out, cap, n_out, workspace,
                                  workspace_bytes, stream_);
}
