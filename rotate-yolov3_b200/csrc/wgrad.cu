// Weight gradient of the conv blocks as an sm_90a wgmma GEMM whose K dimension is the PIXEL index:
//     dW[tap][co][ci] = sum_p dz[p, co] * x[p + off_tap, ci]          (flat padded-NHWC pixel index p, zero halos)
// the adjoint of the forward implicit GEMM in conv.cu (reference: autograd through nn.Conv2d, train.py:278-282).
// Both operands are read in their natural padded-NHWC layout -- 64 channels (128 B) contiguous per pixel row -- which
// makes them "MN-major" wgmma operands: TMA boxes [64 channels x 64 pixels] land in shared memory as 128B-swizzled
// rows = K, and the descriptors / transpose flags say so.  No transposed copies of activations or gradients.
// The tap shift is again only a row-coordinate offset of the x box.  Split-K over CTAs, fp32 register accumulation
// (warp group 1 / 2: filters [0, 64) / [64, 128) of the tile).  With one split the CTA adds its accumulators to dW.  With
// several, every CTA stores them to scratch and wgrad_splitk_reduce_kernel, launched right after on the same stream,
// adds the splits of every dW entry in split order -- one thread per entry over the whole grid, a fixed order, so the
// weight gradient is the same every run (float atomics would add in arrival order).
// Stride-2 layers pass the zero-inserted dz at input resolution.
//
// THIN tiles (cout_pad == 64): the tile has only filters [0, 64), so the producer loads one dz box and the two MMA warp
// groups share those 64 filters and split the stage's (tap, 64-channel box) pairs between them, one m64n64k16 per pair
// (pair q belongs to warp group 1 + q % 2).  Every dW entry keeps its own accumulator chain over the same k-steps; only
// the N width of the instruction that updates it changes.
//
// SEG variant (ryolo_px_wgrad, the parity-precision path): the tensor pipe's fp32 accumulator does not round to nearest,
// and over the thousands of updates of one pixel range its error is biased towards zero.  As in conv_parity.cu, the MMA
// warp groups then restart the accumulator every WG_SEG k-steps (32 MMA updates) and fold it into a second register set
// with round-to-nearest fp32 adds; the split-K reduction and the store are unchanged.
#include "common.cuh"
#include "sm90.cuh"

namespace ryolo {

constexpr int WG_BM = 128;   // filters per tile (two m64 warp groups)
constexpr int WG_BK = 64;    // pixels per k-step
constexpr int WG_THREADS = 384;   // warp group 0: TMA; warp groups 1-2: MMA + store
constexpr int WG_SEG = 8;         // SEG variant: k-steps per accumulator segment
constexpr int WG_REDUCE_THREADS = 256;
constexpr int WG_REDUCE_UNROLL = 16;  // partial loads in flight per thread of the reduce kernel

struct WgradParams {
  int np, wp, taps;   // taps: 1, 4 (2x2, offsets -1..0) or 9 (3x3, offsets -1..1)
  int tap_groups;     // taps / TG: a CTA accumulates the TG taps of one kernel row (they share the dz tile)
  int cout_pad, cin_pad;
  int m_tiles, n_tiles, ksplit, ksteps_total, ksteps_per_split;
  float* dw;   // [taps][cout_pad][cin_pad] fp32, the tile's sum is added to it
  float* partials;          // ksplit > 1: [split][tile][WgradFrag::V][256 MMA threads]
};

// TG = taps per CTA.  For thin layers (cin <= 128) the per-tap GEMM is bound by the L2 -> SM operand stream; the TG taps
// of one kernel row share the dz (A) tile, so a CTA that keeps TG accumulators streams A once per row instead of once per
// tap.  The accumulators live in registers: TG * BN / 2 per thread, at most 128 (THIN: half of that, rounded up to 32).
template <int BN, int TG, bool THIN>
struct WgradCfg {
  static constexpr int kABytes = (THIN ? 64 : WG_BM) * WG_BK * 2;   // one or two [64 ch x 64 px] boxes
  static constexpr int kBBytes = BN * WG_BK * 2;                    // BN/64 boxes per tap
  static constexpr int kStageBytes = kABytes + TG * kBBytes;
  // as many stages as 192 KB holds (one CTA per SM), 4 to 8: the memory-bound launches have small stages (16-32 KB,
  // and the zero-filled part of a narrow box is not fetched), and 4 of them keep too few bytes in flight per SM to
  // cover the HBM latency
  static constexpr int kStages = 196608 / kStageBytes > 8 ? 8 : (196608 / kStageBytes < 4 ? 4 : 196608 / kStageBytes);
  static constexpr int kSmem = kStages * kStageBytes + 2 * kStages * 8 + 1024;
};

// The accumulators of one MMA thread and the dW entries they hold.  MMA thread me (0..255 over warp groups 1-2) keeps
// R arrays of W fp32 slots, V = R * W in all, flat slot v = W * r + e.  Entry e of an m64n{2W} fragment is row
// 16 warp + lane / 4 + 8 ((e / 2) % 2), column 64 (e / 32) + 8 ((e % 32) / 4) + 2 (lane % 4) + e % 2.
//   full tile: array r = tap j of the group, the m64n{BN} fragment of this warp group's 64 filters;
//   THIN:      array r = pair q = 2 r + (me / 128) of the stage's TG * BN / 64 (tap, channel box) pairs, m64n64.
// The direct store, the partials and the reduce kernel all go through coord(), so they agree on the mapping.
template <int BN, int TG, bool THIN>
struct WgradFrag {
  static constexpr int NS = BN / 64;                 // 64-channel boxes per tap
  static constexpr int PAIRS = TG * NS;              // (tap, box) pairs of a stage
  static constexpr int R = THIN ? (PAIRS + 1) / 2 : TG;
  static constexpr int W = THIN ? 32 : BN / 2;
  static constexpr int V = R * W;
  static constexpr int kMmaWarpGroups = THIN && PAIRS == 1 ? 1 : 2;

  // does array r of warp group `half` hold any entries (THIN with an odd pair count: the last one of warp group 2 not)
  __device__ static bool owns(int half, int r) { return !THIN || 2 * r + half < PAIRS; }

  // slot v of MMA thread me of tile (tap group tg, channel tile nt, filter tile mt) -> dW[tap][co][ci]; false when the
  // slot holds no entry of dW (an unused THIN array, a padding filter or channel beyond cout_pad / cin_pad)
  __device__ static bool coord(const WgradParams& p, int tg, int nt, int mt, int me, int v, int& tap, int& co, int& ci) {
    const int half = me >> 7, warp = (me >> 5) & 3, lane = me & 31;
    const int r = v / W, e = v % W;
    int j, n;
    if constexpr (THIN) {
      const int q = 2 * r + half;
      if (q >= PAIRS) return false;
      j = q / NS;
      n = q % NS;
    } else {
      j = r;
      n = e / 32;
    }
    const int f = e % 32;
    tap = TG == 1 ? tg : tg * TG + j;
    co = mt * WG_BM + (THIN ? 0 : half * 64) + warp * 16 + (lane >> 2) + 8 * ((f >> 1) & 1);
    ci = nt * BN + n * 64 + 8 * (f >> 2) + 2 * (lane & 3) + (f & 1);
    return co < p.cout_pad && ci < p.cin_pad;
  }
};

// blockIdx.x of the GEMM = tile + split * tiles, tile = tap group + tap_groups * (nt + n_tiles * mt), tap group fastest:
// the CTAs that are resident together cover ALL taps and channel tiles of a few pixel ranges, so dz / x stream from HBM
// once and the other reads hit L2 (with the split index fastest every tap pass re-streamed both tensors from HBM: 9x the
// traffic on 3x3 layers)
__device__ __forceinline__ void wgrad_tile_decode(const WgradParams& p, int t, int& tg, int& nt, int& mt) {
  tg = t % p.tap_groups; t /= p.tap_groups;
  nt = t % p.n_tiles; t /= p.n_tiles;
  mt = t;
}

template <int BN, int TG, bool SEG, bool THIN>
__global__ void __launch_bounds__(WG_THREADS, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap map_dz, const __grid_constant__ CUtensorMap map_x, const WgradParams p) {
  using C = WgradCfg<BN, TG, THIN>;
  using F = WgradFrag<BN, TG, THIN>;
  constexpr int kABytes = C::kABytes, kBBytes = C::kBBytes, kStageBytes = C::kStageBytes, WG_STAGES = C::kStages;
  constexpr int NS = F::NS, R = F::R, W = F::W;
  static_assert(TG * BN <= (SEG ? 128 : 256), "accumulators (and the SEG sums) must fit the registers");
  extern __shared__ unsigned char smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + WG_STAGES * kStageBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (WG_STAGES + s); };

  const int wg = threadIdx.x >> 7;
  const int tiles = p.tap_groups * p.n_tiles * p.m_tiles;
  const int split = blockIdx.x / tiles;
  int tg, nt, mt;
  wgrad_tile_decode(p, blockIdx.x - split * tiles, tg, nt, mt);
  const int k_begin = split * p.ksteps_per_split;
  const int k_end = min(p.ksteps_total, k_begin + p.ksteps_per_split);
  const int k_iters = k_end - k_begin;
  // pixel offset of tap j of this group: 3x3: (dy, dx) = (tg - 1, j - 1); 2x2: (tg - 1, j - 1); 1x1: 0.  With TG == 1
  // the group index IS the tap index.
  auto tap_off = [&](int j) {
    const int tap = TG == 1 ? tg : tg * TG + j;
    if (p.taps == 9) return (tap / 3 - 1) * p.wp + (tap % 3 - 1);
    if (p.taps == 4) return (tap / 2 - 1) * p.wp + (tap % 2 - 1);
    return 0;
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < WG_STAGES; s++) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 4 * F::kMmaWarpGroups);   // one arrive per MMA warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (k_iters <= 0) return;

  if (wg == 0) {
    regs_dealloc<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kk = 0; kk < k_iters; kk++) {
        const int prow = (k_begin + kk) * WG_BK;
        mbar_wait(empty_bar(stage), phase ^ 1);
        const uint32_t sa = smem_base + stage * kStageBytes;
        mbar_expect_tx(full_bar(stage), kStageBytes);
#pragma unroll
        for (int g = 0; g < kABytes / 8192; g++) tma_load_2d(sa + g * 8192, &map_dz, full_bar(stage), mt * WG_BM + g * 64, prow);
#pragma unroll
        for (int j = 0; j < TG; j++) {
          const int off = tap_off(j);
#pragma unroll
          for (int g = 0; g < NS; g++)
            tma_load_2d(sa + kABytes + j * kBBytes + g * 8192, &map_x, full_bar(stage), nt * BN + g * 64, prow + off);
        }
        if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }
  if (wg > F::kMmaWarpGroups) return;   // THIN with one pair: warp group 2 has nothing to multiply

  regs_alloc<232>();
  const int half = wg - 1;
  const int me = threadIdx.x - 128;   // 0..255 over the two MMA warp groups
  const int lane = threadIdx.x & 31;
  float acc[R][W];   // see WgradFrag
  float sum[SEG ? R : 1][SEG ? W : 1];   // SEG: round-to-nearest running sum of the closed segments
  if constexpr (SEG) {
#pragma unroll
    for (int r = 0; r < R; r++)
#pragma unroll
      for (int v = 0; v < W; v++) sum[r][v] = 0.f;
  }
  int stage = 0, prev = -1;
  uint32_t phase = 0;
  for (int kk = 0; kk < k_iters; kk++) {
    mbar_wait(full_bar(stage), phase);
    const uint32_t sa = smem_base + stage * kStageBytes;
    const bool seg_start = SEG ? kk % WG_SEG == 0 : kk == 0;
    wg_fence();
#pragma unroll
    for (int k = 0; k < WG_BK / 16; k++) {
      // 16 pixels = two 8-row groups = 2048 bytes along K; the tap's BN / 64 channel boxes are 8192 bytes (LBO) apart
      const uint32_t acc_in = (!seg_start || k > 0) ? 1u : 0u;
      if constexpr (THIN) {
        // the tile's 64 filters are box 0; pair q = (tap q / NS, channel box q % NS)
        const uint64_t adesc = make_smem_desc_mn(sa + k * 2048, 8192);
#pragma unroll
        for (int r = 0; r < R; r++) {
          if (!F::owns(half, r)) continue;
          const int q = 2 * r + half;
          wgmma_bf16<64, 1, 1>(acc[r], adesc,
                               make_smem_desc_mn(sa + kABytes + (q / NS) * kBBytes + (q % NS) * 8192 + k * 2048, 8192), acc_in);
        }
      } else {
        // this warp group's 64 filters are the box at half * 8192
        const uint64_t adesc = make_smem_desc_mn(sa + half * 8192 + k * 2048, 8192);
#pragma unroll
        for (int j = 0; j < TG; j++)
          wgmma_bf16<BN, 1, 1>(acc[j], adesc, make_smem_desc_mn(sa + kABytes + j * kBBytes + k * 2048, 8192), acc_in);
      }
    }
    wg_commit();
    bool seg_end = false;
    if constexpr (SEG) {
      seg_end = kk % WG_SEG == WG_SEG - 1 || kk == k_iters - 1;
      if (seg_end) {
        // close the segment: fold it into the round-to-nearest running sum
        wg_wait<0>();
#pragma unroll
        for (int r = 0; r < R; r++) {
          wg_fence_regs(acc[r]);
#pragma unroll
          for (int v = 0; v < W; v++) sum[r][v] = __fadd_rn(sum[r][v], acc[r][v]);
        }
        if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
        if (lane == 0) mbar_arrive(empty_bar(stage));
        prev = -1;
      }
    }
    if (!seg_end) {
      wg_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
      prev = stage;
    }
    if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
  }
  wg_wait<0>();
#pragma unroll
  for (int r = 0; r < R; r++) {
    wg_fence_regs(acc[r]);
    if constexpr (SEG) {
#pragma unroll
      for (int v = 0; v < W; v++) acc[r][v] = sum[r][v];
    }
  }

  if (p.ksplit > 1) {
    // split-K: store the fragment; wgrad_splitk_reduce_kernel adds the splits in split order
    float* mine = p.partials + (size_t)blockIdx.x * F::V * 256 + me;
#pragma unroll
    for (int r = 0; r < R; r++) {
      if (!F::owns(half, r)) continue;
#pragma unroll
      for (int v = 0; v < W; v++) __stcg(mine + (size_t)(r * W + v) * 256, acc[r][v]);
    }
    return;
  }

  // one split: this CTA is the only writer of its dW entries in this launch; slots 2i, 2i + 1 are adjacent columns
#pragma unroll
  for (int v = 0; v < F::V; v += 2) {
    int tap, co, ci;
    if (!F::coord(p, tg, nt, mt, me, v, tap, co, ci)) continue;
    float2* dst = reinterpret_cast<float2*>(p.dw + ((size_t)tap * p.cout_pad + co) * p.cin_pad + ci);
    float2 d = *dst;
    d.x += acc[v / W][v % W];
    d.y += acc[v / W][v % W + 1];
    *dst = d;
  }
}

// Split-K reduction of conv_wgrad_kernel: one thread per (tile, slot, MMA thread), the partials' own order, so a warp
// reads 128 contiguous bytes per split.  Starts from 0, adds splits 0, 1, ..., ksplit - 1 (loads issued ahead, adds in
// order), then dW += sum.  The partials were just written and are still in L2.
template <int BN, int TG, bool THIN>
__global__ void __launch_bounds__(WG_REDUCE_THREADS) wgrad_splitk_reduce_kernel(const WgradParams p) {
  using F = WgradFrag<BN, TG, THIN>;
  const int tiles = p.tap_groups * p.n_tiles * p.m_tiles;
  const size_t per_split = (size_t)tiles * F::V * 256;
  const size_t e = (size_t)blockIdx.x * WG_REDUCE_THREADS + threadIdx.x;
  if (e >= per_split) return;
  const int me = (int)(e % 256);
  const int slot = (int)(e / 256);
  int tg, nt, mt, tap, co, ci;
  wgrad_tile_decode(p, slot / F::V, tg, nt, mt);
  if (!F::coord(p, tg, nt, mt, me, slot % F::V, tap, co, ci)) return;
  float* dst = p.dw + ((size_t)tap * p.cout_pad + co) * p.cin_pad + ci;
  const float d = *dst;   // independent of the partials: in flight with them
  const float* src = p.partials + e;
  float s = 0.f;
  // predicated groups of WG_REDUCE_UNROLL loads, so a short split count (2-16) is one round trip, not ksplit of them
  for (int k = 0; k < p.ksplit; k += WG_REDUCE_UNROLL) {
    float x[WG_REDUCE_UNROLL];
#pragma unroll
    for (int u = 0; u < WG_REDUCE_UNROLL; u++) x[u] = k + u < p.ksplit ? __ldcg(src + (size_t)(k + u) * per_split) : 0.f;
#pragma unroll
    for (int u = 0; u < WG_REDUCE_UNROLL; u++)
      if (k + u < p.ksplit) s += x[u];
  }
  *dst = d + s;
}

template <int BN, int TG, bool SEG, bool THIN>
static int launch_wgrad_tile(const CUtensorMap& mdz, const CUtensorMap& mx, WgradParams p, cudaStream_t stream) {
  using C = WgradCfg<BN, TG, THIN>;
  using F = WgradFrag<BN, TG, THIN>;
  const int tiles = p.tap_groups * p.m_tiles * p.n_tiles;
  p.partials = nullptr;
  if (p.ksplit > 1) {
    p.partials = static_cast<float*>(
        stream_scratch(stream, SCRATCH_WGRAD, (size_t)p.ksplit * tiles * F::V * 256 * sizeof(float)));
    if (!p.partials) return RYOLO_E_CUDA;
  }
  RYOLO_SMEM_OPT_IN((conv_wgrad_kernel<BN, TG, SEG, THIN>), C::kSmem);
  conv_wgrad_kernel<BN, TG, SEG, THIN><<<tiles * p.ksplit, WG_THREADS, C::kSmem, stream>>>(mdz, mx, p);
  RYOLO_LAUNCH_CHECK();
  if (p.ksplit > 1) {
    const size_t threads = (size_t)tiles * F::V * 256;
    wgrad_splitk_reduce_kernel<BN, TG, THIN>
        <<<(unsigned)((threads + WG_REDUCE_THREADS - 1) / WG_REDUCE_THREADS), WG_REDUCE_THREADS, 0, stream>>>(p);
    RYOLO_LAUNCH_CHECK();
  }
  return RYOLO_OK;
}

// THIN for a 64-filter layer (one filter tile of 64): half the MMAs and one dz box per stage
template <int BN, int TG, bool SEG>
static int launch_wgrad(const CUtensorMap& mdz, const CUtensorMap& mx, const WgradParams& p, cudaStream_t stream) {
  if (p.cout_pad == 64) return launch_wgrad_tile<BN, TG, SEG, true>(mdz, mx, p, stream);
  return launch_wgrad_tile<BN, TG, SEG, false>(mdz, mx, p, stream);
}

static int wgrad(const void* dz, int dz_cstride, int cout_pad, const void* x, int x_cstride, int cin_pad, int batch,
                 int in_h, int in_w, int ksize, float* dw, bool seg, cudaStream_t stream) {
  RYOLO_ARG_CHECK(dz && x && dw && batch > 0 && in_h > 0 && in_w > 0);
  RYOLO_ARG_CHECK(ksize == 1 || ksize == 3 || ksize == 2);
  RYOLO_ARG_CHECK(cout_pad > 0 && cout_pad % 64 == 0 && cin_pad > 0 && cin_pad % 64 == 0);
  // strides narrower than the padded tile are fine: TMA zero-fills the box beyond the inner extent
  RYOLO_ARG_CHECK(dz_cstride > 0 && dz_cstride % 8 == 0 && x_cstride > 0 && x_cstride % 8 == 0);
  WgradParams p;
  const long long np = (long long)batch * (in_h + 2) * (in_w + 2);
  RYOLO_ARG_CHECK(np < (1ll << 31) - 4096);
  p.np = (int)np;
  p.wp = in_w + 2;
  p.taps = ksize * ksize;
  p.cout_pad = cout_pad;
  p.cin_pad = cin_pad;
  // 64, 128 or 256 channels per tile; SEG keeps a second register set, so TG * bn <= 128 there
  const int bn = seg ? (cin_pad % 128 == 0 ? 128 : 64) : (cin_pad >= 192 ? 256 : cin_pad);
  p.m_tiles = (cout_pad + WG_BM - 1) / WG_BM;
  p.n_tiles = (cin_pad + bn - 1) / bn;
  p.ksteps_total = (p.np + WG_BK - 1) / WG_BK;
  const int num_sms = gemm_sm_count();
  // taps per CTA: the kernel row (3 or 2 taps) when the accumulators fit the registers (TG * bn <= 256) and the layer
  // is thin enough to be operand-stream bound
  int tg = 1;
  if (bn <= 128) tg = p.taps == 9 ? 3 : (p.taps == 4 ? 2 : 1);
  if (tg * bn > (seg ? 128 : 256)) tg = 1;
  p.tap_groups = p.taps / tg;
  const int tiles = p.tap_groups * p.m_tiles * p.n_tiles;
  // split-K: every (tile, split) CTA ends with tile-size fp32 stores and cannot overlap them with its MMAs, so use the
  // FEWEST waves that still fill the SMs (>= 90 % of the last wave), not a fixed multiple
  int ksplit = 1;
  {
    double best_eff = 0.0;
    for (int waves = 1; waves <= 4; waves++) {
      int ks = waves * num_sms / tiles;
      if (ks < 1) ks = 1;
      const int ctas = tiles * ks;
      const double eff = (double)ctas / ((double)((ctas + num_sms - 1) / num_sms) * num_sms);
      if (eff > best_eff + 1e-9) { best_eff = eff; ksplit = ks; }
      if (eff >= 0.9) break;
    }
  }
  const int max_split = (p.ksteps_total + 15) / 16;                // at least 16 k-steps per CTA
  if (ksplit > max_split) ksplit = max_split;
  if (ksplit < 1) ksplit = 1;
  p.ksteps_per_split = (p.ksteps_total + ksplit - 1) / ksplit;
  p.ksplit = (p.ksteps_total + p.ksteps_per_split - 1) / p.ksteps_per_split;
  p.dw = dw;
  p.partials = nullptr;
  CUtensorMap mdz, mx;
  // inner extent = channel stride of the buffer (reads beyond cout_pad/cin_pad are masked at the store)
  int st = encode_map_2d(&mdz, dz, (uint64_t)dz_cstride, (uint64_t)p.np, (uint64_t)dz_cstride * 2, 64, WG_BK);
  if (st != RYOLO_OK) return st;
  st = encode_map_2d(&mx, x, (uint64_t)x_cstride, (uint64_t)p.np, (uint64_t)x_cstride * 2, 64, WG_BK);
  if (st != RYOLO_OK) return st;
  if (seg) {
    if (bn == 128) return launch_wgrad<128, 1, true>(mdz, mx, p, stream);
    if (tg == 2) return launch_wgrad<64, 2, true>(mdz, mx, p, stream);
    return launch_wgrad<64, 1, true>(mdz, mx, p, stream);
  }
  if (bn == 256) return launch_wgrad<256, 1, false>(mdz, mx, p, stream);
  if (bn == 128) {
    if (tg == 2) return launch_wgrad<128, 2, false>(mdz, mx, p, stream);
    return launch_wgrad<128, 1, false>(mdz, mx, p, stream);
  }
  if (tg == 3) return launch_wgrad<64, 3, false>(mdz, mx, p, stream);
  if (tg == 2) return launch_wgrad<64, 2, false>(mdz, mx, p, stream);
  return launch_wgrad<64, 1, false>(mdz, mx, p, stream);
}

}  // namespace ryolo

using namespace ryolo;

extern "C" int ryolo_conv_wgrad(const void* dz, int dz_cstride, int cout_pad, const void* x, int x_cstride, int cin_pad,
                                int batch, int in_h, int in_w, int ksize, float* dw, void* stream_) {
  return wgrad(dz, dz_cstride, cout_pad, x, x_cstride, cin_pad, batch, in_h, in_w, ksize, dw, false,
               static_cast<cudaStream_t>(stream_));
}

extern "C" int ryolo_px_wgrad(const void* dz, int dz_cstride, int cout_pad, const void* x, int x_cstride, int cin_pad,
                              int batch, int in_h, int in_w, int ksize, float* dw, void* stream_) {
  return wgrad(dz, dz_cstride, cout_pad, x, x_cstride, cin_pad, batch, in_h, in_w, ksize, dw, true,
               static_cast<cudaStream_t>(stream_));
}
