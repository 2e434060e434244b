// Weight gradient of the conv blocks as an sm_90a wgmma GEMM whose K dimension is the PIXEL index:
//     dW[tap][co][ci] = sum_p dz[p, co] * x[p + off_tap, ci]          (flat padded-NHWC pixel index p, zero halos)
// the adjoint of the forward implicit GEMM in conv.cu (reference: autograd through nn.Conv2d, train.py:278-282).
// Both operands are read in their natural padded-NHWC layout -- 64 channels (128 B) contiguous per pixel row -- which
// makes them "MN-major" wgmma operands: TMA boxes [64 channels x 64 pixels] land in shared memory as 128B-swizzled
// rows = K, and the descriptors / transpose flags say so.  No transposed copies of activations or gradients.
// The tap shift is again only a row-coordinate offset of the x box.  Split-K over CTAs, fp32 register accumulation
// (warp group 1 / 2: filters [0, 64) / [64, 128) of the tile).  With several splits every CTA stores its accumulators
// to scratch and the LAST split of a tile to finish (ticket per tile) adds the splits in split order and adds the sum to
// dW -- a fixed order, so the weight gradient is the same every run (float atomics would add in arrival order).
// Stride-2 layers pass the zero-inserted dz at input resolution.
//
// SEG variant (ryolo_px_wgrad, the parity-precision path): the tensor pipe's fp32 accumulator does not round to nearest,
// and over the thousands of updates of one pixel range its error is biased towards zero.  As in conv_parity.cu, the MMA
// warp groups then restart the accumulator every WG_SEG k-steps (32 MMA updates) and fold it into a second register set
// with round-to-nearest fp32 adds; the split-K reduction and the store are unchanged.
#include <stdlib.h>

#include "common.cuh"
#include "sm90.cuh"

namespace ryolo {

constexpr int WG_BM = 128;   // filters per tile (two m64 warp groups)
constexpr int WG_BK = 64;    // pixels per k-step
constexpr int WG_THREADS = 384;   // warp group 0: TMA; warp groups 1-2: MMA + reduction
constexpr int WG_SEG = 8;         // SEG variant: k-steps per accumulator segment

struct WgradParams {
  int np, wp, taps;   // taps: 1, 4 (2x2, offsets -1..0) or 9 (3x3, offsets -1..1)
  int tap_groups;     // taps / TG: a CTA accumulates the TG taps of one kernel row (they share the dz tile)
  int cout_pad, cin_pad;
  int m_tiles, n_tiles, ksplit, ksteps_total, ksteps_per_split;
  float* dw;   // [taps][cout_pad][cin_pad] fp32, the tile's sum is added to it
  float* partials;          // ksplit > 1: [CTA][TG * BN / 2][256 MMA threads]
  unsigned int* tickets;    // ksplit > 1: [tap_groups * n_tiles * m_tiles], zero at launch
};

// TG = taps per CTA.  For thin layers (cin <= 128) the per-tap GEMM is bound by the L2 -> SM operand stream; the TG taps
// of one kernel row share the dz (A) tile, so a CTA that keeps TG accumulators streams A once per row instead of once per
// tap.  The accumulators live in registers: TG * BN / 2 per thread, at most 128.
template <int BN, int TG>
struct WgradCfg {
  static constexpr int kABytes = WG_BM * WG_BK * 2;   // two [64 ch x 64 px] boxes
  static constexpr int kBBytes = BN * WG_BK * 2;      // BN/64 boxes per tap
  static constexpr int kStageBytes = kABytes + TG * kBBytes;
  static constexpr int kStages = kStageBytes > 49152 ? 3 : 4;
  static constexpr int kSmem = kStages * kStageBytes + 2 * kStages * 8 + 1024;
};

template <int BN, int TG, bool SEG>
__global__ void __launch_bounds__(WG_THREADS, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap map_dz, const __grid_constant__ CUtensorMap map_x, const WgradParams p) {
  using C = WgradCfg<BN, TG>;
  constexpr int kABytes = C::kABytes, kBBytes = C::kBBytes, kStageBytes = C::kStageBytes, WG_STAGES = C::kStages;
  constexpr int NS = BN / 64;
  static_assert(TG * BN <= (SEG ? 128 : 256), "accumulators (and the SEG sums) must fit the registers");
  extern __shared__ unsigned char smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + WG_STAGES * kStageBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (WG_STAGES + s); };

  const int wg = threadIdx.x >> 7;
  // tile decode: blockIdx.x -> (tap group, nt, mt, split), tap group fastest: the CTAs that are resident together cover
  // ALL taps and channel tiles of a few pixel ranges, so dz / x stream from HBM once and the other reads hit L2 (with the
  // split index fastest every tap pass re-streamed both tensors from HBM: 9x the traffic on 3x3 layers)
  int t = blockIdx.x;
  const int tg = t % p.tap_groups; t /= p.tap_groups;
  const int nt = t % p.n_tiles; t /= p.n_tiles;
  const int mt = t % p.m_tiles; t /= p.m_tiles;
  const int split = t;
  const int k_begin = split * p.ksteps_per_split;
  const int k_end = min(p.ksteps_total, k_begin + p.ksteps_per_split);
  const int k_iters = k_end - k_begin;
  // pixel offset of tap j of this group: 3x3: (dy, dx) = (tg - 1, j - 1); 2x2: (tg - 1, j - 1); 1x1: 0.  With TG == 1
  // the group index IS the tap index.
  auto tap_of = [&](int j) { return TG == 1 ? tg : tg * TG + j; };
  auto tap_off = [&](int j) {
    const int tap = tap_of(j);
    if (p.taps == 9) return (tap / 3 - 1) * p.wp + (tap % 3 - 1);
    if (p.taps == 4) return (tap / 2 - 1) * p.wp + (tap % 2 - 1);
    return 0;
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < WG_STAGES; s++) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);   // one arrive per MMA warp
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
        for (int g = 0; g < WG_BM / 64; g++) tma_load_2d(sa + g * 8192, &map_dz, full_bar(stage), mt * WG_BM + g * 64, prow);
#pragma unroll
        for (int j = 0; j < TG; j++) {
          const int off = tap_off(j);
#pragma unroll
          for (int g = 0; g < BN / 64; g++)
            tma_load_2d(sa + kABytes + j * kBBytes + g * 8192, &map_x, full_bar(stage), nt * BN + g * 64, prow + off);
        }
        if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  regs_alloc<232>();
  const int half = wg - 1;
  const int tid = threadIdx.x & 127, warp = tid >> 5, lane = tid & 31;
  float acc[TG][BN / 2];   // m64n{BN} fragment per tap: [32 n + v] is entry v of the 64-channel sub-tile n
  float sum[SEG ? TG : 1][SEG ? BN / 2 : 1];   // SEG: round-to-nearest running sum of the closed segments
  if constexpr (SEG) {
#pragma unroll
    for (int j = 0; j < TG; j++)
#pragma unroll
      for (int v = 0; v < BN / 2; v++) sum[j][v] = 0.f;
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
      // 16 pixels = two 8-row groups = 2048 bytes along K; this warp group's 64 filters are the box at half * 8192
      const uint64_t adesc = make_smem_desc_mn(sa + half * 8192 + k * 2048, 8192);
#pragma unroll
      for (int j = 0; j < TG; j++)   // the tap's BN / 64 channel boxes are 8192 bytes (LBO) apart
        wgmma_bf16<BN, 1, 1>(acc[j], adesc, make_smem_desc_mn(sa + kABytes + j * kBBytes + k * 2048, 8192),
                             (!seg_start || k > 0) ? 1u : 0u);
    }
    wg_commit();
    bool seg_end = false;
    if constexpr (SEG) {
      seg_end = kk % WG_SEG == WG_SEG - 1 || kk == k_iters - 1;
      if (seg_end) {
        // close the segment: fold it into the round-to-nearest running sum
        wg_wait<0>();
#pragma unroll
        for (int j = 0; j < TG; j++) {
          wg_fence_regs(acc[j]);
#pragma unroll
          for (int v = 0; v < BN / 2; v++) sum[j][v] = __fadd_rn(sum[j][v], acc[j][v]);
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
  for (int j = 0; j < TG; j++) {
    wg_fence_regs(acc[j]);
    if constexpr (SEG) {
#pragma unroll
      for (int v = 0; v < BN / 2; v++) acc[j][v] = sum[j][v];
    }
  }

  if (p.ksplit > 1) {
    // split-K in a fixed order: store my fragment, take a ticket; the last split of the tile adds splits 0, 1, ...
    constexpr int V = TG * BN / 2;
    const int me = threadIdx.x - 128;                    // 0..255 over the two MMA warp groups
    const int tiles = p.tap_groups * p.n_tiles * p.m_tiles;
    const int tile = blockIdx.x - split * tiles;
    float* mine = p.partials + (size_t)blockIdx.x * V * 256 + me;
#pragma unroll
    for (int j = 0; j < TG; j++)
#pragma unroll
      for (int v = 0; v < BN / 2; v++) __stcg(mine + (size_t)(j * BN / 2 + v) * 256, acc[j][v]);
    __shared__ int s_last;
    __threadfence();
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (me == 0) s_last = atomicAdd(p.tickets + tile, 1u) == (unsigned)(p.ksplit - 1);
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (!s_last) return;
    __threadfence();
#pragma unroll
    for (int j = 0; j < TG; j++)
#pragma unroll
      for (int v = 0; v < BN / 2; v++) acc[j][v] = 0.f;
    for (int s = 0; s < p.ksplit; s++) {
      const float* src = p.partials + (size_t)(s * tiles + tile) * V * 256 + me;
#pragma unroll
      for (int j = 0; j < TG; j++)
#pragma unroll
        for (int v = 0; v < BN / 2; v++) acc[j][v] += __ldcg(src + (size_t)(j * BN / 2 + v) * 256);
    }
  }

  // rows co0, co0 + 8; columns 8 c + 2 (lane % 4) + {0, 1} of every 64-channel sub-tile
  const int co0 = mt * WG_BM + half * 64 + warp * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < TG; j++) {
#pragma unroll
    for (int i = 0; i < 2; i++) {
      const int co = co0 + 8 * i;
      if (co >= p.cout_pad) continue;
      float* drow = p.dw + ((size_t)tap_of(j) * p.cout_pad + co) * p.cin_pad;
#pragma unroll
      for (int n = 0; n < NS; n++) {
        if (nt * BN + n * 64 >= p.cin_pad) continue;   // cin_pad is a multiple of 64: whole sub-tiles are in or out
#pragma unroll
        for (int c = 0; c < 8; c++) {
          const int ci = nt * BN + n * 64 + 8 * c + 2 * (lane & 3);
          // the only writer of these dW entries in this launch
          float2 d = *reinterpret_cast<float2*>(drow + ci);
          d.x += acc[j][32 * n + 4 * c + 2 * i];
          d.y += acc[j][32 * n + 4 * c + 2 * i + 1];
          *reinterpret_cast<float2*>(drow + ci) = d;
        }
      }
    }
  }
}

template <int BN, int TG, bool SEG>
static int launch_wgrad(const CUtensorMap& mdz, const CUtensorMap& mx, const WgradParams& p, cudaStream_t stream) {
  using C = WgradCfg<BN, TG>;
  RYOLO_SMEM_OPT_IN((conv_wgrad_kernel<BN, TG, SEG>), C::kSmem);
  const int grid = p.tap_groups * p.m_tiles * p.n_tiles * p.ksplit;
  conv_wgrad_kernel<BN, TG, SEG><<<grid, WG_THREADS, C::kSmem, stream>>>(mdz, mx, p);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
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
  // is thin enough to be operand-stream bound; RYOLO_WGRAD_TG=1 forces one tap per CTA (measurement knob)
  static int force_tg = -1;
  if (force_tg < 0) {
    const char* e = getenv("RYOLO_WGRAD_TG");
    force_tg = e ? atoi(e) : 0;
  }
  int tg = 1;
  if (bn <= 128 && force_tg != 1) tg = p.taps == 9 ? 3 : (p.taps == 4 ? 2 : 1);
  if (tg * bn > (seg ? 128 : 256)) tg = 1;
  p.tap_groups = p.taps / tg;
  const int tiles = p.tap_groups * p.m_tiles * p.n_tiles;
  // split-K: every (tile, split) CTA ends with tile-size fp32 reductions into dW and cannot overlap them with its
  // MMAs, so use the FEWEST waves that still fill the SMs (>= 90 % of the last wave), not a fixed multiple
  static int force_waves = -1;
  if (force_waves < 0) {
    const char* e = getenv("RYOLO_WGRAD_WAVES");   // measurement knob
    force_waves = e ? atoi(e) : 0;
  }
  int ksplit = 1;
  {
    double best_eff = 0.0;
    for (int waves = 1; waves <= 4; waves++) {
      if (force_waves > 0 && waves != force_waves) continue;
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
  p.tickets = nullptr;
  if (p.ksplit > 1) {
    const int tiles = p.tap_groups * p.m_tiles * p.n_tiles;
    const size_t per_cta = (size_t)(tg * bn / 2) * 256;
    const size_t tbytes = align_up((size_t)tiles * sizeof(unsigned int), 256);
    char* s = static_cast<char*>(stream_scratch(stream, SCRATCH_WGRAD, tbytes + (size_t)tiles * p.ksplit * per_cta * sizeof(float)));
    if (!s) return RYOLO_E_CUDA;
    p.tickets = reinterpret_cast<unsigned int*>(s);
    p.partials = reinterpret_cast<float*>(s + tbytes);
    RYOLO_CUDA_TRY(cudaMemsetAsync(p.tickets, 0, (size_t)tiles * sizeof(unsigned int), stream));
  }
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
