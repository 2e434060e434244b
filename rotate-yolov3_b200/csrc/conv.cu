// Conv2d -> (folded) BatchNorm -> PReLU [-> + residual] as an sm_90a implicit GEMM.
//
// Replaces the nn.Sequential(Conv2d, BatchNorm2d, PReLU) blocks the reference builds in create_modules
// (model/models.py:49-66) plus the shortcut add (models.py:281-282) and the nearest x2 upsample (models.py:93-94)
// that follow some of them; BN is folded as in utils/torch_utils.py:45-69 (scale into the weights at pack time,
// shift into the epilogue bias).
//
// Layout.  Activations are bf16 "padded NHWC": [B][H+2][W+2][Cs] with a one-pixel ZERO halo (zeroed once at
// allocation, never written afterwards).  With the halo in memory, a 3x3 / stride-1 / pad-1 convolution is nine
// GEMMs that differ only by a constant shift of the FLAT pixel index  p = (b*(H+2) + y)*(W+2) + x :
//        out[p, :] = sum_{tap=(dy,dx)}  A[p + dy*(W+2) + dx, :] * W_tap            (valid for every interior p)
// so the A operand of tap t is a plain 2-D TMA box [128 pixels x 64 channels] whose row coordinate is shifted by
// the tap offset; rows that fall outside [0, NP) are zero-filled by TMA.  No im2col buffer, no gather.  The GEMM
// also produces values at halo positions; the epilogue stores zeros there (same-grid outputs) or skips them.  Cost
// of that: (H+2)(W+2)/HW extra MMA rows (5 % at 76^2, 11 % at 38^2, 22 % at 19^2).
// Stride-2 3x3 layers run on a space-to-depth copy of their input as 2x2-tap stride-1 convs (ksize = 2); odd sizes
// fall back to the stride-1 GEMM on the input grid that stores only the even pixels.
//
// Kernel.  Persistent, warp-specialised, one CTA per SM, tile = 128 pixels x BN filters, BK = 64 channels:
//   warp group 0   TMA producer (one thread): per k-step one A box (shifted by the tap offset) + one B box into a
//                  128B-swizzled shared-memory stage, completion on an mbarrier (expect_tx); gives its registers to
//                  the MMA warp groups (setmaxnreg);
//                  A second warp of warp group 0 is the epilogue DMA of same-grid outputs: it stores each filled
//                  staging tile with TMA and, once the store has read it, refills the tile with a later tile's
//                  residual (TMA, completion on an mbarrier) and its BN bias values;
//   warp groups 1, 2   64 pixel rows each: one wgmma m64n{BN}k16 per 16 channels (the A slice is read from shared
//                  memory once for the whole tile width), fp32 accumulators in registers, one k-step kept in flight
//                  (the stage of the previous one is released when it retires); then the epilogue: +bias -> PReLU ->
//                  +residual -> bf16.  Same-grid outputs are written over the residual in the staging tile and leave
//                  through the DMA warp's TMA stores, which drain while the next tile's MMAs run; fp32 NCHW heads are
//                  transposed through the same staging area and stored as per-channel pixel runs; the nearest x2
//                  up-sampled grid and the strided fallback are stored straight from the fragments.  The producer
//                  keeps filling the ring with the next tile's operands while the epilogue runs.
#include <cuda.h>
#include <cuda_bf16.h>

#include "common.cuh"
#include "pack.cuh"
#include "sm90.cuh"

namespace ryolo {

constexpr int BM = 128;  // pixels per tile (two m64 warp groups)
constexpr int BK = 64;   // channels per k-step = one 128-byte swizzle row of bf16
constexpr int CONV_THREADS = 384;   // warp group 0: TMA; warp groups 1-2: MMA + epilogue

struct ConvParams {
  int np;             // B * (H+2) * (W+2): GEMM M
  int hp, wp;         // padded input height / width
  int taps;           // 1, 9 (3x3, offsets -1..1) or 4 (2x2, offsets -1..0, or 0..1 when tap_flip)
  int tap_flip;
  int kchunks;        // cin_pad / 64
  int cout;           // real filters
  int cout_pad;       // rows per tap in the packed weight
  int n_tiles;        // cout_pad / BN
  int m_tiles;
  int stride;         // 1 or 2
  int oh, ow;         // output spatial size (unpadded)
  int out_cs;         // channel stride of the output buffer
  int store_cols;     // bf16 output: columns [0, store_cols) of the padded filter range are stored
  int has_act, upsample2x, out_f32_nchw;
  int same_grid;      // bf16 stride-1 non-upsampled output: the tile's rows ARE output rows, halo rows are stored as 0
  float slope;
  const float* bias;               // [cout_pad]
  void* out;
  FastDiv d_ntiles, d_wp, d_hp;    // divisions of the epilogue's per-tile index arithmetic
};

// RES: the same-grid epilogue adds a residual (shortcut, dgrad accumulate) that TMA loads into the staging tile.
template <int BN, bool RES>
struct ConvSmem {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  // Operand ring next to the output staging tiles.  Residual launches at BN <= 128 double-buffer the staging tile, so
  // that the store of one tile and the residual load of the next are in flight together; the BN = 128 ring gives up a
  // stage for it (5 instead of 6).  At BN = 256 a second 64 KB tile would leave a 2-stage ring, which exposes the
  // operand latency on every k-step, so one tile is kept and the residual of the next tile is loaded as soon as the
  // store has read it.  144 / 192 (160) / 192 KB of ring.
  static constexpr int kStages = BN == 256 ? 3 : (BN == 128 ? (RES ? 5 : 6) : 8);
  static constexpr int kStagingTiles = RES && BN < 256 ? 2 : 1;
  static constexpr int kStagingOffset = kStages * kStageBytes;
  static constexpr int kStagingBytes = BM * BN * 2;   // per warp group and 64 filters: one [64 px x 64 ch] box, 8 KB
  static constexpr int kBiasOffset = kStagingOffset + kStagingTiles * kStagingBytes;   // fp32 [kStagingTiles][BN]
  static constexpr int kBarOffset = kBiasOffset + kStagingTiles * BN * 4;
  static constexpr int kTotal = kBarOffset + (2 * kStages + 2 * kStagingTiles) * 8 + 1024 /*alignment slack*/;
};

template <int BN, bool RES>
__global__ void __launch_bounds__(CONV_THREADS, 1)
conv_igemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                  const __grid_constant__ CUtensorMap map_out, const __grid_constant__ CUtensorMap map_res,
                  const ConvParams p) {
  using S = ConvSmem<BN, RES>;
  constexpr int NS = BN / 64;   // m64n64 sub-tiles per warp group
  constexpr int NT = S::kStagingTiles;
  extern __shared__ unsigned char smem_raw[];
  // 1024-byte alignment required by the 128B swizzle atoms
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  unsigned char* const smem = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t bar_base = smem_base + S::kBarOffset;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (S::kStages + s); };
  // staging tile b is `ready` when it may be written (its last store has read it; the residual and bias have landed),
  // `filled` when the MMA warps have written the tile's output into it
  auto ready_bar = [&](int b) { return bar_base + 8u * (2 * S::kStages + b); };
  auto filled_bar = [&](int b) { return bar_base + 8u * (2 * S::kStages + NT + b); };

  const int wg = threadIdx.x >> 7;
  const int total_tiles = p.m_tiles * p.n_tiles;
  const int k_iters = p.taps * p.kchunks;

  if (threadIdx.x == 0) {
    for (int s = 0; s < S::kStages; s++) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);   // one arrive per MMA warp
    }
    for (int b = 0; b < NT; b++) {
      mbar_init(ready_bar(b), 1);
      mbar_init(filled_bar(b), 8);   // one arrive per MMA warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    regs_dealloc<40>();
    if (threadIdx.x >= 32 && threadIdx.x < 64 && p.same_grid) {
      // ===================== epilogue DMA (same-grid outputs) =====================
      const int lane = threadIdx.x & 31;
      // make staging tile b ready for `tile`: its bias values, then its residual boxes or a plain arrive
      auto prepare = [&](int tile, int b) {
        int mt, nt;
        fast_divmod(tile, p.d_ntiles, mt, nt);
        float* const sb = reinterpret_cast<float*>(smem + S::kBiasOffset) + b * BN;
        for (int c = lane; c < BN; c += 32) sb[c] = __ldg(p.bias + nt * BN + c);
        __syncwarp();
        if (lane != 0) return;
        if constexpr (RES) {
          // The map's inner extent is cout: filters at and above it load as zeros.  A box that starts at or beyond
          // cout also starts at or beyond store_cols = round_up(cout, 32), and one that starts at or beyond np is
          // clipped whole: neither is stored, so neither is loaded.
          const int nc = min(NS, (p.cout - nt * BN + 63) / 64);
          const int nh = mt * BM + 64 < p.np ? 2 : 1;
          mbar_expect_tx(ready_bar(b), (uint32_t)(nh * nc * 8192));
          const uint32_t stg = smem_base + S::kStagingOffset + b * S::kStagingBytes;
          for (int h = 0; h < nh; h++)
            for (int n = 0; n < nc; n++)
              tma_load_2d(stg + (h * NS + n) * 8192, &map_res, ready_bar(b), nt * BN + n * 64, mt * BM + h * 64);
        } else {
          mbar_arrive(ready_bar(b));
        }
      };
      int j = 0;
      for (int tile = blockIdx.x; tile < total_tiles && j < NT; tile += gridDim.x, j++) prepare(tile, j);
      j = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, j++) {
        const int b = j % NT;
        mbar_wait(filled_bar(b), (j / NT) & 1);
        if (lane == 0) {
          // the output map's extents (store_cols channels, np rows) clip what lies beyond them
          int mt, nt;
          fast_divmod(tile, p.d_ntiles, mt, nt);
          const uint32_t stg = smem_base + S::kStagingOffset + b * S::kStagingBytes;
          for (int h = 0; h < 2; h++) {
            const int row0 = mt * BM + h * 64;
            if (row0 >= p.np) break;
            for (int n = 0; n < NS; n++)
              if (nt * BN + n * 64 < p.store_cols) tma_store_2d(&map_out, stg + (h * NS + n) * 8192, nt * BN + n * 64, row0);
          }
          bulk_commit();
        }
        const int next = tile + NT * gridDim.x;
        if (next < total_tiles) {
          // the tiles partition the output: a later tile's residual never overlaps a store still in flight
          if (lane == 0) bulk_wait_read();
          prepare(next, b);
        }
      }
      if (lane == 0) bulk_wait();   // the CTA's last stores are complete before it exits
    }
    if (threadIdx.x == 0) {
      // ===================== TMA producer =====================
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int mt = tile / p.n_tiles, nt = tile % p.n_tiles;
        const int p0 = mt * BM;
        for (int kk = 0; kk < k_iters; kk++) {
          const int tap = kk / p.kchunks, kc = kk % p.kchunks;
          int off = 0;
          if (p.taps == 9) off = (tap / 3 - 1) * p.wp + (tap % 3 - 1);
          else if (p.taps == 4) off = (tap / 2 - 1 + p.tap_flip) * p.wp + (tap % 2 - 1 + p.tap_flip);
          mbar_wait(empty_bar(stage), phase ^ 1);
          const uint32_t sa = smem_base + stage * S::kStageBytes;
          mbar_expect_tx(full_bar(stage), S::kStageBytes);
          tma_load_2d(sa, &map_a, full_bar(stage), kc * BK, p0 + off);
          tma_load_2d(sa + S::kABytes, &map_b, full_bar(stage), kc * BK, tap * p.cout_pad + nt * BN);
          if (++stage == S::kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== MMA + epilogue: warp group `half` owns tile rows [64 half, 64 half + 64) =====================
  regs_alloc<232>();
  const int half = wg - 1;
  const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
  const int quad = lane & 3;
  float acc[BN / 2];   // m64n{BN} fragment: [32 n + i] is entry i of the 64-filter sub-tile n
  int stage = 0;
  uint32_t phase = 0;
  int jt = 0;          // tiles of this CTA so far: staging tile jt % NT
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, jt++) {
    int mt, nt;
    fast_divmod(tile, p.d_ntiles, mt, nt);
    int prev = -1;
    for (int kk = 0; kk < k_iters; kk++) {
      mbar_wait(full_bar(stage), phase);
      const uint32_t sa = smem_base + stage * S::kStageBytes;
      const uint64_t adesc = make_smem_desc(sa + half * 64 * 128);
      // the B box is BN consecutive 128-byte rows: one descriptor covers the whole tile
      const uint64_t bdesc = make_smem_desc(sa + S::kABytes);
      wg_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; k++) {
        // +32 bytes (16 bf16) along K inside the swizzle atom: start-address field += 2
        wgmma_bf16<BN, 0, 0>(acc, adesc + 2 * k, bdesc + 2 * k, (kk | k) != 0);
      }
      wg_commit();
      // the previous k-step has retired: its stage may be refilled
      wg_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
      prev = stage;
      if (++stage == S::kStages) { stage = 0; phase ^= 1; }
    }
    wg_wait<0>();
    wg_fence_regs(acc);
    if (lane == 0) mbar_arrive(empty_bar(prev));

    // ---- epilogue: this thread holds rows r0 and r0 + 8, columns 8 j + 2 quad + {0, 1} of every 64-filter sub-tile
    if (p.same_grid) {
      // The tile's rows ARE output rows: the warp group converts its 64 x BN fragment into its half of the staging tile
      // (one 128B-swizzled [64 px x 64 ch] TMA box per 64 filters: a warp's 8 rows x 16 bytes land in 8 distinct 16-byte
      // chunks, no bank conflicts), over the residual the DMA warp loaded there, and the DMA warp stores it.  Every
      // shared-memory read comes before the first write, so that the compiler may batch the reads.
      const int sbuf = jt % NT;
      mbar_wait(ready_bar(sbuf), (jt / NT) & 1);
      uint32_t* const stg =
          reinterpret_cast<uint32_t*>(smem + S::kStagingOffset + sbuf * S::kStagingBytes + half * NS * 8192);
      const float* const sb = reinterpret_cast<const float*>(smem + S::kBiasOffset) + sbuf * BN;
      // word index of this thread's pair (row warp * 16 + lane / 4 + 8 i, filters n * 64 + 8 j + 2 quad + {0, 1})
      auto widx = [&](int i, int n, int j) {
        const int row = warp * 16 + (lane >> 2) + 8 * i;
        return n * 2048 + row * 32 + ((j ^ (row & 7)) << 2) + quad;
      };
#pragma unroll
      for (int n = 0; n < NS; n++) {
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const float2 bb = *reinterpret_cast<const float2*>(sb + n * 64 + 8 * j + 2 * quad);
#pragma unroll
          for (int i = 0; i < 2; i++) {
            float& x0 = acc[32 * n + 4 * j + 2 * i];
            float& x1 = acc[32 * n + 4 * j + 2 * i + 1];
            // + bias even where it is zero: -0 + 0 = +0
            x0 += bb.x;
            x1 += bb.y;
            if (p.has_act) {
              x0 = x0 > 0.f ? x0 : p.slope * x0;
              x1 = x1 > 0.f ? x1 : p.slope * x1;
            }
            if constexpr (RES) {
              // filters at and above cout read as zeros; __fadd_rn is never contracted with the PReLU multiply
              const uint32_t rw = stg[widx(i, n, j)];
              x0 = __fadd_rn(x0, __uint_as_float(rw << 16));
              x1 = __fadd_rn(x1, __uint_as_float(rw & 0xffff0000u));
            }
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 2; i++) {
        const int pix = mt * BM + half * 64 + warp * 16 + (lane >> 2) + 8 * i;   // flat padded pixel; >= np is clipped
        int b, yp, xp, tt;
        fast_divmod(pix, p.d_wp, tt, xp);
        fast_divmod(tt, p.d_hp, b, yp);
        // halo rows are stored as zeros: the halo stays zero
        const bool valid = pix < p.np && xp >= 1 && xp <= p.wp - 2 && yp >= 1 && yp <= p.hp - 2;
#pragma unroll
        for (int n = 0; n < NS; n++) {
#pragma unroll
          for (int j = 0; j < 8; j++) {
            const __nv_bfloat162 h = __floats2bfloat162_rn(acc[32 * n + 4 * j + 2 * i], acc[32 * n + 4 * j + 2 * i + 1]);
            stg[widx(i, n, j)] = valid ? *reinterpret_cast<const uint32_t*>(&h) : 0u;
          }
        }
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(filled_bar(sbuf));
      continue;
    }
    if (p.out_f32_nchw && p.stride == 1 && !p.upsample2x) {
      // Heads, fp32 [B, cout, oh, ow]: the fragment is transposed through the warp group's staging area 32 filters at a
      // time ([32 ch][64 px] fp32, 8 KB; a pixel's column is XOR-swizzled by (ch / 2) % 4 so that the fragment writes
      // and the row reads are conflict-free), then thread t stores pixel t % 64 of channels t / 64, t / 64 + 2, ..: a
      // warp writes 32 consecutive pixels of one channel, contiguous in the output up to an image-row or halo boundary.
      float* const stg = reinterpret_cast<float*>(smem_raw + (smem_base + S::kStagingOffset - smem_u32(smem_raw))) +
                         half * NS * 2048;
      const int spx = t & 63, sch = t >> 6;
      size_t obase = 0;
      bool ovalid;
      {
        const int pix = mt * BM + half * 64 + spx;
        int b, yp, xp, tt;
        fast_divmod(pix, p.d_wp, tt, xp);
        fast_divmod(tt, p.d_hp, b, yp);
        ovalid = pix < p.np && xp >= 1 && xp <= p.wp - 2 && yp >= 1 && yp <= p.hp - 2 && yp - 1 < p.oh && xp - 1 < p.ow;
        obase = (size_t)b * p.cout * p.oh * p.ow + (size_t)(yp - 1) * p.ow + (xp - 1);
      }
      const size_t plane = (size_t)p.oh * p.ow;
      float* const o = reinterpret_cast<float*>(p.out);
#pragma unroll
      for (int n = 0; n < NS; n++) {
#pragma unroll
        for (int hc = 0; hc < 2; hc++) {
#pragma unroll
          for (int i = 0; i < 2; i++) {
            const int row = warp * 16 + (lane >> 2) + 8 * i;
#pragma unroll
            for (int jj = 0; jj < 4; jj++) {
              const int j = 4 * hc + jj;
              const int col = nt * BN + n * 64 + 8 * j + 2 * quad;   // even filter index of this thread's pair
              const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + col));
              float x0 = acc[32 * n + 4 * j + 2 * i] + bb.x, x1 = acc[32 * n + 4 * j + 2 * i + 1] + bb.y;
              if (p.has_act) {
                x0 = x0 > 0.f ? x0 : p.slope * x0;
                x1 = x1 > 0.f ? x1 : p.slope * x1;
              }
              const int ch = 8 * jj + 2 * quad;                       // (ch / 2) % 4 == quad
              stg[ch * 64 + (row ^ (quad << 3))] = x0;
              stg[(ch + 1) * 64 + (row ^ (quad << 3))] = x1;
            }
          }
          asm volatile("bar.sync %0, 128;" ::"r"(1 + half) : "memory");
          if (ovalid) {
#pragma unroll
            for (int s = 0; s < 16; s++) {
              const int ch = sch + 2 * s;
              const int col = nt * BN + n * 64 + hc * 32 + ch;
              if (col < p.cout) o[obase + (size_t)col * plane] = stg[ch * 64 + (spx ^ (((ch >> 1) & 3) << 3))];
            }
          }
          asm volatile("bar.sync %0, 128;" ::"r"(1 + half) : "memory");   // the area is free for the next 32 filters
        }
      }
      continue;
    }
    // up-sampled or strided outputs: stored straight from the fragments
#pragma unroll
    for (int i = 0; i < 2; i++) {
      const int pix = mt * BM + half * 64 + warp * 16 + (lane >> 2) + 8 * i;   // flat padded input-grid pixel
      if (pix >= p.np) continue;
      int b, yp, xp, tt;
      fast_divmod(pix, p.d_wp, tt, xp);
      fast_divmod(tt, p.d_hp, b, yp);
      bool valid = xp >= 1 && xp <= p.wp - 2 && yp >= 1 && yp <= p.hp - 2;
      int oy = yp - 1, ox = xp - 1;
      if (p.stride == 2) {
        valid = valid && ((oy & 1) == 0) && ((ox & 1) == 0);
        oy >>= 1;
        ox >>= 1;
      }
      valid = valid && oy < p.oh && ox < p.ow;
      if (!valid) continue;
#pragma unroll
      for (int n = 0; n < NS; n++) {
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const int col = nt * BN + n * 64 + 8 * j + 2 * quad;   // even filter index of this thread's pair
          if (!p.out_f32_nchw && col >= p.store_cols) continue;
          const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + col));
          float x0 = acc[32 * n + 4 * j + 2 * i] + bb.x, x1 = acc[32 * n + 4 * j + 2 * i + 1] + bb.y;
          if (p.has_act) {
            x0 = x0 > 0.f ? x0 : p.slope * x0;
            x1 = x1 > 0.f ? x1 : p.slope * x1;
          }
          if (p.out_f32_nchw) {
            // heads: fp32 [B, cout, oh, ow]
            float* o = reinterpret_cast<float*>(p.out);
            const size_t plane = (size_t)p.oh * p.ow;
            const size_t base = ((size_t)b * p.cout) * plane + (size_t)oy * p.ow + ox;
            if (col < p.cout) o[base + (size_t)col * plane] = x0;
            if (col + 1 < p.cout) o[base + (size_t)(col + 1) * plane] = x1;
            continue;
          }
          const __nv_bfloat162 h = __floats2bfloat162_rn(x0, x1);
          const uint32_t hw = *reinterpret_cast<const uint32_t*>(&h);
          __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out);
          const int ohp = (p.upsample2x ? 2 * p.oh : p.oh) + 2, owp = (p.upsample2x ? 2 * p.ow : p.ow) + 2;
          const int reps = p.upsample2x ? 2 : 1;
          for (int ry = 0; ry < reps; ry++)
            for (int rx = 0; rx < reps; rx++) {
              const int yy = (p.upsample2x ? 2 * oy + ry : oy) + 1, xx = (p.upsample2x ? 2 * ox + rx : ox) + 1;
              *reinterpret_cast<uint32_t*>(o + (((size_t)b * ohp + yy) * owp + xx) * p.out_cs + col) = hw;
            }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// weight packing: [cout, cin, k, k] fp32 (* per-filter scale) -> bf16 [k*k][cout_pad][cin_pad], zero padded
// ---------------------------------------------------------------------------------------------------------------
// modes: see pack.cuh
__global__ void conv_pack_weights_kernel(const float* __restrict__ w, const float* __restrict__ scale, int cout, int cin,
                                         int ks, int cout_pad, int cin_pad, int mode, __nv_bfloat16* __restrict__ out) {
  const size_t total = (size_t)ks * ks * cout_pad * cin_pad;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int ci = (int)(i % cin_pad);
    const int co = (int)((i / cin_pad) % cout_pad);
    const int tap = (int)(i / ((size_t)cin_pad * cout_pad));
    float v = 0.f;
    if (ci < cin && co < cout) {
      v = pack_value(w, cout, cin, ks, mode, tap, co, ci);
      if (scale && (mode == 0 || mode == 2)) v *= scale[co];
    }
    out[i] = __float2bfloat16_rn(v);
  }
}

// weight-gradient unpack: dw fp32 [taps][cout_pad][cin_pad] (wgrad output) -> grad [cout][cin][k][k] in nn.Conv2d layout.
// mode 0: plain k x k;  mode 2: space-to-depth form (taps 2x2, cin_eff = 4C) -> [cout][C][3][3]
__global__ void conv_unpack_wgrad_kernel(const float* __restrict__ dw, int cout_pad, int cin_pad, int mode, int cout, int cin,
                                         int ks, float* __restrict__ grad) {
  const size_t total = (size_t)cout * cin * ks * ks;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int kw = (int)(i % ks), kh = (int)((i / ks) % ks);
  const int c = (int)((i / ((size_t)ks * ks)) % cin);
  const int co = (int)(i / ((size_t)ks * ks * cin));
  if (mode == 0) {
    grad[i] = dw[((size_t)(kh * ks + kw) * cout_pad + co) * cin_pad + c];
  } else {
    const int qy = kh == 0 ? 0 : 1, py = kh == 1 ? 0 : 1, qx = kw == 0 ? 0 : 1, px = kw == 1 ? 0 : 1;
    grad[i] = dw[((size_t)(qy * 2 + qx) * cout_pad + co) * cin_pad + (py * 2 + px) * cin + c];
  }
}

static int round_up(int x, int m) { return (x + m - 1) / m * m; }

struct ConvGeom {
  int cin_pad, cout_pad, bn, taps;
};
static ConvGeom conv_geom(const ryolo_conv_desc* d) {
  ConvGeom g;
  g.cin_pad = round_up(d->cin, 64);
  g.bn = d->cout > 128 ? 256 : (d->cout > 64 ? 128 : 64);
  g.cout_pad = round_up(d->cout, g.bn);
  const int k = d->ksize < 0 ? -d->ksize : d->ksize;
  g.taps = k * k;
  return g;
}

// cuTensorMapEncodeTiled is a DRIVER entry point; it is resolved through the runtime at first use so that
// libryolo.so does not link libcuda.so.1 and still loads (for symbol / workspace queries) on a GPU-less host.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
    else
      cudaGetLastError();
  }
  return fn;
}

int encode_map_2d(CUtensorMap* m, const void* base, uint64_t inner, uint64_t rows, uint64_t row_stride_bytes,
                         uint32_t box_inner, uint32_t box_rows) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) {
    set_err("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return RYOLO_E_CUDA;
  }
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_err("cuTensorMapEncodeTiled failed: CUresult %d (inner=%llu rows=%llu stride=%llu box=%ux%u base=%p)", (int)r,
            (unsigned long long)inner, (unsigned long long)rows, (unsigned long long)row_stride_bytes, box_inner, box_rows,
            base);
    return RYOLO_E_CUDA;
  }
  return RYOLO_OK;
}

template <int BN, bool RES>
static int launch_conv(const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& mo, const CUtensorMap& mr,
                       const ConvParams& p, cudaStream_t stream) {
  using S = ConvSmem<BN, RES>;
  static_assert(S::kTotal <= 227 * 1024, "shared memory budget");
  RYOLO_SMEM_OPT_IN((conv_igemm_kernel<BN, RES>), S::kTotal);
  const int num_sms = gemm_sm_count();
  const int total = p.m_tiles * p.n_tiles;
  const int grid = total < num_sms ? total : num_sms;
  conv_igemm_kernel<BN, RES><<<grid, CONV_THREADS, S::kTotal, stream>>>(ma, mb, mo, mr, p);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

template <int BN>
static int launch_conv(const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& mo, const CUtensorMap& mr,
                       bool has_res, const ConvParams& p, cudaStream_t stream) {
  return has_res ? launch_conv<BN, true>(ma, mb, mo, mr, p, stream) : launch_conv<BN, false>(ma, mb, mo, mr, p, stream);
}

}  // namespace ryolo

using namespace ryolo;

extern "C" size_t ryolo_conv_packed_weight_bytes(const ryolo_conv_desc* d) {
  if (!d) return 0;
  const ConvGeom g = conv_geom(d);
  return (size_t)g.taps * g.cout_pad * g.cin_pad * 2;
}

extern "C" int ryolo_conv_unpack_wgrad(const float* dw, int cout_pad, int cin_pad, int mode, int cout, int cin, int ksize,
                                       float* grad, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(dw && grad && cout > 0 && cin > 0 && (mode == 0 || mode == 2));
  RYOLO_ARG_CHECK(mode == 0 ? (ksize == 1 || ksize == 3) : ksize == 3);
  const size_t total = (size_t)cout * cin * ksize * ksize;
  conv_unpack_wgrad_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(dw, cout_pad, cin_pad, mode, cout, cin, ksize,
                                                                                grad);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_conv_pack_weights_ex(const ryolo_conv_desc* d, const float* weight, const float* scale,
                                          void* packed_out, int mode, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(d && weight && packed_out && mode >= 0 && mode <= 3);
  RYOLO_ARG_CHECK(mode < 2 || ((d->ksize == 2 || d->ksize == -2) && (mode == 2 ? d->cin % 4 == 0 : d->cout % 4 == 0)));
  RYOLO_ARG_CHECK(d->ksize == 1 || d->ksize == 3 || d->ksize == 2 || d->ksize == -2);
  const ConvGeom g = conv_geom(d);
  const size_t total = (size_t)g.taps * g.cout_pad * g.cin_pad;
  const int blocks = (int)((total + 255) / 256 > 4096 ? 4096 : (total + 255) / 256);
  conv_pack_weights_kernel<<<blocks, 256, 0, stream>>>(weight, scale, d->cout, d->cin, d->ksize < 0 ? -d->ksize : d->ksize,
                                                        g.cout_pad, g.cin_pad, mode,
                                                        static_cast<__nv_bfloat16*>(packed_out));
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_conv_bn_act_fwd(const ryolo_conv_desc* d, const void* x, const void* packed_w, const float* bias,
                                     const void* residual, void* y, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(d && x && packed_w && bias && y);
  RYOLO_ARG_CHECK(d->batch > 0 && d->in_h > 0 && d->in_w > 0 && d->cin > 0 && d->cout > 0);
  RYOLO_ARG_CHECK(d->ksize == 1 || d->ksize == 3 || d->ksize == 2 || d->ksize == -2);
  RYOLO_ARG_CHECK(d->stride == 1 || (d->stride == 2 && d->ksize != 2 && d->ksize != -2));
  RYOLO_ARG_CHECK(!(d->stride == 2 && d->upsample2x));
  RYOLO_ARG_CHECK(!d->has_residual || (residual != nullptr && d->stride == 1 && !d->upsample2x &&
                                        d->res_stride % 8 == 0 && d->out_dtype == RYOLO_DT_BF16));
  const ConvGeom g = conv_geom(d);
  // a buffer narrower than the 64-wide K chunk is fine: TMA zero-fills the part of the box beyond the inner extent
  RYOLO_ARG_CHECK(d->cin_stride >= d->cin && d->cin_stride % 8 == 0);
  RYOLO_ARG_CHECK(d->out_dtype == RYOLO_DT_BF16 || d->out_dtype == RYOLO_DT_F32);
  RYOLO_ARG_CHECK(!d->has_residual || (reinterpret_cast<uintptr_t>(residual) & 15) == 0);
  if (d->out_dtype == RYOLO_DT_BF16) RYOLO_ARG_CHECK(d->cout_stride % 8 == 0 && d->cout_stride >= round_up(d->cout, 32));
  RYOLO_ARG_CHECK((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0);

  ConvParams p;
  p.hp = d->in_h + 2;
  p.wp = d->in_w + 2;
  const long long np = (long long)d->batch * p.hp * p.wp;
  RYOLO_ARG_CHECK(np < (1ll << 31) - 4096);
  p.np = (int)np;
  p.taps = g.taps;
  p.tap_flip = d->ksize == -2 ? 1 : 0;
  p.kchunks = g.cin_pad / 64;
  p.cout = d->cout;
  p.cout_pad = g.cout_pad;
  p.n_tiles = g.cout_pad / g.bn;
  p.d_ntiles = make_fastdiv(p.n_tiles);
  p.d_wp = make_fastdiv(p.wp);
  p.d_hp = make_fastdiv(p.hp);
  p.m_tiles = (p.np + BM - 1) / BM;
  p.stride = d->stride;
  p.oh = d->stride == 2 ? (d->in_h + 1) / 2 : d->in_h;   // k=3,pad=1 (or k=1,pad=0) with stride 2: ceil(h/2)
  p.ow = d->stride == 2 ? (d->in_w + 1) / 2 : d->in_w;
  p.out_cs = d->cout_stride;
  p.store_cols = round_up(d->cout, 32);   // never touch channels beyond the 32-column chunk that holds the last filter
  p.has_act = d->has_act;
  p.upsample2x = d->upsample2x;
  p.out_f32_nchw = d->out_dtype == RYOLO_DT_F32;
  p.slope = d->slope;
  p.bias = bias;
  p.out = y;
  p.same_grid = (d->out_dtype == RYOLO_DT_BF16 && d->stride == 1 && !d->upsample2x) ? 1 : 0;
  CUtensorMap ma, mb;
  const int a_inner = d->cin_stride < g.cin_pad ? d->cin_stride : g.cin_pad;
  int st = encode_map_2d(&ma, x, (uint64_t)a_inner, (uint64_t)p.np, (uint64_t)d->cin_stride * 2, BK, BM);
  if (st != RYOLO_OK) return st;
  st = encode_map_2d(&mb, packed_w, (uint64_t)g.cin_pad, (uint64_t)g.taps * g.cout_pad, (uint64_t)g.cin_pad * 2, BK,
                     (uint32_t)g.bn);
  if (st != RYOLO_OK) return st;
  // same-grid output: the epilogue's TMA store map.  Base = the output view, inner extent = store_cols: channels at or
  // beyond it (a concat neighbour, the rest of a wider buffer) are never written.  Other outputs leave it unused.
  CUtensorMap mo, mr;
  memset(&mo, 0, sizeof(mo));
  memset(&mr, 0, sizeof(mr));
  if (p.same_grid) {
    st = encode_map_2d(&mo, y, (uint64_t)p.store_cols, (uint64_t)p.np, (uint64_t)p.out_cs * 2, 64, BM / 2);
    if (st != RYOLO_OK) return st;
  }
  // residual (same grid: checked above): the same boxes as the store map; inner extent cout, so TMA zero-fills the
  // filters at and above it.  It may be the output view itself, a view into a wider buffer, or a separate buffer.
  const bool has_res = d->has_residual != 0;
  if (has_res) {
    st = encode_map_2d(&mr, residual, (uint64_t)d->cout, (uint64_t)p.np, (uint64_t)d->res_stride * 2, 64, BM / 2);
    if (st != RYOLO_OK) return st;
  }
  if (g.bn == 256) return launch_conv<256>(ma, mb, mo, mr, has_res, p, stream);
  if (g.bn == 128) return launch_conv<128>(ma, mb, mo, mr, has_res, p, stream);
  return launch_conv<64>(ma, mb, mo, mr, has_res, p, stream);
}
