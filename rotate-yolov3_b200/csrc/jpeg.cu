// Decodes a batch of baseline / extended sequential Huffman JPEG streams into uint8 HWC BGR images, byte for byte what
// cv2.imread returns (libjpeg-turbo's ISLOW IDCT, fancy upsampling and YCbCr -> BGR; csrc/jpeg.cuh restates each step).
//
// Entropy stage, over the chunks of every restart interval (segment) of the batch (Weissenberger & Schmidt, "Massively
// Parallel Huffman Decoding on GPUs", ICPP 2018):
//   pass A    one thread per chunk decodes from the chunk's first byte to its end and keeps the state it stops in.
//             Huffman codes resynchronise: a decoder that starts mid-symbol soon falls onto the true symbol boundaries.
//   pass B    one thread per chunk decodes on from where the previous chunk's pass A stopped (the segment start for a
//             segment's first chunk) until, at the end of some chunk j, its state equals pass A's state there; it
//             records j and the blocks it began.  A thread whose start is true covers chunks k..j on the true path and
//             hands over to j + 1, whose start (pass A's state at j) is then true too.
//   resolve   one warp per segment follows that chain from the segment's first chunk and gives each chunk on it the
//             number of blocks begun before it; a chain that breaks (no synchronisation) or ends short sets the status.
//   write     each chunk on the chain decodes its range again and stores the coefficients; every coefficient position
//             of every block is written by exactly one thread.
//   DC        one CTA per (segment, component) turns DC differences into values by a prefix sum.
// Pixel stage: one thread per block dequantises and runs the ISLOW IDCT into the component planes, and flags a block
// outside the range where libjpeg-turbo's IDCTs agree (RYOLO_JPEG_ST_RANGE); one CTA per output
// row upsamples, converts the colour and stores B, G, R with the Exif orientation applied.
#include "common.cuh"
#include "jpeg.cuh"

namespace ryolo {

using jpeg::State;

namespace {

constexpr int kChunkThreads = 128;
constexpr int kDcThreads = 256;
constexpr int kDcPerThread = 4;
constexpr int kIdctThreads = 128;
constexpr int kPixThreads = 256;

struct ChunkWs {
  uint32_t* exits;    // [nchunks][2] pass A's state at the chunk's end
  int32_t* jump;      // pass B: last chunk covered (absolute), -1 when it did not synchronise
  int32_t* nblk;      // pass B: blocks begun
  int32_t* base;      // resolve: blocks of the segment begun before the chunk; -1 off the true path
};

ChunkWs carve(void* ws, int nchunks, uint8_t** area) {
  Carver cv(ws);
  ChunkWs w;
  w.exits = cv.take<uint32_t>(2 * (size_t)nchunks);
  w.jump = cv.take<int32_t>(nchunks);
  w.nblk = cv.take<int32_t>(nchunks);
  w.base = cv.take<int32_t>(nchunks);
  *area = cv.take<uint8_t>(0);
  return w;
}

__global__ void __launch_bounds__(kChunkThreads)
    jpeg_pass_a_kernel(const ryolo_jpeg_image* __restrict__ images, const ryolo_jpeg_segment* __restrict__ segs,
                       const int32_t* __restrict__ chunk_seg, int nchunks, int chunk_bytes,
                       const uint8_t* __restrict__ data, const ryolo_jpeg_huff* __restrict__ huff, ChunkWs w) {
  const int c = blockIdx.x * kChunkThreads + threadIdx.x;
  if (c >= nchunks) return;
  const ryolo_jpeg_segment sg = segs[chunk_seg[c]];
  const State s = jpeg::chunk_pass_a(data, sg, images[sg.image], huff, c - sg.first_chunk, chunk_bytes);
  jpeg::pack(s, w.exits + 2 * (size_t)c);
}

__global__ void __launch_bounds__(kChunkThreads)
    jpeg_pass_b_kernel(const ryolo_jpeg_image* __restrict__ images, const ryolo_jpeg_segment* __restrict__ segs,
                       const int32_t* __restrict__ chunk_seg, int nchunks, int chunk_bytes,
                       const uint8_t* __restrict__ data, const ryolo_jpeg_huff* __restrict__ huff, ChunkWs w) {
  const int c = blockIdx.x * kChunkThreads + threadIdx.x;
  if (c >= nchunks) return;
  const ryolo_jpeg_segment sg = segs[chunk_seg[c]];
  const int k = c - sg.first_chunk;
  const State s = k == 0 ? jpeg::segment_start(sg) : jpeg::unpack(w.exits + 2 * (size_t)(c - 1));
  int nb = 0;
  const int j = jpeg::chunk_pass_b(data, sg, images[sg.image], huff, k, chunk_bytes, s,
                                   w.exits + 2 * (size_t)sg.first_chunk, &nb);
  w.jump[c] = j < 0 ? -1 : sg.first_chunk + j;
  w.nblk[c] = nb;
  w.base[c] = -1;
}

// one warp per segment: lanes take 32 consecutive chunks from the chain's current chunk p and apply jpeg::on_chain /
// next_chain (csrc/jpeg.cuh): every chunk before the first lane whose pass B did not stop in its own chunk is on the
// chain, and so is that lane's chunk when its pass B synchronised; the chain continues behind the chunk it stopped in
__global__ void __launch_bounds__(32)
    jpeg_resolve_kernel(const ryolo_jpeg_image* __restrict__ images, const ryolo_jpeg_segment* __restrict__ segs,
                        int32_t* __restrict__ status, ChunkWs w) {
  const ryolo_jpeg_segment sg = segs[blockIdx.x];
  const int lane = threadIdx.x, end = sg.first_chunk + sg.nchunk;
  int p = sg.first_chunk, base = 0;
  bool broken = false;
  while (p < end) {
    const int idx = p + lane;
    const bool valid = idx < end;
    const int j = valid ? w.jump[idx] : 0;
    const int nb = valid ? w.nblk[idx] : 0;
    const unsigned jumps = __ballot_sync(0xffffffffu, valid && j != idx);
    const int first = jumps ? __ffs(jumps) - 1 : 32;
    const int jf = __shfl_sync(0xffffffffu, j, first & 31);
    const bool link = valid && jpeg::on_chain(lane, first, jf);
    int incl = link ? nb : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (link) w.base[idx] = base + incl - nb;
    base += __shfl_sync(0xffffffffu, incl, 31);
    p = jpeg::next_chain(p, first, jf);
    if (p < 0) {
      broken = true;
      break;
    }
  }
  if (lane == 0) {
    int st = broken ? RYOLO_JPEG_ST_NO_SYNC : 0;
    if (!broken && base < sg.nmcu * images[sg.image].bpm) st |= RYOLO_JPEG_ST_TRUNCATED;
    if (st) atomicOr(status + sg.image, st);
  }
}

__global__ void __launch_bounds__(kChunkThreads)
    jpeg_write_kernel(const ryolo_jpeg_image* __restrict__ images, const ryolo_jpeg_segment* __restrict__ segs,
                      const int32_t* __restrict__ chunk_seg, int nchunks, int chunk_bytes,
                      const uint8_t* __restrict__ data, const ryolo_jpeg_huff* __restrict__ huff, ChunkWs w,
                      uint8_t* __restrict__ area, int32_t* __restrict__ status) {
  const int c = blockIdx.x * kChunkThreads + threadIdx.x;
  if (c >= nchunks) return;
  const int first_block = w.base[c];
  if (first_block < 0 || w.jump[c] < 0) return;
  const ryolo_jpeg_segment sg = segs[chunk_seg[c]];
  const ryolo_jpeg_image& im = images[sg.image];
  const int k = c - sg.first_chunk;
  const State s = k == 0 ? jpeg::segment_start(sg) : jpeg::unpack(w.exits + 2 * (size_t)(c - 1));
  int16_t* blocks = reinterpret_cast<int16_t*>(area + im.coef_off) + (int64_t)sg.first_mcu * im.bpm * 64;
  const int st = jpeg::chunk_write(data, sg, im, huff, w.jump[c] - sg.first_chunk, chunk_bytes, s, first_block, blocks);
  if (st) atomicOr(status + sg.image, st);
}

// DC differences -> DC values for one (segment, component): a CTA-wide wrapping int32 prefix sum in tiles
__global__ void __launch_bounds__(kDcThreads)
    jpeg_dc_kernel(const ryolo_jpeg_image* __restrict__ images, const ryolo_jpeg_segment* __restrict__ segs,
                   uint8_t* __restrict__ area) {
  __shared__ uint32_t warp_sum[kDcThreads / 32];
  const ryolo_jpeg_segment sg = segs[blockIdx.x];
  const ryolo_jpeg_image& im = images[sg.image];
  const int ci = blockIdx.y;
  if (ci >= im.ncomp) return;
  int16_t* coefs = reinterpret_cast<int16_t*>(area + im.coef_off);
  const int64_t n = (int64_t)sg.nmcu * im.h[ci] * im.v[ci];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t carry = 0;
  for (int64_t t0 = 0; t0 < n; t0 += kDcThreads * kDcPerThread) {
    const int64_t e0 = t0 + (int64_t)threadIdx.x * kDcPerThread;
    uint32_t v[kDcPerThread];
    uint32_t sum = 0;
#pragma unroll
    for (int i = 0; i < kDcPerThread; i++) {
      v[i] = e0 + i < n ? (uint32_t)(int32_t)coefs[jpeg::dc_block(im, sg, ci, e0 + i) * 64] : 0u;
      sum += v[i];
    }
    uint32_t incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) warp_sum[warp] = incl;
    __syncthreads();
    uint32_t before = carry, total = 0;
#pragma unroll
    for (int i = 0; i < kDcThreads / 32; i++) {
      before += i < warp ? warp_sum[i] : 0u;
      total += warp_sum[i];
    }
    __syncthreads();
    uint32_t run = before + incl - sum;
#pragma unroll
    for (int i = 0; i < kDcPerThread; i++) {
      run += v[i];
      if (e0 + i < n) coefs[jpeg::dc_block(im, sg, ci, e0 + i) * 64] = (int16_t)(run & 0xFFFFu);
    }
    carry += total;
  }
}

__global__ void __launch_bounds__(kIdctThreads)
    jpeg_idct_kernel(const ryolo_jpeg_image* __restrict__ images, const uint16_t* __restrict__ quant,
                     uint8_t* __restrict__ area, int32_t* __restrict__ status) {
  const ryolo_jpeg_image& im = images[blockIdx.y];
  const int64_t b = (int64_t)blockIdx.x * kIdctThreads + threadIdx.x;
  if (b >= (int64_t)im.mcux * im.mcuy * im.bpm) return;
  int row, col;
  const int ci = jpeg::block_position(im, b, row, col);
  union {
    int4 v[8];
    int16_t s[64];
  } blk;
  const int4* src = reinterpret_cast<const int4*>(area + im.coef_off) + b * 8;
#pragma unroll
  for (int i = 0; i < 8; i++) blk.v[i] = src[i];
  const int pitch = im.pitch[ci];
  const int st =
      jpeg::idct_islow(blk.s, quant + im.qtab[ci], area + im.plane_off[ci] + (int64_t)row * pitch + col, pitch);
  if (st) atomicOr(status + blockIdx.y, st);
}

__global__ void __launch_bounds__(kPixThreads)
    jpeg_pixels_kernel(const ryolo_jpeg_image* __restrict__ images, const uint8_t* __restrict__ area,
                       uint8_t* __restrict__ out) {
  const ryolo_jpeg_image& im = images[blockIdx.y];
  const int oy = blockIdx.x;
  if (oy >= im.out_h) return;
  uint8_t* o = out + im.out_off + (int64_t)oy * im.out_w * 3;
  for (int ox = threadIdx.x; ox < im.out_w; ox += kPixThreads) {
    uint8_t bgr[3];
    jpeg::pixel_bgr(im, area, ox, oy, bgr);
    o[3 * ox] = bgr[0], o[3 * ox + 1] = bgr[1], o[3 * ox + 2] = bgr[2];
  }
}

}  // namespace
}  // namespace ryolo

using namespace ryolo;

extern "C" size_t ryolo_jpeg_workspace_bytes(int nchunks, long long image_bytes) {
  if (nchunks < 0 || image_bytes < 0) return 0;
  uint8_t* area = nullptr;
  carve(nullptr, nchunks, &area);
  return (size_t)(area - (uint8_t*)nullptr) + (size_t)image_bytes;
}

extern "C" int ryolo_jpeg_decode(const ryolo_jpeg_image* images, int nimages, const ryolo_jpeg_segment* segs,
                                 int nsegs, const int32_t* chunk_seg, int nchunks, int chunk_bytes,
                                 const uint8_t* data, long long data_bytes, const ryolo_jpeg_huff* huff,
                                 const uint16_t* quant, int max_blocks, int max_out_h, uint8_t* out, int32_t* status,
                                 void* workspace, size_t workspace_bytes, long long image_bytes, int stages,
                                 void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(images && nimages > 0 && nimages <= 65535 && workspace && image_bytes >= 0);
  RYOLO_ARG_CHECK(stages >= 1 && stages <= (RYOLO_JPEG_ENTROPY | RYOLO_JPEG_PIXELS));
  RYOLO_ARG_CHECK(workspace_bytes >= ryolo_jpeg_workspace_bytes(nchunks, image_bytes));
  uint8_t* area = nullptr;
  const ChunkWs w = carve(workspace, nchunks, &area);
  if (stages & RYOLO_JPEG_ENTROPY) {
    RYOLO_ARG_CHECK(segs && nsegs > 0 && chunk_seg && nchunks >= nsegs && chunk_bytes >= 1 && data && huff && status);
    RYOLO_ARG_CHECK(data_bytes > 0 && data_bytes < ((long long)1 << 32) - 8);
    RYOLO_ARG_CHECK(nsegs <= 2147483647 / 32);
    RYOLO_CUDA_TRY(cudaMemsetAsync(status, 0, sizeof(int32_t) * nimages, stream));
    const int cgrid = (nchunks + kChunkThreads - 1) / kChunkThreads;
    jpeg_pass_a_kernel<<<cgrid, kChunkThreads, 0, stream>>>(images, segs, chunk_seg, nchunks, chunk_bytes, data, huff,
                                                            w);
    RYOLO_LAUNCH_CHECK();
    jpeg_pass_b_kernel<<<cgrid, kChunkThreads, 0, stream>>>(images, segs, chunk_seg, nchunks, chunk_bytes, data, huff,
                                                            w);
    RYOLO_LAUNCH_CHECK();
    jpeg_resolve_kernel<<<nsegs, 32, 0, stream>>>(images, segs, status, w);
    RYOLO_LAUNCH_CHECK();
    jpeg_write_kernel<<<cgrid, kChunkThreads, 0, stream>>>(images, segs, chunk_seg, nchunks, chunk_bytes, data, huff,
                                                           w, area, status);
    RYOLO_LAUNCH_CHECK();
    jpeg_dc_kernel<<<dim3(nsegs, 3), kDcThreads, 0, stream>>>(images, segs, area);
    RYOLO_LAUNCH_CHECK();
  }
  if (stages & RYOLO_JPEG_PIXELS) {
    RYOLO_ARG_CHECK(quant && out && status && max_blocks > 0 && max_out_h > 0);
    jpeg_idct_kernel<<<dim3((max_blocks + kIdctThreads - 1) / kIdctThreads, nimages), kIdctThreads, 0, stream>>>(
        images, quant, area, status);
    RYOLO_LAUNCH_CHECK();
    jpeg_pixels_kernel<<<dim3(max_out_h, nimages), kPixThreads, 0, stream>>>(images, area, out);
    RYOLO_LAUNCH_CHECK();
  }
  return RYOLO_OK;
}
