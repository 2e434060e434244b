// Restores the zero invariants of padded-NHWC buffers that live in a shared activation pool (pool.py).  A plan's
// buffers promise a zero halo (no kernel writes it; the 3x3 taps and the TMA boxes read it as the conv padding) and zero
// channels [c_real, c_stride) wherever no kernel writes them (the GEMM k-steps read them against zero weight rows).  When
// the storage was last used by a plan of another shape, both hold that plan's bytes.  One launch walks a job table
// (device memory, built once per plan): grid.y = job, the block strides over that job's 16-byte units -- every channel
// chunk of the ring pixels, and the chunks of [c_real, c_stride) of the interior pixels.  The interior's real channels
// are left alone: every step writes them before it reads them.
#include <cuda_bf16.h>

#include "common.cuh"

namespace ryolo {

__global__ void __launch_bounds__(256) zero_halo_multi_kernel(const ryolo_halo_job* __restrict__ jobs) {
  const ryolo_halo_job jb = jobs[blockIdx.y];
  const long long hp = jb.h + 2, wp = jb.w + 2;
  const long long chunks = jb.c_stride / 8;                    // 16-byte units per pixel
  const int lo = jb.c_real < jb.c_stride ? jb.c_real : jb.c_stride;
  const long long lo_chunk = lo / 8;                           // first interior unit (may be partly real)
  const long long ring_px = 2 * wp + 2 * (long long)jb.h;      // per image
  const long long ring_units = (long long)jb.batch * ring_px * chunks;
  const long long int_units = lo < jb.c_stride ? (long long)jb.batch * jb.h * jb.w * (chunks - lo_chunk) : 0;
  __nv_bfloat16* base = static_cast<__nv_bfloat16*>(jb.ptr);
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
  for (long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x; u < ring_units + int_units;
       u += (long long)gridDim.x * blockDim.x) {
    long long px, cu;
    if (u < ring_units) {
      cu = u % chunks;
      const long long p = u / chunks, b = p / ring_px, q = p - b * ring_px;
      long long y, x;
      if (q < wp) {
        y = 0, x = q;
      } else if (q < 2 * wp) {
        y = hp - 1, x = q - wp;
      } else {
        const long long r = q - 2 * wp;
        y = 1 + r / 2, x = (r & 1) ? wp - 1 : 0;
      }
      px = (b * hp + y) * wp + x;
      reinterpret_cast<uint4*>(base + px * jb.c_stride)[cu] = z;
      continue;
    }
    const long long v = u - ring_units, per = chunks - lo_chunk;
    cu = lo_chunk + v % per;
    const long long p = v / per, b = p / ((long long)jb.h * jb.w), r = p - b * (long long)jb.h * jb.w;
    px = (b * hp + 1 + r / jb.w) * wp + 1 + r % jb.w;
    __nv_bfloat16* dst = base + px * jb.c_stride + cu * 8;
    if (cu * 8 >= lo) {
      *reinterpret_cast<uint4*>(dst) = z;
    } else {                                                   // the chunk that straddles c_real: its pad lanes only
      for (int e = lo - (int)(cu * 8); e < 8; e++) dst[e] = __float2bfloat16_rn(0.f);
    }
  }
}

}  // namespace ryolo

using namespace ryolo;

extern "C" int ryolo_zero_halo_multi(const ryolo_halo_job* jobs_dev, int njobs, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(jobs_dev && njobs > 0 && njobs <= 65535);
  zero_halo_multi_kernel<<<dim3(128, njobs), 256, 0, stream>>>(jobs_dev);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}
