// Dense part of compute_loss (SURVEY.md 8 row a6, reference model/loss.py:340-348): the objectness term
// BCEWithLogitsLoss(pos_weight)(pi[..., 5], tobj) runs over EVERY cell of the three head maps (64 x 72 x (19^2 + 38^2 +
// 76^2) = 35 M cells per step).  Written as framework element-wise ops it costs ~20 passes over strided views of the head
// tensors (forward + autograd) plus a permute copy each way; its HBM bound at batch 64 is ~0.5 ms (8 B read per cell
// forward, 8 B read + the 7-channel fp32 cotangent written backward; DESIGN.md section 8 has the measured kernel times).
// Here: one kernel for the loss sum,
// one kernel that writes the WHOLE head cotangent (objectness channel = d(loss)/dx, every other channel zero; the few
// matched rows are scattered on top by the caller), both reading the head tensor through its strides so that the NCHW
// buffer the head convolution wrote is consumed in place (no permute().contiguous() copy), and a transposing
// NCHW fp32 -> padded-NHWC bf16 pass for the cotangent on its way into the head convolutions' dgrad / wgrad.
//
// BCE with logits, PyTorch's formulation (aten/native/Loss.cpp binary_cross_entropy_with_logits):
//   lw = 1 + (pos_weight - 1) t;   l = (1 - t) x + lw (log1p(exp(-|x|)) + max(-x, 0));   dl/dx = (1 - t) + lw (sigmoid(x) - 1)
// Focal form (arcs with 'F', reference model/loss.py:126-146: FocalLoss(BCEobj, gamma), alpha = 1), per cell:
//   base = 1.000001f - exp(-l) = (1.000001f - 1) - expm1(-l)   (>= 9.5e-7: the expm1 form does not cancel for small l)
//   lf = l base^gamma;   dlf/dx = dl/dx (base^gamma + gamma l exp(-l) base^(gamma - 1))
// gamma = 0 gives the BCE bits (pow(base, 0) = 1, the second term is 0).  The same two kernels serve both forms through
// the FOCAL template flag; the BCE instantiation compiles to the code it had before the flag existed.
#include <cuda_bf16.h>

#include "common.cuh"

namespace ryolo {

struct HeadView {            // logical [B, na, ny, nx, no] tensor with arbitrary element strides
  long long sb, sa, sy, sx, sc;
  int B, na, ny, nx, no;
  int cells32;                 // B * na * ny * nx < 2^31: cell_offset divides by multiply + shift
  FastDiv fx, fy, fa;
};

__device__ __forceinline__ size_t cell_offset(const HeadView& v, size_t cell) {
  if (v.cells32) {
    int r, x, y, a, b;
    fast_divmod((int)cell, v.fx, r, x);
    fast_divmod(r, v.fy, r, y);
    fast_divmod(r, v.fa, b, a);
    return (size_t)(b * v.sb + a * v.sa + y * v.sy + x * v.sx);
  }
  const int x = (int)(cell % v.nx);
  size_t r = cell / v.nx;
  const int y = (int)(r % v.ny);
  r /= v.ny;
  const int a = (int)(r % v.na);
  const int b = (int)(r / v.na);
  return (size_t)(b * v.sb + a * v.sa + y * v.sy + x * v.sx);
}

// 1.000001f - 1 (= 2^-20): the reference's constant as the fp32 arithmetic of its focal factor sees it
constexpr float FOCAL_EPS = 1.000001f - 1.f;
// base of the focal factor; l >= 0 for targets in [0, 1], the clamp keeps base >= FOCAL_EPS when rounding says otherwise
__device__ __forceinline__ float focal_base(float l) { return FOCAL_EPS - expm1f(-fmaxf(l, 0.f)); }

// gamma is the last parameter so that the BCE instantiation (which never reads it) keeps its parameter layout
template <bool FOCAL>
__global__ void __launch_bounds__(256) obj_bce_fwd_kernel(const float* __restrict__ x, HeadView v, int ch,
                                                          const float* __restrict__ tobj, float pw,
                                                          double* __restrict__ partials /*[gridDim.x]*/, float gamma) {
  const size_t n = (size_t)v.B * v.na * v.ny * v.nx;
  double acc = 0.0;
  for (size_t cell = (size_t)blockIdx.x * blockDim.x + threadIdx.x; cell < n; cell += (size_t)gridDim.x * blockDim.x) {
    const float xv = x[cell_offset(v, cell) + (size_t)ch * v.sc];
    const float t = tobj[cell];
    const float lw = 1.f + (pw - 1.f) * t;
    float l = (1.f - t) * xv + lw * (log1pf(expf(-fabsf(xv))) + fmaxf(-xv, 0.f));
    if (FOCAL) l *= powf(focal_base(l), gamma);
    acc += (double)l;
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ double part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < 8; w++) s += part[w];
    partials[blockIdx.x] = s;
  }
}
// *out += the CTA partials, added in a fixed order (lane l takes partials l, l + 32, ...; then a fixed butterfly)
__global__ void __launch_bounds__(32) ordered_sum_add_kernel(const double* __restrict__ partials, int n, double* __restrict__ out) {
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += 32) s += partials[i];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (threadIdx.x == 0) *out += s;
}
// out[j] += the column j of rows x n partials, added in a fixed order: thread (column, part q) takes rows q, q + 8, ...,
// then the 8 parts in order.  CTA = 32 columns.
__global__ void __launch_bounds__(256) ordered_rows_add_kernel(const float* __restrict__ partials, int rows, int n,
                                                               float* __restrict__ out) {
  __shared__ float s_part[8][32];
  const int lane = threadIdx.x & 31, q = threadIdx.x >> 5, j = blockIdx.x * 32 + lane;
  float s = 0.f;
  if (j < n) {
#pragma unroll 4
    for (int r = q; r < rows; r += 8) s += __ldcg(partials + (size_t)r * n + j);
  }
  s_part[q][lane] = s;
  __syncthreads();
  if (q == 0 && j < n) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; k++) t += s_part[k][lane];
    out[j] += t;
  }
}

// g[cell, k] = k == ch ? scale * dl/dx : 0, for every channel k (g has the strides of the head tensor); FOCAL: dlf/dx
template <bool FOCAL>
__global__ void __launch_bounds__(256) obj_bce_bwd_kernel(const float* __restrict__ x, HeadView v, int ch,
                                                          const float* __restrict__ tobj, float pw,
                                                          const float* __restrict__ scale_dev, float* __restrict__ g,
                                                          float gamma) {
  const size_t n = (size_t)v.B * v.na * v.ny * v.nx;
  const float scale = __ldg(scale_dev);
  for (size_t cell = (size_t)blockIdx.x * blockDim.x + threadIdx.x; cell < n; cell += (size_t)gridDim.x * blockDim.x) {
    const size_t off = cell_offset(v, cell);
    const float xv = x[off + (size_t)ch * v.sc];
    const float t = tobj[cell];
    const float lw = 1.f + (pw - 1.f) * t;
    const float sg = 1.f / (1.f + expf(-xv));
    float d;
    if (FOCAL) {
      const float l = (1.f - t) * xv + lw * (log1pf(expf(-fabsf(xv))) + fmaxf(-xv, 0.f));
      const float base = focal_base(l);
      const float pg = powf(base, gamma);
      const float fac = pg + gamma * l * expf(-l) * (pg / base);     // base^(gamma - 1) = base^gamma / base
      d = scale * (((1.f - t) + lw * (sg - 1.f)) * fac);
    } else {
      d = scale * ((1.f - t) + lw * (sg - 1.f));
    }
    for (int k = 0; k < v.no; k++) g[off + (size_t)k * v.sc] = k == ch ? d : 0.f;
  }
}

// NCHW fp32 [B, C, ny, nx] -> padded-NHWC bf16 (channel stride dcs), plus the per-channel sums of g (the head convolution's
// bias gradient) on the way.  One block = one image row: chunks of 32 consecutive x, 8 channels per warp and step (eight
// 128-byte coalesced loads in flight per warp), transposed through shared memory with 16-byte stores whose row pitch is an
// odd number of 16-byte units (conflict-free), 16-byte global stores of each pixel's contiguous channels.
__device__ __forceinline__ size_t pad_off(int b, int y, int x, int h, int w, int cs) {
  return (((size_t)b * (h + 2) + y + 1) * (w + 2) + x + 1) * cs;
}
// sum over the 32 lanes of 8 per-lane values in 9 shuffles (halving exchange instead of 8 x 5 butterflies): on return
// lanes 0, 4, .., 28 hold the total of value index lane / 4
__device__ __forceinline__ float warp_sum8(const float* v, int lane) {
  float a[4], b2[2], c1;
  const bool h16 = lane & 16, h8 = lane & 8, h4 = lane & 4;
#pragma unroll
  for (int e = 0; e < 4; e++) {
    const float send = h16 ? v[e] : v[e + 4], keep = h16 ? v[e + 4] : v[e];
    a[e] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
  }
#pragma unroll
  for (int e = 0; e < 2; e++) {
    const float send = h8 ? a[e] : a[e + 2], keep = h8 ? a[e + 2] : a[e];
    b2[e] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
  {
    const float send = h4 ? b2[0] : b2[1], keep = h4 ? b2[1] : b2[0];
    c1 = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
  c1 += __shfl_xor_sync(0xffffffffu, c1, 2);
  c1 += __shfl_xor_sync(0xffffffffu, c1, 1);
  return c1;   // value index = 4 * (lane bit 4) + 2 * (lane bit 3) + (lane bit 2)
}

// STORE = false: the bias sums only (the same loads, warp sums and row partials, so the same bits), no dst traffic
template <bool STORE>
__global__ void __launch_bounds__(256) head_grad_nchw_kernel(const float* __restrict__ g, int c, int ny, int nx,
                                                             __nv_bfloat16* __restrict__ dst, int dcs,
                                                             float* __restrict__ bias_partials /*[blocks][c]*/,
                                                             int rows_per_block) {
  float* const bias_grad = bias_partials;   // null: no bias gradient
  extern __shared__ __align__(16) unsigned char hg_smem[];
  const int c8 = (c + 7) & ~7;
  const int cpad = c8 + ((c8 >> 3) & 1 ? 0 : 8);                      // pitch = odd multiple of 16 bytes
  __nv_bfloat16* tile = reinterpret_cast<__nv_bfloat16*>(hg_smem);   // [32][cpad]
  float* s_bias = reinterpret_cast<float*>(hg_smem + (STORE ? (size_t)32 * cpad * 2 : 0));   // [c8]: one warp per channel
  const int b = blockIdx.y;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < c8; i += 256) s_bias[i] = 0.f;
  __syncthreads();
  const size_t plane = (size_t)ny * nx;
  const int y_end = min(ny, (int)(blockIdx.x + 1) * rows_per_block);
  for (int y = blockIdx.x * rows_per_block; y < y_end; y++) {
    const float* grow = g + ((size_t)b * c * ny + y) * nx;
    for (int x0 = 0; x0 < nx; x0 += 32) {
      const int npx = min(32, nx - x0);
#pragma unroll 1
      for (int ch0 = wid * 8; ch0 < c8; ch0 += 64) {
        float v[8];
#pragma unroll
        for (int e = 0; e < 8; e++) v[e] = (lane < npx && ch0 + e < c) ? __ldg(grow + (size_t)(ch0 + e) * plane + x0 + lane) : 0.f;
        if (STORE) {
          __nv_bfloat162 h[4];
#pragma unroll
          for (int e = 0; e < 4; e++) h[e] = __floats2bfloat162_rn(v[2 * e], v[2 * e + 1]);
          *reinterpret_cast<uint4*>(tile + lane * cpad + ch0) = *reinterpret_cast<uint4*>(h);
        }
        if (bias_grad) {
          const float t = warp_sum8(v, lane);
          if ((lane & 3) == 0) s_bias[ch0 + (lane >> 2)] += t;
        }
      }
      if (!STORE) continue;
      __syncthreads();
      const int chunks = c >> 3;
      for (int idx = threadIdx.x; idx < npx * chunks; idx += 256) {
        const int px = idx / chunks, k = idx - px * chunks;
        *reinterpret_cast<uint4*>(dst + pad_off(b, y, x0 + px, ny, nx, dcs) + k * 8) =
            *reinterpret_cast<const uint4*>(tile + px * cpad + k * 8);
      }
      const int tail = c & 7;
      for (int idx = threadIdx.x; idx < npx * tail; idx += 256) {
        const int px = idx / tail, e = (c & ~7) + idx % tail;
        dst[pad_off(b, y, x0 + px, ny, nx, dcs) + e] = tile[px * cpad + e];
      }
      __syncthreads();
    }
  }
  if (!STORE) __syncthreads();   // s_bias[ch] is written by one warp and read below by another thread
  if (bias_grad)   // this block's row of per-channel sums; ordered_rows_add_kernel adds the rows in a fixed order
    for (int i = threadIdx.x; i < c; i += 256)
      bias_partials[(size_t)(blockIdx.y * gridDim.x + blockIdx.x) * c + i] = s_bias[i];
}

// The matched (anchor, target) rows of compute_loss: gather of the head values at (b, a, gj, gi), the objectness targets,
// and the scatter of the rows' gradients -- three tiny kernels instead of framework advanced indexing (each index op there
// launches ~6 kernels: bounds reductions, asserts, the op itself).  Rows whose indices fall outside the map (a target on
// the right / bottom border, where the reference raises an IndexError) and rows with mask == 0 read as 0 / write nothing.
struct RowIdx {
  const long long *b, *a, *gj, *gi;
  const unsigned char* mask;
  int rows;
};
__device__ __forceinline__ bool row_cell(const RowIdx& r, const HeadView& v, int i, size_t* off, size_t* cell) {
  if (!r.mask[i]) return false;
  const long long b = r.b[i], a = r.a[i], y = r.gj[i], x = r.gi[i];
  if (b < 0 || b >= v.B || a < 0 || a >= v.na || y < 0 || y >= v.ny || x < 0 || x >= v.nx) return false;
  *off = (size_t)(b * v.sb + a * v.sa + y * v.sy + x * v.sx);
  *cell = (((size_t)b * v.na + a) * v.ny + y) * v.nx + x;
  return true;
}
__global__ void rows_gather_kernel(const float* __restrict__ x, HeadView v, RowIdx r, float* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= r.rows * v.no) return;
  const int i = t / v.no, k = t - i * v.no;
  size_t off, cell;
  out[t] = row_cell(r, v, i, &off, &cell) ? x[off + (size_t)k * v.sc] : 0.f;
}
// Several rows may name the same cell (targets sharing a grid cell and anchor).  Their gradients are added in ROW order
// by the first row of the cell, so that the sum is the same every run: keys[i] = the cell of row i (~0 for rows that
// write nothing), then one WARP per row: a live row looks for an earlier row of its cell, 128 keys per step (four
// independent coalesced loads, one ballot each); the row that finds none owns the cell and walks the keys from itself to
// the end the same way, and for every row j of the cell, in increasing j, lane k adds vals[j, k] * scale to channel k:
//   g[cell, k] = fmaf(vals[jn, k], scale, ... fmaf(vals[j1, k], scale, g[cell, k]))
// A live row reads at most R keys wherever it sits; all `no` channels ride on one walk (one walk per 32 channels).
constexpr int SCATTER_UNROLL = 4;
__global__ void rows_key_kernel(HeadView v, RowIdx r, unsigned long long* __restrict__ keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= r.rows) return;
  size_t off, cell;
  keys[i] = row_cell(r, v, i, &off, &cell) ? (unsigned long long)cell : ~0ull;
}
// bit u * 32 + l of the result: keys[j0 + u * 32 + l] == key and j0 + u * 32 + l < end (lanes agree on the result)
__device__ __forceinline__ void match_keys(const unsigned long long* __restrict__ keys, int j0, int end,
                                           unsigned long long key, int lane, unsigned (&m)[SCATTER_UNROLL]) {
  unsigned long long k[SCATTER_UNROLL];
#pragma unroll
  for (int u = 0; u < SCATTER_UNROLL; u++) {
    const int j = j0 + u * 32 + lane;
    k[u] = j < end ? __ldg(keys + j) : ~0ull;
  }
#pragma unroll
  for (int u = 0; u < SCATTER_UNROLL; u++) m[u] = __ballot_sync(0xffffffffu, k[u] == key);
}
__global__ void __launch_bounds__(256) rows_scatter_add_kernel(float* __restrict__ g, HeadView v, RowIdx r,
                                                               const unsigned long long* __restrict__ keys,
                                                               const float* __restrict__ vals,
                                                               const float* __restrict__ scale_dev) {
  const int i = (int)(((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= r.rows) return;
  const unsigned long long key = __ldg(keys + i);
  if (key == ~0ull) return;
  unsigned m[SCATTER_UNROLL];
  for (int j0 = 0; j0 < i; j0 += 32 * SCATTER_UNROLL) {
    match_keys(keys, j0, i, key, lane, m);
    unsigned any = 0u;
#pragma unroll
    for (int u = 0; u < SCATTER_UNROLL; u++) any |= m[u];
    if (any) return;                                  // an earlier row owns this cell
  }
  size_t off, cell;
  row_cell(r, v, i, &off, &cell);
  const float scale = __ldg(scale_dev);
  for (int k0 = 0; k0 < v.no; k0 += 32) {
    const int k = k0 + lane;
    float* const gk = g + off + (size_t)k * v.sc;
    float acc = k < v.no ? *gk : 0.f;
    for (int j0 = i; j0 < r.rows; j0 += 32 * SCATTER_UNROLL) {
      match_keys(keys, j0, r.rows, key, lane, m);
#pragma unroll
      for (int u = 0; u < SCATTER_UNROLL; u++) {
        for (unsigned bits = m[u]; bits; bits &= bits - 1) {
          const int j = j0 + u * 32 + __ffs(bits) - 1;
          if (k < v.no) acc = fmaf(__ldg(vals + (size_t)j * v.no + k), scale, acc);
        }
      }
    }
    if (k < v.no) *gk = acc;
  }
}
__global__ void rows_set_tobj_kernel(float* __restrict__ tobj, HeadView v, RowIdx r) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= r.rows) return;
  size_t off, cell;
  if (row_cell(r, v, i, &off, &cell)) tobj[cell] = 1.f;
}

static inline int loss_grid(size_t n) {
  const size_t want = (n + 255) / 256;
  const size_t cap = (size_t)device_sm_count() * 8;
  return (int)(want < cap ? (want ? want : 1) : cap);
}

}  // namespace ryolo

using namespace ryolo;

static inline bool mk_view(const long long* strides, int batch, int na, int ny, int nx, int no, HeadView* v) {
  if (!strides || batch <= 0 || na <= 0 || ny <= 0 || nx <= 0 || no <= 0) return false;
  for (int i = 0; i < 5; i++)
    if (strides[i] < 0) return false;
  v->sb = strides[0]; v->sa = strides[1]; v->sy = strides[2]; v->sx = strides[3]; v->sc = strides[4];
  v->B = batch; v->na = na; v->ny = ny; v->nx = nx; v->no = no;
  v->cells32 = (long long)batch * na * ny * nx < (1ll << 31);
  v->fx = make_fastdiv(nx); v->fy = make_fastdiv(ny); v->fa = make_fastdiv(na);
  return true;
}

template <bool FOCAL>
static int obj_fwd(const float* x, const long long* strides, int batch, int na, int ny, int nx, int no, int ch,
                   const float* tobj, float pos_weight, float gamma, double* sum_out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  HeadView v;
  RYOLO_ARG_CHECK(x && tobj && sum_out && mk_view(strides, batch, na, ny, nx, no, &v) && ch >= 0 && ch < no);
  const size_t n = (size_t)batch * na * ny * nx;
  const int grid = loss_grid(n);
  double* partials = static_cast<double*>(stream_scratch(stream, SCRATCH_LOSS, (size_t)grid * sizeof(double)));
  if (!partials) return RYOLO_E_CUDA;
  obj_bce_fwd_kernel<FOCAL><<<grid, 256, 0, stream>>>(x, v, ch, tobj, pos_weight, partials, gamma);
  RYOLO_LAUNCH_CHECK();
  ordered_sum_add_kernel<<<1, 32, 0, stream>>>(partials, grid, sum_out);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

template <bool FOCAL>
static int obj_bwd(const float* x, const long long* strides, int batch, int na, int ny, int nx, int no, int ch,
                   const float* tobj, float pos_weight, float gamma, const float* scale_dev, float* grad, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  HeadView v;
  RYOLO_ARG_CHECK(x && tobj && scale_dev && grad && mk_view(strides, batch, na, ny, nx, no, &v) && ch >= 0 && ch < no);
  const size_t n = (size_t)batch * na * ny * nx;
  obj_bce_bwd_kernel<FOCAL><<<loss_grid(n), 256, 0, stream>>>(x, v, ch, tobj, pos_weight, scale_dev, grad, gamma);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_obj_bce_fwd(const float* x, const long long* strides, int batch, int na, int ny, int nx, int no, int ch,
                                 const float* tobj, float pos_weight, double* sum_out, void* stream_) {
  return obj_fwd<false>(x, strides, batch, na, ny, nx, no, ch, tobj, pos_weight, 0.f, sum_out, stream_);
}

extern "C" int ryolo_obj_bce_bwd(const float* x, const long long* strides, int batch, int na, int ny, int nx, int no, int ch,
                                 const float* tobj, float pos_weight, const float* scale_dev, float* grad, void* stream_) {
  return obj_bwd<false>(x, strides, batch, na, ny, nx, no, ch, tobj, pos_weight, 0.f, scale_dev, grad, stream_);
}

extern "C" int ryolo_obj_focal_fwd(const float* x, const long long* strides, int batch, int na, int ny, int nx, int no,
                                   int ch, const float* tobj, float pos_weight, float gamma, double* sum_out, void* stream_) {
  RYOLO_ARG_CHECK(gamma >= 0.f && gamma < INFINITY);
  return obj_fwd<true>(x, strides, batch, na, ny, nx, no, ch, tobj, pos_weight, gamma, sum_out, stream_);
}

extern "C" int ryolo_obj_focal_bwd(const float* x, const long long* strides, int batch, int na, int ny, int nx, int no,
                                   int ch, const float* tobj, float pos_weight, float gamma, const float* scale_dev,
                                   float* grad, void* stream_) {
  RYOLO_ARG_CHECK(gamma >= 0.f && gamma < INFINITY);
  return obj_bwd<true>(x, strides, batch, na, ny, nx, no, ch, tobj, pos_weight, gamma, scale_dev, grad, stream_);
}

// dst null: the bias sums only (head_grad_nchw_kernel<false>, no tile in shared memory); same grid, so the same bits
static int head_grad_nchw(const float* g, int batch, int c, int ny, int nx, void* dst, int dst_cstride, float* bias_grad,
                          cudaStream_t stream) {
  const int c8 = (c + 7) & ~7;
  const int cpad = c8 + ((c8 >> 3) & 1 ? 0 : 8);
  const size_t smem = (dst ? (size_t)32 * cpad * 2 : 0) + (size_t)c8 * sizeof(float);
  // rows per block: keep ~2k blocks in the grid (one row of c bias partials per block)
  int rpb = (int)(((long long)ny * batch + 2047) / 2048);
  if (rpb < 1) rpb = 1;
  dim3 grid((unsigned)((ny + rpb - 1) / rpb), (unsigned)batch);
  const int blocks = (int)(grid.x * grid.y);
  float* partials = nullptr;
  if (bias_grad) {
    partials = static_cast<float*>(stream_scratch(stream, SCRATCH_LOSS, (size_t)blocks * c * sizeof(float)));
    if (!partials) return RYOLO_E_CUDA;
  }
  if (dst) {
    RYOLO_SMEM_OPT_IN(head_grad_nchw_kernel<true>, 160 * 1024);
    head_grad_nchw_kernel<true><<<grid, 256, smem, stream>>>(g, c, ny, nx, static_cast<__nv_bfloat16*>(dst), dst_cstride,
                                                             partials, rpb);
  } else {
    head_grad_nchw_kernel<false><<<grid, 256, smem, stream>>>(g, c, ny, nx, nullptr, 0, partials, rpb);
  }
  RYOLO_LAUNCH_CHECK();
  if (bias_grad) {
    ordered_rows_add_kernel<<<(c + 31) / 32, 256, 0, stream>>>(partials, blocks, c, bias_grad);
    RYOLO_LAUNCH_CHECK();
  }
  return RYOLO_OK;
}

extern "C" int ryolo_head_grad_nchw_to_padded(const float* g, int batch, int c, int ny, int nx, void* dst, int dst_cstride,
                                              float* bias_grad, void* stream_) {
  RYOLO_ARG_CHECK(g && dst && batch > 0 && c > 0 && ny > 0 && nx > 0);
  RYOLO_ARG_CHECK(dst_cstride >= c && dst_cstride % 8 == 0 && batch <= 65535 && c <= 2048);
  return head_grad_nchw(g, batch, c, ny, nx, dst, dst_cstride, bias_grad, static_cast<cudaStream_t>(stream_));
}

extern "C" int ryolo_head_bias_grad(const float* g, int batch, int c, int ny, int nx, float* bias_grad, void* stream_) {
  RYOLO_ARG_CHECK(g && bias_grad && batch > 0 && c > 0 && ny > 0 && nx > 0 && batch <= 65535 && c <= 2048);
  return head_grad_nchw(g, batch, c, ny, nx, nullptr, 0, bias_grad, static_cast<cudaStream_t>(stream_));
}

static inline RowIdx mk_rows(const long long* b, const long long* a, const long long* gj, const long long* gi,
                             const unsigned char* mask, int rows) {
  RowIdx r;
  r.b = b; r.a = a; r.gj = gj; r.gi = gi; r.mask = mask; r.rows = rows;
  return r;
}

extern "C" int ryolo_loss_rows_gather(const float* x, const long long* strides, int batch, int na, int ny, int nx, int no,
                                      const long long* b, const long long* a, const long long* gj, const long long* gi,
                                      const unsigned char* mask, int rows, float* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  HeadView v;
  RYOLO_ARG_CHECK(rows >= 0 && mk_view(strides, batch, na, ny, nx, no, &v));
  if (rows == 0) return RYOLO_OK;
  RYOLO_ARG_CHECK(x && b && a && gj && gi && mask && out);
  rows_gather_kernel<<<(rows * no + 255) / 256, 256, 0, stream>>>(x, v, mk_rows(b, a, gj, gi, mask, rows), out);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_loss_rows_scatter_add(float* grad, const long long* strides, int batch, int na, int ny, int nx, int no,
                                           const long long* b, const long long* a, const long long* gj, const long long* gi,
                                           const unsigned char* mask, int rows, const float* vals, const float* scale_dev,
                                           void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  HeadView v;
  RYOLO_ARG_CHECK(rows >= 0 && mk_view(strides, batch, na, ny, nx, no, &v));
  if (rows == 0) return RYOLO_OK;
  RYOLO_ARG_CHECK(grad && b && a && gj && gi && mask && vals && scale_dev);
  unsigned long long* keys =
      static_cast<unsigned long long*>(stream_scratch(stream, SCRATCH_LOSS_KEYS, (size_t)rows * sizeof(unsigned long long)));
  if (!keys) return RYOLO_E_CUDA;
  const RowIdx ri = mk_rows(b, a, gj, gi, mask, rows);
  rows_key_kernel<<<(rows + 255) / 256, 256, 0, stream>>>(v, ri, keys);
  RYOLO_LAUNCH_CHECK();
  rows_scatter_add_kernel<<<(unsigned)(((size_t)rows * 32 + 255) / 256), 256, 0, stream>>>(grad, v, ri, keys, vals, scale_dev);
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}

extern "C" int ryolo_loss_rows_set_tobj(float* tobj, int batch, int na, int ny, int nx, const long long* b, const long long* a,
                                        const long long* gj, const long long* gi, const unsigned char* mask, int rows,
                                        void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  RYOLO_ARG_CHECK(rows >= 0 && batch > 0 && na > 0 && ny > 0 && nx > 0);
  if (rows == 0) return RYOLO_OK;
  RYOLO_ARG_CHECK(tobj && b && a && gj && gi && mask);
  HeadView v;
  v.sb = v.sa = v.sy = v.sx = v.sc = 0;
  v.B = batch; v.na = na; v.ny = ny; v.nx = nx; v.no = 1;
  v.cells32 = 0;
  v.fx = v.fy = v.fa = make_fastdiv(1);
  rows_set_tobj_kernel<<<(rows + 255) / 256, 256, 0, stream>>>(tobj, v, mk_rows(b, a, gj, gi, mask, rows));
  RYOLO_LAUNCH_CHECK();
  return RYOLO_OK;
}
