// resample.cu -- windowed-sinc polyphase resampling of [rows, T] waveforms on sm_90a.
//
// Replaces julius.resample_frac as called by AudioSignal.resample (ref:audiotools/core/audio_signal.py:716-736):
// with old/new the gcd-reduced rates and K = 2*width + old taps per output phase,
//     out[m*new + i] = sum_k kernel[i][k] * x[clamp(m*old + k - width, 0, T-1)],   i in [0,new), m >= 0
// (replicate padding, one strided correlation per phase, phases interleaved, first floor(new*T/old)
// samples kept).  The per-phase kernels come in transposed [K][new] so that consecutive output samples
// (consecutive phases) read consecutive taps.
//
// One CTA produces OUT_PER_CTA consecutive output samples of one row: the input span they touch
// ((frames-1)*old + K samples) is staged once in shared memory (edge replicate resolved there), then every
// thread accumulates 4 outputs over the K taps in FP32.  Algorithmic traffic: read x once, write out once.
#include "b2a_common.h"

namespace b2a {
namespace resample {

constexpr int THREADS = 256;
constexpr int OPT = 4;                       // outputs per thread
constexpr int OUT_PER_CTA = THREADS * OPT;   // 1024

__global__ void __launch_bounds__(THREADS)
resample_kernel(const float* __restrict__ x, float* __restrict__ out, const float* __restrict__ kt, int T,
                int64_t out_len, int old_, int new_, int width, int K, int tiles_per_row, int span_max) {
  B2A_DYN_SMEM(smem);
  float* xs = reinterpret_cast<float*>(smem);
  const int row = blockIdx.x / tiles_per_row, tile = blockIdx.x - row * tiles_per_row;
  const int64_t o0 = (int64_t)tile * OUT_PER_CTA;          // first output sample of this CTA
  const int m0 = (int)(o0 / new_);                          // first frame touched
  const int64_t o_end = min(o0 + OUT_PER_CTA, out_len);
  const int m1 = (int)((o_end - 1) / new_);                 // last frame touched
  const int span = (m1 - m0) * old_ + K;
  const float* xr = x + (size_t)row * (size_t)T;
  const int base = m0 * old_ - width;                       // x-coordinate of xs[0]
  for (int i = threadIdx.x; i < span; i += THREADS) {
    int u = base + i;
    u = u < 0 ? 0 : (u > T - 1 ? T - 1 : u);                // replicate padding
    xs[i] = __ldg(xr + u);
  }
  __syncthreads();
  float acc[OPT];
  int xo[OPT], ph[OPT];
#pragma unroll
  for (int j = 0; j < OPT; ++j) {
    const int64_t o = o0 + threadIdx.x + (int64_t)THREADS * j;
    const int m = (int)(o / new_);
    ph[j] = (int)(o - (int64_t)m * new_);
    xo[j] = (m - m0) * old_;
    if (o >= o_end) { xo[j] = 0; ph[j] = 0; }
    acc[j] = 0.f;
  }
  for (int k = 0; k < K; ++k) {
    const float* kr = kt + (size_t)k * new_;
#pragma unroll
    for (int j = 0; j < OPT; ++j) acc[j] = fmaf(__ldg(kr + ph[j]), xs[xo[j] + k], acc[j]);
  }
  float* orow = out + (size_t)row * (size_t)out_len;
#pragma unroll
  for (int j = 0; j < OPT; ++j) {
    const int64_t o = o0 + threadIdx.x + (int64_t)THREADS * j;
    if (o < o_end) orow[o] = acc[j];
  }
}

// ---------------------------------------------------------------------------------------------
// Backward (adjoint of the forward above, either route).  With u = q*old + r (input phase r) and k = u + width - m*old,
//     gx_ext[u] = sum_j sum_i kt[r + width + j*old][i] * g[(q - j)*new + i],   0 <= r + width + j*old < K,
// g zero outside [0, out_len): every input of one phase reads the same ~(K/old)*new taps.  One CTA takes QT
// consecutive q for every phase r; the g frames [q0 - JM, q0 + QT + JM) are staged in shared memory with an odd
// row stride (lanes of a warp, consecutive q, hit distinct banks); a work item is (phase, 64 consecutive q), a warp
// holds one item at a time, so its taps are broadcast loads and each lane accumulates two q 32 apart.  When the frames
// of a large new rate do not fit shared memory, the phase index i is tiled (IC at a time): each tile is staged in turn
// and the same thread adds its partial sums to the gradient it wrote for the previous tile (fixed order).
// The interior kernel writes gx[1 .. T-2]; gx[0] and gx[T-1] take the replicate fold of every extended position
// u < 1 resp. u > T-2 (bwd_edge_kernel).  Every sum runs in a fixed order.
// ---------------------------------------------------------------------------------------------
constexpr int BWD_Q = 64;  // q per work item (two per lane)

__global__ void __launch_bounds__(THREADS)
resample_bwd_kernel(const float* __restrict__ g, float* __restrict__ gx, const float* __restrict__ kt, int T,
                    int64_t out_len, int old_, int new_, int width, int JM, int QT, int IC, int NS,
                    int tiles_per_row) {
  B2A_DYN_SMEM(smem);
  float* gs = reinterpret_cast<float*>(smem);  // [QT + 2 JM][NS]: phases [i0, i0 + IC) of the frames
  const int row = blockIdx.x / tiles_per_row, tile = blockIdx.x - row * tiles_per_row;
  const int q0 = tile * QT;
  const int FS = QT + 2 * JM;
  const float* gr = g + (size_t)row * (size_t)out_len;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int chunks = QT / BWD_Q;
  float* gxr = gx + (size_t)row * (size_t)T;
  for (int i0 = 0; i0 < new_; i0 += IC) {
    const int ni = min(IC, new_ - i0);
    if (i0 > 0) __syncthreads();  // every warp is done with the previous tile
    for (int e = threadIdx.x; e < FS * ni; e += THREADS) {
      const int f = e / ni, i = e - f * ni;
      const int64_t m = (int64_t)q0 - JM + f, o = m * new_ + i0 + i;
      gs[f * NS + i] = (m >= 0 && o < out_len) ? __ldg(gr + o) : 0.f;
    }
    __syncthreads();
    for (int item = warp; item < old_ * chunks; item += THREADS / 32) {
      const int r = item / chunks, c = item - r * chunks;
      const int ql = c * BWD_Q + lane;  // q - q0 of the first accumulator; the second is ql + 32
      const int jlo = -((r + width) / old_), jhi = (width + old_ - 1 - r) / old_;
      float a0 = 0.f, a1 = 0.f;
      for (int j = jlo; j <= jhi; ++j) {
        const float* kr = kt + (size_t)(r + width + j * old_) * new_ + i0;
        const float* s0 = gs + (ql - j + JM) * NS;
        const float* s1 = s0 + 32 * NS;
        for (int i = 0; i < ni; ++i) {
          const float t = __ldg(kr + i);
          a0 = fmaf(t, s0[i], a0);
          a1 = fmaf(t, s1[i], a1);
        }
      }
      const int64_t u0 = (int64_t)(q0 + ql) * old_ + r, u1 = u0 + 32 * (int64_t)old_;
      if (u0 >= 1 && u0 <= T - 2) gxr[u0] = i0 == 0 ? a0 : gxr[u0] + a0;
      if (u1 >= 1 && u1 <= T - 2) gxr[u1] = i0 == 0 ? a1 : gxr[u1] + a1;
    }
  }
}

__device__ __forceinline__ int floordiv(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// gx[0] = sum of gx_ext over u in [-width, 0] (all of [-width, T + width + old) when T == 1), gx[T-1] over
// [T-1, T + width + old): blockIdx.y = edge; thread-strided positions, then a fixed-order tree.
__global__ void __launch_bounds__(THREADS)
resample_bwd_edge_kernel(const float* __restrict__ g, float* __restrict__ gx, const float* __restrict__ kt, int T,
                         int64_t out_len, int old_, int new_, int width, int K) {
  __shared__ float part[THREADS];
  const int row = blockIdx.x, edge = blockIdx.y;
  if (edge == 1 && T == 1) return;
  const int ulo = edge == 0 ? -width : T - 1;
  const int uhi = (edge == 0 && T > 1) ? 1 : T + width + old_;
  const float* gr = g + (size_t)row * (size_t)out_len;
  float acc = 0.f;
  for (int u = ulo + (int)threadIdx.x; u < uhi; u += THREADS) {
    int mlo = floordiv(u + width - K, old_) + 1;
    const int mhi = floordiv(u + width, old_);  // u + width >= 0
    if (mlo < 0) mlo = 0;
    float s = 0.f;
    for (int m = mlo; m <= mhi; ++m) {
      const float* kr = kt + (size_t)(u + width - m * old_) * new_;
      const float* gm = gr + (size_t)m * new_;
      const int64_t n = out_len - (int64_t)m * new_;
      const int ni = n < new_ ? (int)n : new_;
      for (int i = 0; i < ni; ++i) s = fmaf(__ldg(kr + i), __ldg(gm + i), s);
    }
    acc += s;
  }
  part[threadIdx.x] = acc;
  __syncthreads();
  for (int h = THREADS / 2; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) part[threadIdx.x] += part[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) gx[(size_t)row * T + (edge == 0 ? 0 : T - 1)] = part[0];
}

}  // namespace resample
}  // namespace b2a

extern "C" int64_t b2a_resample_out_len(int64_t T, int old_r, int new_r) {
  if (T < 1 || old_r < 1 || new_r < 1) return -1;
  return (int64_t)(((__int128)new_r * T) / old_r);  // floor(new * T / old)
}

extern "C" int b2a_resample_f32(const float* x, int64_t rows, int64_t T, int old_r, int new_r, int width,
                                const float* kernel_t, float* out, void* stream) {
  using namespace b2a::resample;
  B2A_REQUIRE(x && kernel_t && out, B2A_E_INVALID, "resample: null pointer");
  B2A_REQUIRE(rows >= 1 && T >= 1 && old_r >= 1 && new_r >= 1 && width >= 1, B2A_E_INVALID, "resample: bad argument");
  B2A_REQUIRE(T < ((int64_t)1 << 30), B2A_E_UNSUPPORTED, "resample: rows longer than 2^30 samples");
  const int64_t out_len = b2a_resample_out_len(T, old_r, new_r);
  B2A_REQUIRE(out_len >= 1, B2A_E_INVALID, "resample: empty output");
  const int K = 2 * width + old_r;
  const int64_t tiles = (out_len + OUT_PER_CTA - 1) / OUT_PER_CTA;
  B2A_REQUIRE(rows * tiles < (int64_t)2147483647, B2A_E_UNSUPPORTED, "resample: grid too large");
  const int frames_max = (OUT_PER_CTA + new_r - 1) / new_r + 1;
  const int span_max = (frames_max - 1) * old_r + K;
  const size_t smem = (size_t)span_max * 4;
  B2A_REQUIRE(smem <= 200 * 1024, B2A_E_UNSUPPORTED, "resample: %d -> %d needs %zu bytes of shared memory", old_r,
              new_r, smem);
  B2A_CUDA_OK(cudaFuncSetAttribute(resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  B2A_LAUNCH(resample_kernel, dim3((unsigned)(rows * tiles)), dim3(THREADS), smem, stream, x, out, kernel_t, (int)T,
             out_len, old_r, new_r, width, K, (int)tiles, span_max);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" int b2a_resample_backward_f32(const float* grad_out, int64_t rows, int64_t T, int old_r, int new_r, int width,
                                         const float* kernel_t, float* grad_x, void* stream) {
  using namespace b2a::resample;
  B2A_REQUIRE(grad_out && kernel_t && grad_x, B2A_E_INVALID, "resample_backward: null pointer");
  B2A_REQUIRE(rows >= 1 && T >= 1 && old_r >= 1 && new_r >= 1 && width >= 1, B2A_E_INVALID,
              "resample_backward: bad argument");
  B2A_REQUIRE(T < ((int64_t)1 << 30), B2A_E_UNSUPPORTED, "resample_backward: rows longer than 2^30 samples");
  const int64_t out_len = b2a_resample_out_len(T, old_r, new_r);
  B2A_REQUIRE(out_len >= 1, B2A_E_INVALID, "resample_backward: empty output");
  const int K = 2 * width + old_r;
  const int JM = (width + old_r - 1) / old_r;  // phases read frames q - JM .. q + JM
  // enough work items (phase x 64 q) per CTA to keep its 8 warps busy when there are few phases
  int chunks = (16 + old_r - 1) / old_r;
  if (chunks > 16) chunks = 16;
  const int64_t nq = T >= 3 ? (T - 2) / old_r + 1 : 0;  // q of the interior inputs 1 .. T-2
  while (chunks > 1 && (int64_t)(chunks / 2) * BWD_Q >= nq) chunks /= 2;
  constexpr size_t SMEM_MAX = 200 * 1024;
  while (chunks > 1 && (size_t)(chunks * BWD_Q + 2 * JM) * (new_r | 1) * 4 > SMEM_MAX) chunks /= 2;
  const int QT = chunks * BWD_Q;
  int IC = new_r;  // phases per staged tile; odd row stride NS = IC | 1 (lanes, consecutive q, hit distinct banks)
  while (IC > 1 && (size_t)(QT + 2 * JM) * (IC | 1) * 4 > SMEM_MAX) IC = (IC + 1) / 2;
  const int NS = IC | 1;
  const size_t smem = (size_t)(QT + 2 * JM) * NS * 4;
  B2A_REQUIRE(smem <= SMEM_MAX, B2A_E_UNSUPPORTED, "resample_backward: %d -> %d needs %zu bytes of shared memory",
              old_r, new_r, smem);
  if (nq > 0) {
    const int64_t tiles = (nq + QT - 1) / QT;
    B2A_REQUIRE(rows * tiles < (int64_t)2147483647, B2A_E_UNSUPPORTED, "resample_backward: grid too large");
    B2A_CUDA_OK(cudaFuncSetAttribute(resample_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    B2A_LAUNCH(resample_bwd_kernel, dim3((unsigned)(rows * tiles)), dim3(THREADS), smem, stream, grad_out, grad_x,
               kernel_t, (int)T, out_len, old_r, new_r, width, JM, QT, IC, NS, (int)tiles);
  }
  B2A_LAUNCH(resample_bwd_edge_kernel, dim3((unsigned)rows, 2), dim3(THREADS), 0, stream, grad_out, grad_x, kernel_t,
             (int)T, out_len, old_r, new_r, width, K);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}
