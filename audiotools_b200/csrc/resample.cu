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
