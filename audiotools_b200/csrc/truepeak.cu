// truepeak.cu -- BS.1770 true-peak level of a batch (K17 in DESIGN.md): the largest |value| of the signal
// oversampled by L (4 below 96 kHz, 2 below 192 kHz, else 1) with this package's 12-tap polyphase interpolator.
//
//   phase 0          the sample itself, exactly, so the true peak is never below max |x|
//   phase p >= 1     y[n, p] = sum_{d=-6..5} h_p[d] x[n - d],  x = 0 outside [0, T)
//                    h_p[d] = float(sinc(u) * (1 + cos(pi u / 6)) / 2),  u = d + p / L  (designed in double here)
//   instants         every (n, p) with n < T - 1, plus (T - 1, 0): no ringing outside the row is counted
//
// The structure is that of BS.1770-4 Annex 2 (a 4x polyphase FIR at 48 kHz); the taps are not the Annex's table.
//
// Two launches, no host sync.  true_peak_kernel: a 1-D grid over the work items (row, chunk of CHUNK samples) with a
// 64-bit index; the CTA stages its chunk plus an 8-sample halo in shared memory, each thread keeps RUN consecutive
// samples and their halo in registers
// and runs the 3 x 12 taps (kernel parameters: constant-bank operands of the FFMAs) over them.  The running maximum is
// exact, so the per-warp atomicMax into the zeroed row buffer gives the same bits in any order.  NaN: fmaxf would drop
// it, so phase 0 is compared as uint bits of |x| (every NaN sorts above inf); a NaN among the interpolated values needs
// a non-finite sample, which phase 0 already reports.  item_db_kernel: the channel maximum and 20 log10.
// The constants, the taps, the run staging and the phase evaluation are in truepeak_internal.h.
#include "truepeak_internal.h"

namespace b2a {
namespace truepeak {

constexpr int TILE = CHUNK + 2 * HALO;

// v[k + HALO] = x[n0 + k].  Folds |x[n0 + k]| into m0 (as bits) and |y[n0 + k, p]| into mi.  EDGE: the run reaches the
// row's last sample, so only the instants inside the row count.
template <int NP, bool EDGE>
__device__ __forceinline__ void run_max(const float (&v)[RUN + 2 * HALO], const Taps& taps, int64_t n0, int64_t T,
                                        unsigned& m0, float& mi) {
#pragma unroll
  for (int k = 0; k < RUN; ++k) {
    if (!EDGE || n0 + k < T) m0 = max(m0, __float_as_uint(v[k + HALO]) & 0x7fffffffu);
#pragma unroll
    for (int p = 0; p < NP; ++p) {
      const float y = phase(taps, p, v, k);
      if (!EDGE || n0 + k < T - 1) mi = fmaxf(mi, fabsf(y));
    }
  }
}

// row_bits [rows] zeroed by the caller; on return the bits of each row's true peak.  NP = L - 1 interpolated phases.
template <int NP>
__global__ void __launch_bounds__(TPB) true_peak_kernel(const float* __restrict__ x, int64_t T, int64_t n_chunks,
                                                        int64_t work, const Taps taps, unsigned* __restrict__ row_bits) {
  __shared__ __align__(16) float s[TILE];
  for (int64_t w = blockIdx.x; w < work; w += gridDim.x) {
    const int64_t row = w / n_chunks, c0 = (w - row * n_chunks) * CHUNK;
    const float* xr = x + row * T;
    for (int i = threadIdx.x; i < TILE; i += TPB) {
      const int64_t n = c0 - HALO + i;
      s[i] = (n >= 0 && n < T) ? __ldg(xr + n) : 0.f;
    }
    __syncthreads();
    const int64_t n0 = c0 + (int64_t)threadIdx.x * RUN;
    unsigned m0 = 0;
    float mi = 0.f;
    if (n0 < T) {
      float v[RUN + 2 * HALO];
      stage_run(s + threadIdx.x * RUN, v);
      if (n0 + RUN < T)
        run_max<NP, false>(v, taps, n0, T, m0, mi);
      else
        run_max<NP, true>(v, taps, n0, T, m0, mi);
    }
    unsigned m = max(m0, __float_as_uint(mi));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m != 0) atomicMax(row_bits + row, m);
    __syncthreads();  // the next work item overwrites s
  }
}

__global__ void __launch_bounds__(TPB) item_db_kernel(const unsigned* __restrict__ row_bits, int64_t B, int C,
                                                      float* __restrict__ item_db) {
  const int64_t b = (int64_t)blockIdx.x * TPB + threadIdx.x;
  if (b >= B) return;
  unsigned m = 0;
  for (int c = 0; c < C; ++c) m = max(m, row_bits[b * C + c]);
  item_db[b] = 20.f * log10f(__uint_as_float(m));
}

}  // namespace truepeak
}  // namespace b2a

using namespace b2a::truepeak;

extern "C" int b2a_true_peak_factor(double rate) {
  B2A_REQUIRE(rate > 0 && rate < INFINITY, B2A_E_INVALID, "true_peak: bad sample rate %g", rate);
  return rate < 96000 ? 4 : rate < 192000 ? 2 : 1;
}

extern "C" int b2a_true_peak_taps(int factor, float* taps_h) {
  Taps t;
  const int rc = design(factor, &t);
  if (rc != B2A_OK) return rc;
  B2A_REQUIRE(taps_h || factor == 1, B2A_E_INVALID, "true_peak_taps: null pointer");
  if (factor > 1) memcpy(taps_h, t.h, sizeof(float) * NTAP * (factor - 1));
  return B2A_OK;
}

extern "C" int b2a_true_peak_f32(const float* x, int64_t B, int C, int64_t T, int factor, float* row_peak,
                                 float* item_db, void* stream) {
  B2A_REQUIRE(x && row_peak, B2A_E_INVALID, "true_peak: null pointer");
  B2A_REQUIRE(B >= 1 && C >= 1 && T >= 1, B2A_E_INVALID, "true_peak: bad shape B=%lld C=%d T=%lld", (long long)B, C,
              (long long)T);
  B2A_REQUIRE(T <= INT64_MAX / B / C, B2A_E_INVALID, "true_peak: B * C * T overflows");
  Taps taps;
  const int rc = design(factor, &taps);
  if (rc != B2A_OK) return rc;
  const int64_t rows = B * C, n_chunks = (T + CHUNK - 1) / CHUNK, work = rows * n_chunks;
  // one CTA per work item (a CTA loops only past 2^31 - 1 of them): a persistent grid that prefetches the next item
  // into registers measured 10 % slower on the H100 (64 registers: 4 CTAs per SM instead of 6)
  const unsigned grid = (unsigned)(work < INT32_MAX ? work : INT32_MAX);
  auto kern = factor == 4 ? true_peak_kernel<3> : factor == 2 ? true_peak_kernel<1> : true_peak_kernel<0>;
  unsigned* bits = reinterpret_cast<unsigned*>(row_peak);
  B2A_CUDA_OK(cudaMemsetAsync(bits, 0, (size_t)rows * sizeof(unsigned), (cudaStream_t)stream));
  B2A_LAUNCH(kern, dim3(grid), dim3(TPB), 0, stream, x, T, n_chunks, work, taps, bits);
  B2A_CUDA_OK(cudaGetLastError());
  if (item_db) {
    B2A_LAUNCH(item_db_kernel, dim3((unsigned)((B + TPB - 1) / TPB)), dim3(TPB), 0, stream, bits, B, C, item_db);
    B2A_CUDA_OK(cudaGetLastError());
  }
  return B2A_OK;
}
