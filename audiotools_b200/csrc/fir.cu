// fir.cu -- direct (time-domain) strided FIR for short filters on sm_90a.
//
//   out[row][m] = sum_{k<K} taps[f][k] * xv[row][m*stride + k - left[f]],   f = row / rows_per_filt, m < out_len
//   (correlation form; xv extends x by zeros or edge replication).
//
// Serves the short end of the hot path's FIRs, where the partitioned FFT engine (fftconv.cu) is overkill:
//   * julius.LowPassFilter / HighPassFilter with a few hundred taps (ref:audiotools/core/dsp.py:153-215):
//     stride 1, per-item taps, left = half, optional out = x - y;
//   * julius.resample_frac when the reduced new rate is 1 (48k -> 16k, 44.1k -> 22.05k, ...:
//     ref:audiotools/core/audio_signal.py:732-734): stride = old, one 2*width+old tap kernel, left = width.
//
// One CTA = 256 threads x 8 consecutive outputs.  The input span of the tile is staged once in shared
// memory, de-interleaved by phase p = (sample index) mod stride so that for each phase the thread slides an
// 8+8 register window over a unit-stride stream: per 8 taps, 8 new samples and 8 (broadcast) taps are loaded
// for 64 FMAs -- as FOUR 128-bit shared loads (two for the samples, two broadcast ones for the taps).  Streams are padded
// 4 words per 32 so that the 8-word lane stride is 16 B aligned and conflict free for 128-bit accesses (a quarter warp
// covers word offsets 0, 8, 16, 24, 36, 44, 52, 60: eight distinct 4-word bank groups).
#include "b2a_common.h"

namespace b2a {
namespace fir {

constexpr int THREADS = 256;
constexpr int R = 8;                  // outputs per thread
constexpr int TILE = THREADS * R;     // outputs per CTA

__device__ __forceinline__ int pad32(int n) { return n + ((n >> 5) << 2); }

struct Params {
  const float* x;
  const float* taps;       // [n_filt, K]
  const int32_t* left;     // [n_filt] nullable
  const int32_t* bypass;   // [n_filt] nullable: non-zero = copy the rows of this filter through (mask-aware transforms)
  float* out;
  int T, K, stride, rows_per_filt, left0, pad_mode, subtract, tiles_per_row;
  int64_t out_len;
  int np;                  // stream length per phase (samples)
  int sp;                  // padded stream stride (words)
  int qmax;                // taps per phase, rounded up to 8
  int off_taps;            // byte offset of the tap table in shared memory
};

__global__ void __launch_bounds__(THREADS) fir_direct_kernel(Params p) {
  B2A_DYN_SMEM(smem);
  float* xs = reinterpret_cast<float*>(smem);               // [stride][sp]   de-interleaved, padded
  float* tp = reinterpret_cast<float*>(smem + p.off_taps);  // [stride][qmax] taps of phase p, zero padded
  const int tid = threadIdx.x;
  const int row = blockIdx.x / p.tiles_per_row, tile = blockIdx.x - row * p.tiles_per_row;
  const int f = row / p.rows_per_filt;
  const int left = p.left0 + (p.left ? __ldg(p.left + f) : 0);
  const int64_t m_base = (int64_t)tile * TILE;
  const int64_t j0 = m_base * p.stride - left;  // x-coordinate of stream position 0, phase 0
  const float* xr = p.x + (size_t)row * (size_t)p.T;
  const int S = p.stride;
  if (p.bypass && __ldg(p.bypass + f)) {  // item not selected by the transform's mask: out = x (stride 1), CTA-uniform
    float* orow = p.out + (size_t)row * (size_t)p.out_len;
    for (int i = tid; i < TILE; i += THREADS) {
      const int64_t m = m_base + i;
      if (m < p.out_len) orow[m] = __ldg(xr + m);
    }
    return;
  }
  // ---- stage the span, phase-de-interleaved
  // (phase-major loops: no integer division per sample; the S phases read the same cache lines back to back)
  const bool inside = (j0 >= 0) && (j0 + (int64_t)p.np * S <= (int64_t)p.T);  // CTA-uniform: no padding in this tile
  for (int ph = 0; ph < S; ++ph) {
    float* dst = xs + ph * p.sp;
    if (inside) {
      const float* src = xr + j0 + ph;
      for (int n = tid; n < p.np; n += THREADS) dst[pad32(n)] = __ldg(src + (size_t)n * S);
    } else {
      for (int n = tid; n < p.np; n += THREADS) {
        const int64_t u = j0 + (int64_t)n * S + ph;
        float v;
        if (u >= 0 && u < p.T) v = __ldg(xr + u);
        else if (p.pad_mode == B2A_PAD_REPLICATE) v = __ldg(xr + (u < 0 ? 0 : p.T - 1));
        else v = 0.f;
        dst[pad32(n)] = v;
      }
    }
  }
  const float* tr = p.taps + (size_t)f * p.K;
  for (int ph = 0; ph < S; ++ph)
    for (int q = tid; q < p.qmax; q += THREADS) {
      const int k = q * S + ph;
      tp[ph * p.qmax + q] = (k < p.K) ? __ldg(tr + k) : 0.f;
    }
  __syncthreads();

  float acc[R];
#pragma unroll
  for (int r = 0; r < R; ++r) acc[r] = 0.f;
  const int ml = tid * R;  // first output of this thread within the tile == its stream offset
  for (int ph = 0; ph < S; ++ph) {
    const float* s = xs + ph * p.sp;
    const float* t = tp + ph * p.qmax;
    float w[2 * R];
    {  // ml is a multiple of 8: its 8 samples are two aligned float4s inside one padded 32-group
      const float4 a = *reinterpret_cast<const float4*>(s + pad32(ml)), b = *reinterpret_cast<const float4*>(s + pad32(ml) + 4);
      w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
    }
    for (int q0 = 0; q0 < p.qmax; q0 += R) {
      {
        const float* sn = s + pad32(ml + q0 + R);
        const float4 a = *reinterpret_cast<const float4*>(sn), b = *reinterpret_cast<const float4*>(sn + 4);
        w[R] = a.x; w[R + 1] = a.y; w[R + 2] = a.z; w[R + 3] = a.w; w[R + 4] = b.x; w[R + 5] = b.y; w[R + 6] = b.z; w[R + 7] = b.w;
      }
      const float4 h0 = *reinterpret_cast<const float4*>(t + q0), h1 = *reinterpret_cast<const float4*>(t + q0 + 4);
      const float h[R] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
#pragma unroll
      for (int u = 0; u < R; ++u) {
#pragma unroll
        for (int r = 0; r < R; ++r) acc[r] = fmaf(h[u], w[u + r], acc[r]);
      }
#pragma unroll
      for (int j = 0; j < R; ++j) w[j] = w[R + j];
    }
  }
  float* orow = p.out + (size_t)row * (size_t)p.out_len;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int64_t m = m_base + ml + r;
    if (m < p.out_len) {
      float v = acc[r];
      if (p.subtract) v = __ldg(xr + m) - v;  // stride 1 only (checked on the host)
      orow[m] = v;
    }
  }
}

}  // namespace fir
}  // namespace b2a

extern "C" int b2a_fir_direct_supported(int64_t T, int K, int stride) {
  using namespace b2a::fir;
  if (K < 1 || stride < 1 || T < 1 || T >= ((int64_t)1 << 30)) return 0;
  const int qmax = (((K + stride - 1) / stride) + R - 1) / R * R;
  const int np = TILE + qmax + R;
  const int sp = ((np + ((np >> 5) << 2) + 4 + 3) / 4) * 4;
  const size_t bytes = (size_t)stride * sp * 4 + (size_t)stride * qmax * 4;
  return bytes <= 160 * 1024;
}

extern "C" int b2a_fir_direct_f32(const float* x, int64_t rows, int64_t T, const float* taps, int64_t n_filt, int K,
                                  int rows_per_filt, const int32_t* left, int left0, int stride, int64_t out_len,
                                  int pad_mode, int subtract_from_input, const int32_t* bypass, float* out,
                                  void* stream) {
  using namespace b2a::fir;
  B2A_REQUIRE(x && taps && out, B2A_E_INVALID, "fir: null pointer");
  B2A_REQUIRE(rows >= 1 && T >= 1 && n_filt >= 1 && K >= 1 && rows_per_filt >= 1 && stride >= 1 && out_len >= 1,
              B2A_E_INVALID, "fir: bad argument");
  B2A_REQUIRE((rows + rows_per_filt - 1) / rows_per_filt <= n_filt, B2A_E_INVALID, "fir: not enough filters");
  B2A_REQUIRE(pad_mode == B2A_PAD_CONSTANT || pad_mode == B2A_PAD_REPLICATE, B2A_E_INVALID, "fir: pad_mode %d", pad_mode);
  B2A_REQUIRE(!subtract_from_input || (stride == 1 && out_len <= T), B2A_E_INVALID, "fir: x - y needs stride 1");
  B2A_REQUIRE(b2a_fir_direct_supported(T, K, stride), B2A_E_UNSUPPORTED,
              "fir: K=%d stride=%d does not fit the direct kernel (use b2a_fftconv_f32)", K, stride);
  B2A_REQUIRE(out != x, B2A_E_INVALID, "fir: in-place is not supported");
  B2A_REQUIRE(!bypass || (stride == 1 && out_len <= T), B2A_E_INVALID, "fir: bypass needs stride 1");
  Params p;
  memset(&p, 0, sizeof(p));
  p.x = x; p.taps = taps; p.left = left; p.out = out; p.bypass = bypass;
  p.T = (int)T; p.K = K; p.stride = stride; p.rows_per_filt = rows_per_filt; p.left0 = left0;
  p.pad_mode = pad_mode; p.subtract = subtract_from_input; p.out_len = out_len;
  p.qmax = (((K + stride - 1) / stride) + R - 1) / R * R;
  p.np = TILE + p.qmax + R;
  p.sp = ((p.np + ((p.np >> 5) << 2) + 4 + 3) / 4) * 4;
  p.off_taps = stride * p.sp * 4;
  const size_t smem = (size_t)p.off_taps + (size_t)stride * p.qmax * 4;
  const int64_t tiles = (out_len + TILE - 1) / TILE;
  p.tiles_per_row = (int)tiles;
  B2A_REQUIRE(rows * tiles < (int64_t)2147483647, B2A_E_UNSUPPORTED, "fir: grid too large");
  B2A_CUDA_OK(cudaFuncSetAttribute(fir_direct_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  B2A_LAUNCH(fir_direct_kernel, dim3((unsigned)(rows * tiles)), dim3(THREADS), smem, stream, p);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

// ---------------------------------------------------------------------------------------------
// Replicate-padding fold of a stride-1 FIR's adjoint.  For y[m] = sum_k h[k] xv[m + k - left] (xv = x extended by
// replicate padding), the adjoint is the zero-padded correlation with reversed taps (computed elsewhere) plus what the
// padded positions carry back to the edge samples:
//     gx[0]   += sum_{n < left}          P[left - 1 - n] g[n],        P[k] = h[0] + ... + h[k]
//     gx[T-1] += sum_{n >= T + left - K + 1} S[T + left - n] g[n],    S[k] = h[k] + ... + h[K-1]
// (P clamped at K-1; holds for any T, also T < K).  P and S per filter come from fir_scan_kernel (one thread per
// filter and direction, sequential: fixed order); the fold is one warp per row that reads at most 2 K samples.
// ---------------------------------------------------------------------------------------------
namespace b2a {
namespace fir {

__global__ void __launch_bounds__(64) fir_scan_kernel(const float* __restrict__ h, int n_filt, int K,
                                                      float* __restrict__ ps) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 2 * n_filt) return;
  const int f = t >> 1;
  const float* hr = h + (size_t)f * K;
  float* o = ps + (size_t)f * 2 * K;
  float s = 0.f;
  if ((t & 1) == 0) {
    for (int k = 0; k < K; ++k) { s += __ldg(hr + k); o[k] = s; }
  } else {
    for (int k = K - 1; k >= 0; --k) { s += __ldg(hr + k); o[K + k] = s; }
  }
}

__global__ void __launch_bounds__(256) fir_pad_fold_kernel(const float* __restrict__ g, int rows, int T,
                                                           const float* __restrict__ ps, int K, int rows_per_filt,
                                                           const int32_t* __restrict__ left, int left0,
                                                           const int32_t* __restrict__ bypass, float* __restrict__ gx) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int f = row / rows_per_filt;
  if (bypass && __ldg(bypass + f)) return;  // a copied row: its gradient is the plain copy
  const int lf = left0 + (left ? __ldg(left + f) : 0);
  const float* P = ps + (size_t)f * 2 * K;
  const float* S = P + K;
  const float* gr = g + (size_t)row * T;
  float sl = 0.f, sr = 0.f;
  const int nl = lf < T ? lf : T;
  for (int n = lane; n < nl; n += 32) {
    const int k = lf - 1 - n;
    sl = fmaf(P[k < K - 1 ? k : K - 1], __ldg(gr + n), sl);
  }
  int n0 = T + lf - K + 1;
  if (n0 < 0) n0 = 0;
  for (int n = n0 + lane; n < T; n += 32) sr = fmaf(S[T + lf - n], __ldg(gr + n), sr);
  sl = warp_sum(sl);
  sr = warp_sum(sr);
  if (lane == 0) {
    float* o = gx + (size_t)row * T;
    o[0] += sl;
    o[T - 1] += sr;
  }
}

}  // namespace fir
}  // namespace b2a

extern "C" size_t b2a_fir_pad_fold_workspace_bytes(int64_t n_filt, int K) {
  if (n_filt < 1 || K < 1) return 0;
  return (size_t)n_filt * 2 * (size_t)K * sizeof(float);
}

extern "C" int b2a_fir_pad_fold_f32(const float* grad_out, int64_t rows, int64_t T, const float* taps, int64_t n_filt,
                                    int K, int rows_per_filt, const int32_t* left, int left0, const int32_t* bypass,
                                    float* grad_x, void* ws, size_t ws_bytes, void* stream) {
  using namespace b2a::fir;
  B2A_REQUIRE(grad_out && taps && grad_x && ws, B2A_E_INVALID, "fir_pad_fold: null pointer");
  B2A_REQUIRE(rows >= 1 && T >= 1 && T < ((int64_t)1 << 30) && n_filt >= 1 && n_filt < (1 << 24) && K >= 1 &&
                  rows_per_filt >= 1 && left0 >= 0,
              B2A_E_INVALID, "fir_pad_fold: bad shape");
  B2A_REQUIRE((rows + rows_per_filt - 1) / rows_per_filt <= n_filt, B2A_E_INVALID,
              "fir_pad_fold: %lld rows / %d per filter need more than %lld filters", (long long)rows, rows_per_filt,
              (long long)n_filt);
  B2A_REQUIRE(ws_bytes >= b2a_fir_pad_fold_workspace_bytes(n_filt, K), B2A_E_INVALID, "fir_pad_fold: workspace too small");
  B2A_REQUIRE(rows / 8 < (int64_t)2147483647, B2A_E_UNSUPPORTED, "fir_pad_fold: too many rows");
  float* ps = reinterpret_cast<float*>(ws);
  B2A_LAUNCH(fir_scan_kernel, dim3((unsigned)((2 * n_filt + 63) / 64)), dim3(64), 0, stream, taps, (int)n_filt, K, ps);
  B2A_LAUNCH(fir_pad_fold_kernel, dim3((unsigned)((rows + 7) / 8)), dim3(256), 0, stream, grad_out, (int)rows, (int)T, ps,
             K, rows_per_filt, left, left0, bypass, grad_x);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}
