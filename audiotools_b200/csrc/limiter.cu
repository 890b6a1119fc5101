// limiter.cu -- look-ahead true-peak limiter of a batch (K18 in DESIGN.md): one gain series per item that dips around
// every instant whose true-peak envelope passes the ceiling and is exactly 1 elsewhere.
//
//   envelope   y[n, p] of truepeak.cu (its factor, its taps), between samples n and n + 1;
//              e_c[n] = max(|x[n]|, max_p |y[n, p]|, max_p |y[n - 1, p]|) over the instants inside the row,
//              e[n] = max_c e_c[n]  (the channels are linked)
//   reduction  q[n] = 0 where e[n] <= c, else 1 - c / e[n]  (NaN where e[n] is not finite)
//   hold       h[n] = max q[j], |j - n| <= A, j in [0, T)
//   release    d[n] = max(h[n], a d[n - 1]), d[-1] = 0; afterwards d < 2^-26 counts as 0
//   attack     r[n] = mean d[j], |j - n| <= A, j in [0, T)  (divided by the number of such j)
//   output     out[c, n] = x[c, n] (1 - r[n]),  x = float(gain[b] x) when a gain is given
//
// Three launches, no host sync, the carries of the release cross a launch boundary:
//   envelope_hold_kernel   a CTA per (item, chunk of CHUNK samples): for every channel the chunk plus a halo of
//                          Ap + 8 samples (Ap = A rounded up to 16) in shared memory, the 3 x 12 taps over runs of 16
//                          samples in registers as in truepeak.cu, the channel maximum as uint bits (NaN sorts above
//                          inf); q; the sliding maximum by log-step doubling between two shared buffers; h to the
//                          workspace; and the release of the chunk's own h (from 0) at its end and Ap before its end.
//   carry_kernel           a warp per item: D_k = max(local end_k, a^CHUNK D_{k-1}) as a warp scan in double over 32
//                          chunks at a time (exact: nothing is truncated), and from it the value of d just before
//                          each chunk's left halo, H_{k+1} = max(local mid_k, a^(CHUNK - Ap) D_{k-1}).
//   release_apply_kernel   a CTA per (item, chunk): h of the chunk and Ap on either side; the release from H_k (a
//                          sequential run of 16 per thread, a decayed-maximum scan over the runs: the step of width o
//                          multiplies by the constant a^(16 o), so no coefficient travels with the value); d and the
//                          run sums to shared memory; the window mean as a sliding sum in double per run of 16; then
//                          out = x (1 - r) for the C rows.  A chunk whose h (with halo) is all 0 and whose H_k is
//                          below 2^-26 skips all of that: it copies, or in place without a gain does nothing.
// Every maximum is taken on the bits of non-negative floats, so NaN propagates without a branch; sums are per item and
// in a fixed order: reruns and batch-versus-single calls are bit-identical.
#include "truepeak_internal.h"

namespace b2a {
namespace limiter {

// truepeak_internal.h: TPB threads per CTA of the envelope kernel, runs of RUN samples per thread, chunks of CHUNK
// samples of an item per CTA work item (tests cover T = CHUNK +- 1), the taps' reach HALO, Taps, design, stage_run, phase
using namespace truepeak;

constexpr int AMAX = 1024;           // largest look-ahead in samples
constexpr int TPB3 = 384;            // release kernel: one thread per run of the chunk plus both halos
constexpr float TINY = 1.4901161193847656e-08f;  // 2^-26

struct Decay {
  float p1[RUN + 1];       // a^k
  float p16[33];           // a^(16 m)
  float p512[TPB3 / 32 + 1];  // a^(512 m)
};

// shared arrays read and written in runs of 16 per thread: one pad word per 16 keeps a warp's 32 runs on 32 banks
__device__ __forceinline__ int sk(int i) { return i + (i >> 4); }
// maximum of two non-negative (sign bit clear) floats on their bits: NaN sorts above inf and so propagates
__device__ __forceinline__ float maxb(float a, float b) {
  return __uint_as_float(max(__float_as_uint(a), __float_as_uint(b)));
}
// the same for doubles, as a comparison
__device__ __forceinline__ double maxn(double a, double b) { return (a > b || a != a) ? a : b; }

// v[j] = x[n0 - HALO + j].  e[k] = bits of e_c[n0 + k].  EDGE: some instant n0 - 1 .. n0 + RUN - 1 lies outside the row.
template <int NP, bool EDGE>
__device__ __forceinline__ void run_envelope(const float (&v)[RUN + 2 * HALO], const Taps& taps, int64_t n0, int64_t T,
                                             unsigned (&e)[RUN]) {
  unsigned prev = 0;
#pragma unroll
  for (int k = -1; k < RUN; ++k) {
    unsigned m = 0;
#pragma unroll
    for (int p = 0; p < NP; ++p) m = max(m, __float_as_uint(fabsf(phase(taps, p, v, k))));
    if (EDGE && !(n0 + k >= 0 && n0 + k < T - 1)) m = 0;
    if (k >= 0) e[k] = max(__float_as_uint(fabsf(v[k + HALO])), max(m, prev));  // x is 0 outside the row
    prev = m;
  }
}

// Inclusive decayed-maximum scan over the CTA's threads: thread t holds the value of d at the end of run t computed from
// the run alone; returns d just before run t given `carry` just before run 0.  s_warp: one float per warp.
__device__ __forceinline__ float scan_exclusive(float v, float carry, const Decay& dec, float* s_warp) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v = maxb(v, dec.p16[o] * u);
  }
  if (lane == 31) s_warp[wid] = v;
  __syncthreads();
  float cw = carry;  // d just before this warp's first run
  for (int j = 0; j < wid; ++j) cw = maxb(s_warp[j], dec.p512[1] * cw);
  const float left = __shfl_up_sync(0xffffffffu, v, 1);
  return lane == 0 ? cw : maxb(left, dec.p16[lane] * cw);
}

// h_out [B, T]; em_out [B, n_chunks, 2]: the release of the chunk's own h at its last sample and Ap samples earlier.
template <int NP>
__global__ void __launch_bounds__(TPB) envelope_hold_kernel(const float* __restrict__ x, const float* __restrict__ gain,
                                                            int C, int64_t T, int64_t n_chunks, int64_t work, int A,
                                                            int Ap, const float* __restrict__ ceiling,
                                                            B2A_GRID_CONSTANT const Taps taps,
                                                            B2A_GRID_CONSTANT const Decay dec, float* __restrict__ h_out,
                                                            float* __restrict__ em_out) {
  B2A_DYN_SMEM(smem);
  __shared__ float s_warp[TPB / 32];
  const int W = CHUNK + 2 * Ap, n_runs = W / RUN, win = 2 * A + 1;
  float* sx = reinterpret_cast<float*>(smem);          // [W + 2 HALO] staged samples; later a doubling buffer [sk(W)]
  unsigned* se = reinterpret_cast<unsigned*>(smem) + sk(W);  // [sk(W)] bits of e, then of q
  for (int64_t w = blockIdx.x; w < work; w += gridDim.x) {
    const int64_t b = w / n_chunks, chunk = w - b * n_chunks, c0 = chunk * CHUNK, s0 = c0 - Ap;
    const float g0 = gain ? __ldg(gain + b) : 1.f, cl = __ldg(ceiling + b);
    for (int c = 0; c < C; ++c) {
      const float* xr = x + (b * C + c) * T;
      for (int i = threadIdx.x; i < W + 2 * HALO; i += TPB) {
        const int64_t n = s0 - HALO + i;
        sx[i] = (n >= 0 && n < T) ? __ldg(xr + n) * g0 : 0.f;
      }
      __syncthreads();
      for (int r = threadIdx.x; r < n_runs; r += TPB) {
        const int64_t n0 = s0 + (int64_t)r * RUN;
        unsigned e[RUN];
        if (n0 + RUN <= 0 || n0 >= T) {
#pragma unroll
          for (int k = 0; k < RUN; ++k) e[k] = 0;
        } else {
          float v[RUN + 2 * HALO];
          stage_run(sx + r * RUN, v);
          if (n0 >= 1 && n0 + RUN < T)
            run_envelope<NP, false>(v, taps, n0, T, e);
          else
            run_envelope<NP, true>(v, taps, n0, T, e);
        }
        unsigned* er = se + sk(r * RUN);
        if (c > 0) {
#pragma unroll
          for (int k = 0; k < RUN; ++k) e[k] = max(e[k], er[k]);
        }
        if (c == C - 1) {
#pragma unroll
          for (int k = 0; k < RUN; ++k) {
            const float ef = __uint_as_float(e[k]);
            const float q = ef > cl ? 1.f - cl / ef : 0.f;
            e[k] = e[k] >= 0x7f800000u ? 0x7fffffffu : __float_as_uint(q);
          }
        }
#pragma unroll
        for (int k = 0; k < RUN; ++k) er[k] = e[k];
      }
      __syncthreads();  // sx is staged again, or becomes the doubling buffer
    }
    // sliding maximum over win = 2 A + 1: after the pass of width L, src[i] = max q[i .. i + 2 L)
    unsigned* src = se;
    unsigned* dst = reinterpret_cast<unsigned*>(sx);
    int L = 1;
    for (; 2 * L <= win; L *= 2) {
      for (int i = threadIdx.x; i < W; i += TPB)
        dst[sk(i)] = i + L < W ? max(src[sk(i)], src[sk(i + L)]) : src[sk(i)];
      __syncthreads();
      unsigned* t = src;
      src = dst, dst = t;
    }
    float* hs = reinterpret_cast<float*>(dst);  // h of the chunk, 0 past the row's end
    for (int t = threadIdx.x; t < CHUNK; t += TPB) {
      const int i = t + Ap - A;
      const unsigned hv = c0 + t < T ? max(src[sk(i)], src[sk(i + win - L)]) : 0u;
      hs[sk(t)] = __uint_as_float(hv);
      if (c0 + t < T) h_out[b * T + c0 + t] = __uint_as_float(hv);
    }
    __syncthreads();
    float d = 0.f;
#pragma unroll
    for (int k = 0; k < RUN; ++k) d = maxb(hs[sk(threadIdx.x * RUN + k)], dec.p1[1] * d);
    const float before = scan_exclusive(d, 0.f, dec, s_warp);
    d = maxb(d, dec.p1[RUN] * before);
    float* em = em_out + (b * n_chunks + chunk) * 2;
    if (threadIdx.x == TPB - 1) em[0] = d;
    if (threadIdx.x == TPB - 1 - Ap / RUN) em[1] = d;
    __syncthreads();  // the next work item overwrites the shared buffers and s_warp
  }
}

// hc [B, n_chunks]: d just before sample k CHUNK - Ap, the start of chunk k's left halo.
__global__ void __launch_bounds__(TPB) carry_kernel(const float* __restrict__ em, int64_t B, int64_t n_chunks, double l2a,
                                                    int Ap, float* __restrict__ hc) {
  const int64_t b = ((int64_t)blockIdx.x * TPB + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (b >= B) return;  // whole warps
  double pw[5];
#pragma unroll
  for (int s = 0; s < 5; ++s) pw[s] = exp2(l2a * (double)(CHUNK << s));
  const double p_lane = exp2(l2a * (double)(CHUNK * (lane + 1))), p_mid = exp2(l2a * (double)(CHUNK - Ap));
  double carry = 0.0;  // D of the chunk before this batch of 32
  if (lane == 0) hc[b * n_chunks] = 0.f;
  for (int64_t base = 0; base < n_chunks - 1; base += 32) {  // the last chunk has no successor
    const int64_t k = base + lane;
    const bool valid = k < n_chunks - 1;
    const double mid = valid ? (double)em[(b * n_chunks + k) * 2 + 1] : 0.0;
    double v = valid ? (double)em[(b * n_chunks + k) * 2] : 0.0;
#pragma unroll
    for (int s = 0; s < 5; ++s) {
      const double u = __shfl_up_sync(0xffffffffu, v, 1 << s);
      if (lane >= (1 << s)) v = maxn(v, pw[s] * u);
    }
    v = maxn(v, p_lane * carry);  // D_k
    double before = __shfl_up_sync(0xffffffffu, v, 1);
    if (lane == 0) before = carry;  // D_{k-1}
    if (valid) hc[b * n_chunks + k + 1] = (float)maxn(mid, p_mid * before);
    carry = __shfl_sync(0xffffffffu, v, 31);
  }
}

// blockDim.x = the chunk's runs plus both halos', rounded up to a warp (<= TPB3).  red: nullable [B, T].
template <bool VEC>
__global__ void __launch_bounds__(TPB3) release_apply_kernel(const float* x, const float* __restrict__ gain, int C,
                                                             int64_t T, int64_t n_chunks, int64_t work, int A, int Ap,
                                                             const float* __restrict__ h, const float* __restrict__ hc,
                                                             B2A_GRID_CONSTANT const Decay dec, float* out, float* red) {
  B2A_DYN_SMEM(smem);
  __shared__ float s_warp[TPB3 / 32];
  __shared__ unsigned s_any;
  const int W = CHUNK + 2 * Ap, n_runs = W / RUN, NT = blockDim.x;
  double* ss = reinterpret_cast<double*>(smem);        // [TPB3] sum of d over each run
  float* sd = reinterpret_cast<float*>(ss + TPB3);     // [sk(W)] h, then d
  float* sg = sd + sk(W);                              // [sk(CHUNK)] r of the chunk
  const int lane = threadIdx.x & 31;
  for (int64_t w = blockIdx.x; w < work; w += gridDim.x) {
    const int64_t b = w / n_chunks, chunk = w - b * n_chunks, c0 = chunk * CHUNK, s0 = c0 - Ap;
    const float carry = __ldg(hc + b * n_chunks + chunk);
    if (threadIdx.x == 0) s_any = 0;
    unsigned nz = 0;
    for (int i = threadIdx.x; i < W; i += NT) {
      const int64_t n = s0 + i;
      const float v = (n >= 0 && n < T) ? __ldg(h + b * T + n) : 0.f;
      sd[sk(i)] = v;
      nz |= __float_as_uint(v);
    }
    __syncthreads();
    nz = __ballot_sync(0xffffffffu, nz != 0);
    if (lane == 0 && nz) atomicMax(&s_any, 1u);
    __syncthreads();
    const bool quiet = s_any == 0 && carry < TINY;  // every d of the span is below 2^-26: r = 0 (a NaN carry is not quiet)
    if (!quiet) {
      const int r = threadIdx.x;
      float dl[RUN], d = 0.f;
      if (r < n_runs) {
#pragma unroll
        for (int k = 0; k < RUN; ++k) dl[k] = d = maxb(sd[sk(r * RUN + k)], dec.p1[1] * d);
      } else {
#pragma unroll
        for (int k = 0; k < RUN; ++k) dl[k] = 0.f;
      }
      const float before = scan_exclusive(d, carry, dec, s_warp);
      if (r < n_runs) {
        double sum = 0.0;
#pragma unroll
        for (int k = 0; k < RUN; ++k) {
          float v = maxb(dl[k], dec.p1[k + 1] * before);
          v = v < TINY ? 0.f : v;
          if (s0 + r * RUN + k >= T) v = 0.f;  // past the row's end nothing is averaged
          sd[sk(r * RUN + k)] = v;
          sum += (double)v;
        }
        ss[r] = sum;
      }
      __syncthreads();
      if (threadIdx.x < TPB) {
        const int t = threadIdx.x, R = Ap / RUN + t, u = A >> 4, v = A & 15;
        double s = 0.0;
        for (int j = R - u; j < R + u; ++j) s += ss[j];
        for (int i = 0; i < v; ++i) s += (double)sd[sk((R - u) * RUN - v + i)];
        for (int i = 0; i <= v; ++i) s += (double)sd[sk((R + u) * RUN + i)];
#pragma unroll
        for (int k = 0; k < RUN; ++k) {
          const int i = R * RUN + k;
          const int64_t n = c0 + t * RUN + k;
          const int64_t lo = n - A > 0 ? n - A : 0, hi = n + A < T - 1 ? n + A : T - 1;
          float rr = (float)s / (float)(hi - lo + 1);
          rr = rr < 0.5f * TINY ? 0.f : rr;  // the sliding sum's rounding residue; 1 - rr is 1 either way
          sg[sk(t * RUN + k)] = n < T ? rr : 0.f;
          if (k + 1 < RUN) s += (double)sd[sk(i + A + 1)] - (double)sd[sk(i - A)];
        }
      }
      __syncthreads();
    }
    const float g0 = gain ? __ldg(gain + b) : 1.f;
    const bool copy = !(quiet && gain == nullptr && out == x);
    const int64_t len = T - c0 < CHUNK ? T - c0 : CHUNK;
    if (VEC) {
      for (int t = 4 * threadIdx.x; t < len; t += 4 * NT) {
        float4 rr = make_float4(0.f, 0.f, 0.f, 0.f);
        if (!quiet) rr = make_float4(sg[sk(t)], sg[sk(t + 1)], sg[sk(t + 2)], sg[sk(t + 3)]);
        if (red) st_stream4(red + b * T + c0 + t, rr);
        const float4 g = make_float4(1.f - rr.x, 1.f - rr.y, 1.f - rr.z, 1.f - rr.w);
        if (copy)
          for (int c = 0; c < C; ++c) {
            const int64_t at = (b * C + c) * T + c0 + t;
            float4 q = *reinterpret_cast<const float4*>(x + at);  // not the read-only path: out may be x
            q = make_float4(q.x * g0 * g.x, q.y * g0 * g.y, q.z * g0 * g.z, q.w * g0 * g.w);
            st_stream4(out + at, q);
          }
      }
    } else {
      for (int t = threadIdx.x; t < len; t += NT) {
        const float rr = quiet ? 0.f : sg[sk(t)];
        if (red) red[b * T + c0 + t] = rr;
        if (copy)
          for (int c = 0; c < C; ++c) {
            const int64_t at = (b * C + c) * T + c0 + t;
            out[at] = x[at] * g0 * (1.f - rr);
          }
      }
    }
    __syncthreads();  // the next work item overwrites the shared buffers
  }
}

}  // namespace limiter
}  // namespace b2a

using namespace b2a::limiter;

static int64_t limiter_chunks(int64_t T) { return (T + CHUNK - 1) / CHUNK; }

extern "C" size_t b2a_limiter_workspace_bytes(int64_t B, int C, int64_t T) {
  if (B < 1 || C < 1 || T < 1 || T > INT64_MAX / 8 / B / C) return 0;
  return (size_t)(B * T + 3 * B * limiter_chunks(T)) * sizeof(float);
}

extern "C" int b2a_limiter_f32(const float* x, const float* gain, int64_t B, int C, int64_t T, int factor,
                               const float* ceiling, int lookahead, float release_a, float* out, float* reduction,
                               void* ws, void* stream) {
  B2A_REQUIRE(x && ceiling && out && ws, B2A_E_INVALID, "limiter: null pointer");
  B2A_REQUIRE(B >= 1 && C >= 1 && T >= 1, B2A_E_INVALID, "limiter: bad shape B=%lld C=%d T=%lld", (long long)B, C,
              (long long)T);
  B2A_REQUIRE(T <= INT64_MAX / 8 / B / C, B2A_E_INVALID, "limiter: B * C * T overflows");
  B2A_REQUIRE(lookahead >= 0 && lookahead <= AMAX, B2A_E_INVALID, "limiter: lookahead of %d samples is not in 0 .. %d",
              lookahead, AMAX);
  B2A_REQUIRE(release_a >= 0.f && release_a < 1.f, B2A_E_INVALID,
              "limiter: release coefficient %g is not in [0, 1): the release must be positive and at most about 1e7 samples",
              (double)release_a);
  Taps taps;
  const int rc = design(factor, &taps);
  if (rc != B2A_OK) return rc;
  const double a = (double)release_a;
  Decay dec;
  for (int k = 0; k <= RUN; ++k) dec.p1[k] = (float)pow(a, (double)k);
  for (int m = 0; m <= 32; ++m) dec.p16[m] = (float)pow(a, 16.0 * m);
  for (int m = 0; m <= TPB3 / 32; ++m) dec.p512[m] = (float)pow(a, 512.0 * m);
  const int A = lookahead, Ap = (A + RUN - 1) / RUN * RUN, W = CHUNK + 2 * Ap;
  const int64_t n_chunks = limiter_chunks(T), work = B * n_chunks;
  const unsigned grid = (unsigned)(work < INT32_MAX ? work : INT32_MAX);
  float* h = static_cast<float*>(ws);
  float* em = h + B * T;
  float* hc = em + 2 * B * n_chunks;
  const int Wp = W + (W >> 4);
  const int smem1 = 2 * Wp * (int)sizeof(float);
  const int smem3 = TPB3 * (int)sizeof(double) + (Wp + CHUNK + (CHUNK >> 4)) * (int)sizeof(float);
  auto k1 = factor == 4 ? envelope_hold_kernel<3> : factor == 2 ? envelope_hold_kernel<1> : envelope_hold_kernel<0>;
  const bool vec = T % 4 == 0 && (((uintptr_t)x | (uintptr_t)out | (uintptr_t)reduction) & 15) == 0;
  auto k3 = vec ? release_apply_kernel<true> : release_apply_kernel<false>;
  B2A_CUDA_OK(cudaFuncSetAttribute(k1, cudaFuncAttributeMaxDynamicSharedMemorySize, smem1));
  B2A_CUDA_OK(cudaFuncSetAttribute(k3, cudaFuncAttributeMaxDynamicSharedMemorySize, smem3));
  B2A_LAUNCH(k1, dim3(grid), dim3(TPB), smem1, stream, x, gain, C, T, n_chunks, work, A, Ap, ceiling, taps, dec, h, em);
  B2A_CUDA_OK(cudaGetLastError());
  B2A_LAUNCH(carry_kernel, dim3((unsigned)((B * 32 + TPB - 1) / TPB)), dim3(TPB), 0, stream, em, B, n_chunks, log2(a),
             Ap, hc);
  B2A_CUDA_OK(cudaGetLastError());
  const int nt3 = (W / RUN + 31) / 32 * 32;
  B2A_LAUNCH(k3, dim3(grid), dim3(nt3), smem3, stream, x, gain, C, T, n_chunks, work, A, Ap, h, hc, dec, out, reduction);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}
