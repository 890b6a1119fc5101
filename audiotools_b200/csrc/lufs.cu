// lufs.cu -- integrated loudness (ITU-R BS.1770) for [B, C, T] float32 waveforms on sm_90a.
//
// Replaces the device work of Meter.integrated_loudness with the exact-IIR semantics of
// Meter.apply_filter_cpu (ref:audiotools/core/loudness.py:102-126) -- NOT the 512-tap FIR
// approximation the reference falls back to on CUDA (:69-100) -- followed by the 400 ms / 75 %
// block energies (:164-174, 214) and the two-pass gating (:208-247).
//
// Kernel 1  kweight_energy_warp_kernel   (HBM-bound: 4 B/sample, plus the warm-up reads)
//   The cascade of NS biquads is a linear recurrence with a 2*NS-dim state.  A row is cut into RUNS of run_len
//   consecutive segments (segment = 32 lanes x L2 = 64 samples = 2048 samples); a WARP owns a run and walks it segment
//   by segment, with no CTA barrier and no inter-warp communication: samples -> warp-private, double-buffered
//   shared-memory window (cp.async; the next segment lands underneath the arithmetic of the current one), zero-state
//   end state of every lane chunk (a 66-tap linear map read from the window, split table), affine shuffle scan over
//   the 32 chunks (state' = A^64 state + e), true lane start states from the state carried in registers, float32 DF-I
//   recursion (second read of the window), y^2 into "elementary interval" bins:
//   with K = q*stride + r, interval A_j = [j*stride, j*stride+r), B_j = [j*stride+r, (j+1)*stride),
//   so that block i = sum_{j=i}^{i+q-1}(A_j + B_j) + A_{i+q} -- bit-exact block indexing for any
//   rate (K is not always 4*stride, e.g. 11025 Hz).  Warp partials are added into float64 bins.
//
//   The state entering a run comes from a WARM-UP, not from an exact carry across runs (which would need a serial
//   hand-off from the warp of the previous run, or a second pass over x): the warp first runs the carry part (no
//   energies) over the n_warm segments in front of its run, starting from zero.  The K-weighting poles have radius
//   rho < 1 (0.9946 for the 38 Hz high-pass at 44.1 kHz), so whatever happened before the warm-up reaches the run
//   attenuated by rho^(n_warm * 2048); the host picks n_warm with rho^(n_warm * 2048) <= 2^-40 (3 segments at
//   44.1 kHz, 18 % extra reads at run_len 17).  That bound is five orders of magnitude below the rounding noise the
//   float32 recursion itself carries (each step rounds at 6e-8 |y| and the feedback amplifies it by ~1/(1 - rho)),
//   i.e. the results are those of the exact carry to float32 rounding; only a row whose level drops by more than
//   2^40 across one warm-up can tell the two apart.
//
//   State basis.  The high-pass is a (near) double pole at rho ~ 1 - 2 pi 38 Hz / rate.  On the output history
//   (y[n-1], y[n-2]) its powers A^n have entries up to ~1 / (e (1 - rho)) (74 at 48 kHz, 300 at 192 kHz) that cancel
//   to an O(1) result, so float32-rounded tables put a systematic error into every lane start state, and bass-heavy
//   rows came out ~10x less accurate than the sequential float32 cascade.  The scan, the carry and the start states
//   therefore run on w = (y[n-1] - rho y[n-2], y[n-2]) per stage (rho rounded to float32, so y[n-1] = fma(rho, w1, w0)
//   converts back with one rounding): there A^n is a Jordan block without cancellation.  The end-state map keeps a
//   cancelling sum in any basis, so its table is split into float32 high and low halves, summed in two accumulators
//   (a rounded table is a systematic error; the accumulators' roundings are not).  tests/probes/kweight_state_probe.py
//   measures each stage.
// Kernel 2  lufs_gate_kernel             (tiny: one CTA per item)
//   z -> l -> absolute gate -> relative gate -> LUFS, with the reference's dtypes (float32 z,
//   float64 logs) and its NaN / inf scrubbing; optionally max(.,-70) and normalize()'s gain.
#include "b2a_common.h"

namespace b2a {
namespace lufs {

constexpr int L2 = 64;              // samples per lane
constexpr int SEG = 32 * L2;        // samples per warp segment
constexpr int CHS = L2 + 4;         // shared-memory words per lane chunk: 16 B aligned, conflict-free LDS.128
constexpr int WPB = 12;             // warps per CTA (one CTA per SM: 12 x 17 KB of windows)
constexpr int NBUF = 2;             // windows per warp: the next segment lands underneath the arithmetic
constexpr int BUF = 32 * CHS;       // floats per window
constexpr int MAX_STAGES = 2;
// Unit of the input range b2a_lufs_f32 accepts: rows shorter than 2^31 - 2 TILE samples (every sample index the
// kernels form, including the segment that runs past a row's end, fits an int), fewer than 2^31 tiles per batch.
constexpr int TILE = 8192;

template <int NS>
struct Coef {  // from the float32-rounded, a0-normalised b (stage gain folded in): d0 = b0, d1 = b0 + b1, d2 = b0 + b1 + b2
  float d0[NS], d1[NS], d2[NS], a1[NS], a2[NS];
};

__host__ __device__ inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

struct WsLayout {
  size_t bins, zeroed_bytes, zws, total;
};
// the interval bins are accumulated with atomics and come first: the call zeroes [0, zeroed_bytes)
__host__ inline WsLayout ws_layout(int64_t rows, int64_t nbins, int64_t nblk) {
  WsLayout w;
  size_t o = 0;
  w.bins = o; o = align256(o + sizeof(double) * rows * nbins);
  w.zeroed_bytes = o;
  w.zws = o; o = align256(o + sizeof(float) * rows * nblk);
  w.total = o;
  return w;
}

// one step of the cascade: DF-I with the feed-forward sum b0 in0 + b1 in1 + b2 in2 in difference form,
// d0 (in0 - in1) + d1 (in1 - in2) + d2 in2.  For the high-pass (b = g (1, -2, 1): d1 = -d0, d2 = 0) the differences of
// slowly varying samples are exact, so the sum carries a rounding of its own size, not of the samples' (the direct form
// under FMA contraction rounds one product only and leaves u |x|, which the poles near 1 amplify by ~1 / (1 - rho)^2 on
// DC and bass).  The FMAs are written out so that the simulator rounds as the GPU does.
template <int NS, class F>
__host__ __device__ __forceinline__ F cascade_step(const F (&d0)[NS], const F (&d1)[NS], const F (&d2)[NS],
                                                    const F (&a1)[NS], const F (&a2)[NS], F in0, F in1, F in2,
                                                    F (&y1)[NS], F (&y2)[NS]) {
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    F f = fma(d0[s], in0 - in1, fma(d1[s], in1 - in2, d2[s] * in2));
    F y0 = fma(-a1[s], y1[s], fma(-a2[s], y2[s], f));
    in0 = y0; in1 = y1[s]; in2 = y2[s];
    y2[s] = y1[s]; y1[s] = y0;
  }
  return in0;
}

// ---------------------------------------------------------------------------------------------
// tables: state-transition matrix powers and the lane-chunk end-state map, float64 on the host (a few microseconds),
// handed to the kernel as a __grid_constant__ parameter -- no set-up launch, no device buffer
// ---------------------------------------------------------------------------------------------
template <int D>
static void matmul(const double* a, const double* b, double* c) {
  double t[D * D];
  for (int i = 0; i < D; ++i)
    for (int j = 0; j < D; ++j) {
      double s = 0;
      for (int k = 0; k < D; ++k) s += a[i * D + k] * b[k * D + j];
      t[i * D + j] = s;
    }
  for (int i = 0; i < D * D; ++i) c[i] = t[i];
}

template <int NS>
struct Tables {  // on the state basis w = B (y1, y2): per stage (y1 - rho y2, y2)
  static constexpr int D = 2 * NS;
  float Wa[L2 + 2][D];        // zero-state end state of a lane chunk as a linear map of its 66 inputs: high half
  float Wlo[L2 + 2][D];       // and low half (Wa + Wlo = the float64 map to ~2^-48)
  float Mlane[32][D * D];     // A^(L2 l)
  float Mscan[5][D * D];      // A^(L2 2^k)
  float Mseg[D * D];          // A^SEG
  float rho[NS];              // y1 = rho y2 + w0
};

template <int NS>
static double max_pole_radius(const Coef<NS>& cf, int s0 = 0, int s1 = NS);

template <int NS>
static void build_tables(const Coef<NS>& cf, Tables<NS>* tb) {
  constexpr int D = 2 * NS;
  double b0[NS], b1[NS], b2[NS], a1[NS], a2[NS];
  for (int s = 0; s < NS; ++s) {
    b0[s] = cf.d0[s]; b1[s] = cf.d1[s]; b2[s] = cf.d2[s]; a1[s] = cf.a1[s]; a2[s] = cf.a2[s];
  }
  double A[D * D];
  for (int k = 0; k < D; ++k) {
    double y1[NS], y2[NS];
    for (int s = 0; s < NS; ++s) { y1[s] = (k == 2 * s) ? 1.0 : 0.0; y2[s] = (k == 2 * s + 1) ? 1.0 : 0.0; }
    cascade_step<NS, double>(b0, b1, b2, a1, a2, 0.0, 0.0, 0.0, y1, y2);
    for (int s = 0; s < NS; ++s) { A[(2 * s) * D + k] = y1[s]; A[(2 * s + 1) * D + k] = y2[s]; }
  }
  // basis change w = Bm y and its inverse, per stage [[1, -rho], [0, 1]]
  double Bm[D * D], Bi[D * D];
  for (int i = 0; i < D * D; ++i) Bm[i] = Bi[i] = (i / D == i % D) ? 1.0 : 0.0;
  for (int s = 0; s < NS; ++s) {
    tb->rho[s] = (float)max_pole_radius<NS>(cf, s, s + 1);
    Bm[(2 * s) * D + 2 * s + 1] = -(double)tb->rho[s];
    Bi[(2 * s) * D + 2 * s + 1] = (double)tb->rho[s];
  }
  matmul<D>(Bm, A, A);
  matmul<D>(A, Bi, A);  // A on the w basis
  double P[D * D];  // A^L2
  for (int i = 0; i < D * D; ++i) P[i] = A[i];
  for (int l = 1; l < L2; l <<= 1) matmul<D>(P, P, P);
  double Q[D * D];
  for (int i = 0; i < D * D; ++i) Q[i] = (i / D == i % D) ? 1.0 : 0.0;
  for (int l = 0; l < 32; ++l) {
    for (int i = 0; i < D * D; ++i) tb->Mlane[l][i] = (float)Q[i];
    matmul<D>(P, Q, Q);
  }
  for (int i = 0; i < D * D; ++i) tb->Mseg[i] = (float)Q[i];  // Q == A^SEG
  double S[D * D];
  for (int i = 0; i < D * D; ++i) S[i] = P[i];
  for (int k = 0; k < 5; ++k) {
    for (int i = 0; i < D * D; ++i) tb->Mscan[k][i] = (float)S[i];
    matmul<D>(S, S, S);
  }
  for (int j = 0; j < L2 + 2; ++j) {
    double y1[NS], y2[NS];
    for (int s = 0; s < NS; ++s) { y1[s] = 0.0; y2[s] = 0.0; }
    for (int i = 0; i < L2; ++i) {
      const double in0 = (i + 2 == j) ? 1.0 : 0.0, in1 = (i + 1 == j) ? 1.0 : 0.0, in2 = (i == j) ? 1.0 : 0.0;
      cascade_step<NS, double>(b0, b1, b2, a1, a2, in0, in1, in2, y1, y2);
    }
    for (int s = 0; s < NS; ++s) {
      const double w[2] = {y1[s] - (double)tb->rho[s] * y2[s], y2[s]};
      for (int c = 0; c < 2; ++c) {
        tb->Wa[j][2 * s + c] = (float)w[c];
        tb->Wlo[j][2 * s + c] = (float)(w[c] - (double)tb->Wa[j][2 * s + c]);
      }
    }
  }
}

// largest pole radius of stages [s0, s1) of the cascade (a1, a2 already normalised by a0)
template <int NS>
static double max_pole_radius(const Coef<NS>& cf, int s0, int s1) {
  double rho = 0.0;
  for (int s = s0; s < s1; ++s) {
    const double a1 = cf.a1[s], a2 = cf.a2[s], disc = a1 * a1 - 4.0 * a2;
    double r;
    if (disc < 0) r = sqrt(a2 > 0 ? a2 : 0.0);
    else r = 0.5 * (fabs(a1) + sqrt(disc));
    if (r > rho) rho = r;
  }
  return rho;
}

// cp.async (16 B) global -> shared; plain copy under the CPU simulator
__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gmem_src) {
#ifdef B2A_SIM
  *reinterpret_cast<float4*>(smem_dst) = *reinterpret_cast<const float4*>(gmem_src);
#else
  const unsigned sa = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(gmem_src) : "memory");
#endif
}
__device__ __forceinline__ void cp_async_wait_all() {
#ifndef B2A_SIM
  asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
#endif
}

template <int D>
__device__ __forceinline__ float row_dot(const float* M, int i, const float* v) {
  float a = 0.f;
#pragma unroll
  for (int j = 0; j < D; ++j) a = fmaf(M[i * D + j], v[j], a);
  return a;
}

// Stage segment `seg` of row `xr` into a warp window (cp.async when the 8 KB are inside the row and 16 B aligned).
__device__ __forceinline__ void stage_segment(const float* __restrict__ xr, int seg, int T, float* win, int lane) {
  const int t0 = seg * SEG;
  if ((t0 + SEG <= T) && ((((uintptr_t)(xr + t0)) & 15) == 0)) {
#pragma unroll
    for (int i = 0; i < L2 / 4; ++i) {
      const int s = 128 * i + 4 * lane;  // sample index within the segment (16 B per lane: coalesced)
      cp_async16(&win[CHS * (s >> 6) + (s & 63)], xr + t0 + s);
    }
  } else {
    for (int s = lane; s < SEG; s += 32) {
      const int n = t0 + s;
      win[CHS * (s >> 6) + (s & 63)] = (n < T) ? __ldg(xr + n) : 0.f;
    }
  }
}

template <int NS>
__global__ void __launch_bounds__(32 * WPB, 1)
kweight_energy_warp_kernel(const float* __restrict__ x, int rows, int T, int Tp, int nseg, int run_len, int n_runs,
                           int n_warm, Coef<NS> cf, const B2A_GRID_CONSTANT Tables<NS> tbv,
                           double* __restrict__ bins, int stride, int r, int nbins) {
  constexpr int D = 2 * NS;
  B2A_DYN_SMEM(smem);
  float* wins = reinterpret_cast<float*>(smem);  // [WPB][NBUF][BUF]
  __shared__ float s_mlane[32][D * D];
  __shared__ float s_mscan[5][D * D];
  __shared__ float s_mseg[D * D];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < 32 * D * D; i += blockDim.x) (&s_mlane[0][0])[i] = (&tbv.Mlane[0][0])[i];
  for (int i = tid; i < 5 * D * D; i += blockDim.x) (&s_mscan[0][0])[i] = (&tbv.Mscan[0][0])[i];
  if (tid < D * D) s_mseg[tid] = tbv.Mseg[tid];
  __syncthreads();  // the only CTA barrier: tables
  const int total = rows * n_runs;
  float* win0 = wins + (size_t)warp * NBUF * BUF;

#pragma unroll 1
  for (int cur = (int)blockIdx.x * WPB + warp; cur < total; cur += (int)gridDim.x * WPB) {
    const int run = cur / rows, row = cur - run * rows;
    const int seg0 = run * run_len, seg1 = min(nseg, seg0 + run_len);
    const int segw = max(0, seg0 - n_warm);  // warm-up starts here, from a zero state
    const float* xr = x + (size_t)row * (size_t)T;
    double* rb = bins + (size_t)row * (size_t)nbins;
    float carry[D];  // state entering the current segment (all lanes hold it)
#pragma unroll
    for (int j = 0; j < D; ++j) carry[j] = 0.f;
    stage_segment(xr, segw, T, win0, lane);
    int par = 0;
#pragma unroll 1
    for (int seg = segw; seg < seg1; ++seg, par ^= (NBUF - 1)) {
      cp_async_wait_all();
      __syncwarp();
      const float* win = win0 + par * BUF;
      if (NBUF == 2 && seg + 1 < seg1) stage_segment(xr, seg + 1, T, win0 + (par ^ 1) * BUF, lane);
      const int t0 = seg * SEG;
      float h0, h1;  // the two samples in front of this lane's chunk
      if (lane == 0) {
        h0 = (t0 >= 2 && t0 - 2 < T) ? __ldg(xr + t0 - 2) : 0.f;
        h1 = (t0 >= 1 && t0 - 1 < T) ? __ldg(xr + t0 - 1) : 0.f;
      } else {
        const float2 h = *reinterpret_cast<const float2*>(&win[CHS * (lane - 1) + L2 - 2]);
        h0 = h.x; h1 = h.y;
      }
      const float4* c4 = reinterpret_cast<const float4*>(&win[CHS * lane]);
      // ---- zero-state end state of the lane's chunk as a linear map of its 66 inputs (high and low table halves)
      float g[D];
      {
        float gl[D];
#pragma unroll
        for (int i = 0; i < D; ++i) {
          g[i] = fmaf(tbv.Wa[0][i], h0, tbv.Wa[1][i] * h1);
          gl[i] = fmaf(tbv.Wlo[0][i], h0, tbv.Wlo[1][i] * h1);
        }
#pragma unroll
        for (int i4 = 0; i4 < L2 / 4; ++i4) {
          const float4 q = c4[i4];
          const float qs[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
#pragma unroll
            for (int i = 0; i < D; ++i) {  // constant-bank operands
              g[i] = fmaf(tbv.Wa[2 + 4 * i4 + e][i], qs[e], g[i]);
              gl[i] = fmaf(tbv.Wlo[2 + 4 * i4 + e][i], qs[e], gl[i]);
            }
          }
        }
#pragma unroll
        for (int i = 0; i < D; ++i) g[i] += gl[i];
      }
#pragma unroll
      for (int k = 0; k < 5; ++k) {  // inclusive affine scan over the 32 chunks
        float o[D];
#pragma unroll
        for (int j = 0; j < D; ++j) o[j] = __shfl_up_sync(0xffffffffu, g[j], 1u << k);
        if (lane >= (1 << k)) {
#pragma unroll
          for (int i = 0; i < D; ++i) g[i] += row_dot<D>(tbv.Mscan[k], i, o);  // (k is unrolled: constant-bank operands)
        }
      }
      float ex[D], agg[D];
#pragma unroll
      for (int j = 0; j < D; ++j) {
        ex[j] = __shfl_up_sync(0xffffffffu, g[j], 1);
        if (lane == 0) ex[j] = 0.f;
        agg[j] = __shfl_sync(0xffffffffu, g[j], 31);
      }
      if (seg >= seg0) {
        // ---- true start state, recursion, energies into the interval bins
        float y1[NS], y2[NS];
        {
          float st[D];
#pragma unroll
          for (int i = 0; i < D; ++i) st[i] = ex[i] + row_dot<D>(s_mlane[lane], i, carry);
#pragma unroll
          for (int s = 0; s < NS; ++s) { y1[s] = fmaf(tbv.rho[s], st[2 * s + 1], st[2 * s]); y2[s] = st[2 * s + 1]; }
        }
        const int n0 = t0 + lane * L2;
        const int nv = min(L2, max(0, Tp - n0));
        int j0 = n0 / stride, rem0 = n0 - j0 * stride;
        int b0 = 2 * j0 + (rem0 >= r ? 1 : 0);
        int end0 = (b0 & 1) ? (j0 + 1) * stride : j0 * stride + r;
        const int s1 = min(end0 - n0, L2);
        int s2 = L2, b1 = b0, b2 = b0;
        if (s1 < L2) {
          const int n1 = n0 + s1, j1 = n1 / stride, rem1 = n1 - j1 * stride;
          b1 = 2 * j1 + (rem1 >= r ? 1 : 0);
          const int end1 = (b1 & 1) ? (j1 + 1) * stride : j1 * stride + r;
          s2 = min(end1 - n0, L2);
          if (s2 < L2) {
            const int n2 = n0 + s2, j2 = n2 / stride, rem2 = n2 - j2 * stride;
            b2 = 2 * j2 + (rem2 >= r ? 1 : 0);
          }
        }
        const bool simple = (s1 >= L2) && (nv == L2);
        const bool clean = __all_sync(0xffffffffu, simple);  // warp-uniform: no lane straddles an interval boundary
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
        float xm2 = h0, xm1 = h1;
        if (clean) {
          float acc = 0.f;
#pragma unroll
          for (int i4 = 0; i4 < L2 / 4; ++i4) {
            const float4 q = c4[i4];
            const float qs[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float y = cascade_step<NS, float>(cf.d0, cf.d1, cf.d2, cf.a1, cf.a2, qs[e], xm1, xm2, y1, y2);
              xm2 = xm1; xm1 = qs[e];
              acc = fmaf(y, y, acc);
            }
          }
          a0 = acc;
        } else {
          // one sum per interval, restarted at each boundary (differences of a running sum would put the rounding
          // of a loud interval into a quiet neighbour)
          float acc = 0.f, p1 = 0.f, p2 = 0.f;
#pragma unroll
          for (int i4 = 0; i4 < L2 / 4; ++i4) {
            const float4 q = c4[i4];
            const float qs[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int i = 4 * i4 + e;
              p1 = (i == s1) ? acc : p1;
              p2 = (i == s2) ? acc : p2;
              acc = (i == s1 || i == s2) ? 0.f : acc;
              const float y = cascade_step<NS, float>(cf.d0, cf.d1, cf.d2, cf.a1, cf.a2, qs[e], xm1, xm2, y1, y2);
              xm2 = xm1; xm1 = qs[e];
              acc = (i < nv) ? fmaf(y, y, acc) : acc;
            }
          }
          if (s1 >= L2) { p1 = acc; acc = 0.f; }
          else if (s2 >= L2) { p2 = acc; acc = 0.f; }
          a0 = p1; a1 = p2; a2 = acc;
        }
        // one atomic per interval the warp touched (intervals are monotonic in the lane index)
        const int blast = (s2 < L2) ? b2 : ((s1 < L2) ? b1 : b0);  // last interval this lane's chunk reaches
        const int bf = __shfl_sync(0xffffffffu, b0, 0), bl = __shfl_sync(0xffffffffu, blast, 31);
        for (int id = bf; id <= bl; ++id) {
          float v = (b0 == id) ? a0 : 0.f;
          if (!clean) v += ((s1 < L2 && b1 == id) ? a1 : 0.f) + ((s2 < L2 && b2 == id) ? a2 : 0.f);
          v = warp_sum(v);
          if (lane == 0 && id < nbins) atomicAdd(rb + id, (double)v);
        }
      }
      // ---- carry into the next segment: A^SEG carry + (zero-state end state of this segment)
      float cn[D];
#pragma unroll
      for (int i = 0; i < D; ++i) cn[i] = agg[i] + row_dot<D>(tbv.Mseg, i, carry);
#pragma unroll
      for (int i = 0; i < D; ++i) carry[i] = cn[i];
      __syncwarp();  // every lane is done with this window before it is refilled
      if (NBUF == 1 && seg + 1 < seg1) stage_segment(xr, seg + 1, T, win0, lane);
    }
  }
  cp_async_wait_all();
}

// ---------------------------------------------------------------------------------------------
// gating: ref:audiotools/core/loudness.py:208-247 (+ :315-320 clamp, effects.py:214-217 gain)
// ---------------------------------------------------------------------------------------------
constexpr int GT = 128;

template <class T>
__device__ T block_sum(T v, T* scratch) {
  __syncthreads();
  scratch[threadIdx.x] = v;
  __syncthreads();
  for (int s = GT / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) scratch[threadIdx.x] += scratch[threadIdx.x + s];
    __syncthreads();
  }
  return scratch[0];
}

struct GateParams {
  double G[8];
  float scale;  // float32(1 / (block_s * rate))
  int C, nblk, nbins, q;
};

__global__ void __launch_bounds__(GT)
lufs_gate_kernel(const double* __restrict__ bins, GateParams gp, float* __restrict__ zws,
                 float* __restrict__ z_out, float* __restrict__ lufs_out, float* __restrict__ loud_out,
                 const float* __restrict__ target_db, int n_target, float* __restrict__ gain_out) {
  __shared__ double sd[GT];
  __shared__ int si[GT];
  const int b = blockIdx.x, C = gp.C, nblk = gp.nblk, q = gp.q;
  const int tid = threadIdx.x;
  float* z = zws + (size_t)b * C * nblk;
  // z[c][i] = float32(sum of the block's interval energies) * float32(1/(T_g*rate))   (:214)
  for (int idx = tid; idx < C * nblk; idx += GT) {
    int c = idx / nblk, i = idx - c * nblk;
    const double* rb = bins + ((size_t)b * C + c) * gp.nbins;
    double s = 0.0;
    for (int j = i; j < i + q; ++j) s += rb[2 * j] + rb[2 * j + 1];
    s += rb[2 * (i + q)];
    float zf = (float)s * gp.scale;
    z[idx] = zf;
    if (z_out) z_out[(size_t)b * C * nblk + idx] = zf;
  }
  __syncthreads();
  const double Gamma_a = -70.0;
  // pass 1: absolute gate
  double sum1[8];
  for (int c = 0; c < C; ++c) sum1[c] = 0.0;
  int n1 = 0;
  for (int i = tid; i < nblk; i += GT) {
    double acc = 0.0;
    for (int c = 0; c < C; ++c) acc += gp.G[c] * (double)z[c * nblk + i];
    double l = -0.691 + 10.0 * log10(acc);
    // z[l <= Ga] = 0 (a NaN l is NOT zeroed), masked = l > Ga (a NaN l is NOT counted)
    if (!(l <= Gamma_a))
      for (int c = 0; c < C; ++c) sum1[c] += (double)z[c * nblk + i];
    if (l > Gamma_a) n1++;
  }
  int n1t = block_sum<int>(n1, si);
  double gr_acc = 0.0;
  for (int c = 0; c < C; ++c) {
    float zs = (float)block_sum<double>(sum1[c], sd);  // float32 sum in the reference
    float zavg = zs / (float)n1t;                      // 0/0 -> NaN as in the reference
    gr_acc += (double)zavg * gp.G[c];
  }
  const double Gamma_r = -0.691 + 10.0 * log10(gr_acc) - 10.0;
  // pass 2: absolute + relative gate (comparisons with NaN are false, as in torch)
  double sum2[8];
  for (int c = 0; c < C; ++c) sum2[c] = 0.0;
  int n2 = 0;
  for (int i = tid; i < nblk; i += GT) {
    double acc = 0.0;
    for (int c = 0; c < C; ++c) acc += gp.G[c] * (double)z[c * nblk + i];
    double l = -0.691 + 10.0 * log10(acc);
    // z[l <= Ga] = 0; z[l <= Gr] = 0  ->  a block survives iff !(l <= Ga) && !(l <= Gr)
    bool zeroed = (l <= Gamma_a) || (l <= Gamma_r);
    if (!zeroed)
      for (int c = 0; c < C; ++c) sum2[c] += (double)z[c * nblk + i];
    if ((l > Gamma_a) && (l > Gamma_r)) n2++;
  }
  int n2t = block_sum<int>(n2, si);
  double lacc = 0.0;
  for (int c = 0; c < C; ++c) {
    float zs = (float)block_sum<double>(sum2[c], sd);
    float zavg = zs / (float)n2t;
    if (zavg != zavg) zavg = 0.f;                              // nan -> 0          (:240-242)
    if (zavg == INFINITY) zavg = 3.4028234663852886e38f;       // +inf -> f32 max   (:243)
    if (zavg == -INFINITY) zavg = -3.4028234663852886e38f;     // -inf -> f32 min   (:244)
    lacc += gp.G[c] * (double)zavg;
  }
  if (tid == 0) {
    float lufs = (float)(-0.691 + 10.0 * log10(lacc));
    lufs_out[b] = lufs;
    float loud = fmaxf(lufs, -70.0f);  // MIN_LOUDNESS (:265, :315-320)
    if (loud_out) loud_out[b] = loud;
    if (gain_out) {
      float db = target_db[n_target == 1 ? 0 : b];
      float gdb = db - loud;
      gain_out[b] = expf(gdb * 0.11512925464970229f);  // GAIN_FACTOR = ln(10)/20 (effects.py:12)
    }
  }
}

// ---------------------------------------------------------------------------------------------
// per-item gain
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
gain_kernel(const float* __restrict__ x, float* __restrict__ out, int64_t per_item, const float* __restrict__ gain,
            int vec_ok) {
  const int b = blockIdx.y;
  const float g = __ldg(gain + b);
  const float* xi = x + (size_t)b * per_item;
  float* oi = out + (size_t)b * per_item;
  const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (vec_ok) {
    const int64_t n4 = per_item >> 2;
    for (int64_t i = gid; i < n4; i += nthreads) {
      float4 v = ld_stream4(xi + 4 * i);
      v.x *= g; v.y *= g; v.z *= g; v.w *= g;
      st_stream4(oi + 4 * i, v);
    }
    for (int64_t i = (n4 << 2) + gid; i < per_item; i += nthreads) oi[i] = xi[i] * g;
  } else {
    for (int64_t i = gid; i < per_item; i += nthreads) oi[i] = xi[i] * g;
  }
}

struct Geometry {
  int K, stride, q, r, nblk, nbins, nseg;
};
static int geometry(int64_t Tp, double rate, double block_s, Geometry* g) {
  double kf = block_s * rate;
  int64_t K = (int64_t)kf;                 // int(T_g * rate)            (:168)
  int64_t stride = (int64_t)(kf * 0.25);   // int(T_g * rate * step)     (:169)
  if (K < 1 || stride < 64) return -1;
  int64_t d = (Tp > K ? Tp : K) - K;
  int64_t nblk = (d + stride - 1) / stride + 1;  // julius.core.unfold
  g->K = (int)K; g->stride = (int)stride; g->q = (int)(K / stride); g->r = (int)(K % stride);
  g->nblk = (int)nblk;
  g->nbins = 2 * (int)(nblk + g->q);
  g->nseg = (int)((Tp + SEG - 1) / SEG);  // warp segments per row
  return 0;
}

template <int NS>
static int run(const float* x, int64_t B, int C, int64_t T, int64_t Tp, const Geometry& g, const double* sos_h,
               const double* stage_gain_h, double rate, double block_s, const double* chan_gain_h,
               float* z_blocks, float* lufs_out, float* loud_out, const float* target_db, int n_target,
               float* gain_out, void* ws, size_t ws_bytes, void* stream) {
  const int64_t rows = B * C;
  WsLayout w = ws_layout(rows, g.nbins, g.nblk);
  B2A_REQUIRE(ws_bytes >= w.total, B2A_E_INVALID, "lufs: workspace too small (%zu < %zu)", ws_bytes, w.total);
  Coef<NS> cf;
  for (int s = 0; s < NS; ++s) {
    const double* c = sos_h + 6 * s;
    B2A_REQUIRE(c[3] != 0.0, B2A_E_INVALID, "lufs: a0 == 0 in stage %d", s);
    // the reference casts b and a to float32 (:118-119); lfilter then divides by a0 (== 1.0 for pyloudnorm)
    float a0 = (float)c[3];
    float sg = (float)stage_gain_h[s];
    const float b0 = (float)c[0] / a0 * sg, b1 = (float)c[1] / a0 * sg, b2 = (float)c[2] / a0 * sg;
    cf.d0[s] = b0;
    cf.d1[s] = (float)((double)b0 + b1);
    cf.d2[s] = (float)((double)b0 + b1 + b2);
    cf.a1[s] = (float)c[4] / a0; cf.a2[s] = (float)c[5] / a0;
  }
  char* base = (char*)ws;
  B2A_CUDA_OK(cudaMemsetAsync(base, 0, w.zeroed_bytes, (cudaStream_t)stream));
  // runs per row: as many as there are resident warps for (one CTA of 12 warps per SM), but long enough that the
  // warm-up (n_warm segments in front of every run but the first) stays a small fraction of the work
#ifdef B2A_SIM
  const int64_t resident = 1;
#else
  const int64_t resident = num_sms();
#endif
  const double rho = max_pole_radius<NS>(cf);
  B2A_REQUIRE(rho < 1.0, B2A_E_UNSUPPORTED, "lufs: unstable filter (pole radius %g)", rho);
  int n_warm = 1;
  if (rho > 0.0) {
    const double n_tail = 40.0 * 0.6931471805599453 / -log(rho);  // rho^n_tail = 2^-40
    n_warm = (int)((n_tail + SEG - 1) / SEG);
    if (n_warm < 1) n_warm = 1;
  }
  int64_t rpr = (resident * WPB) / rows;
  if (rpr < 1) rpr = 1;
  int run_len = (int)((g.nseg + rpr - 1) / rpr);
  if (run_len < 4 * n_warm) run_len = 4 * n_warm;  // at most 25 % warm-up
  if (run_len > g.nseg) run_len = g.nseg;
  const int n_runs = (g.nseg + run_len - 1) / run_len;
  Tables<NS> tb;
  build_tables<NS>(cf, &tb);
  const int64_t runs_all = rows * n_runs;
  const int64_t want = (runs_all + WPB - 1) / WPB;
  const unsigned grid = (unsigned)(want < resident ? want : resident);
  const size_t smem = (size_t)WPB * NBUF * BUF * sizeof(float);
  B2A_CUDA_OK(cudaFuncSetAttribute(kweight_energy_warp_kernel<NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  B2A_LAUNCH(kweight_energy_warp_kernel<NS>, dim3(grid), dim3(32 * WPB), smem, stream, x, (int)rows, (int)T, (int)Tp,
             g.nseg, run_len, n_runs, n_warm, cf, tb, (double*)(base + w.bins), g.stride, g.r, g.nbins);
  GateParams gp;
  for (int c = 0; c < 8; ++c) gp.G[c] = c < C ? chan_gain_h[c] : 0.0;
  gp.scale = (float)(1.0 / (block_s * rate));
  gp.C = C; gp.nblk = g.nblk; gp.nbins = g.nbins; gp.q = g.q;
  B2A_LAUNCH(lufs_gate_kernel, dim3((unsigned)B), dim3(GT), 0, stream, (const double*)(base + w.bins), gp,
             (float*)(base + w.zws), z_blocks, lufs_out, loud_out, target_db, n_target, gain_out);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

}  // namespace lufs
}  // namespace b2a

using namespace b2a::lufs;

extern "C" int64_t b2a_lufs_num_blocks(int64_t T_padded, double rate, double block_s) {
  Geometry g;
  if (T_padded < 1 || geometry(T_padded, rate, block_s, &g) != 0) return -1;
  return g.nblk;
}

extern "C" size_t b2a_lufs_workspace_bytes(int64_t B, int C, int64_t T_padded, double rate, double block_s) {
  Geometry g;
  if (B < 1 || C < 1 || T_padded < 1 || geometry(T_padded, rate, block_s, &g) != 0) return 0;
  return ws_layout(B * C, g.nbins, g.nblk).total;
}

extern "C" int b2a_lufs_f32(const float* x, int64_t B, int C, int64_t T, int64_t T_padded, double rate,
                            const double* sos_h, const double* stage_gain_h, int n_stage, double block_s,
                            const double* chan_gain_h, float* z_blocks, float* lufs_out, float* loud_out,
                            const float* target_db, int n_target, float* gain_out, void* ws, size_t ws_bytes,
                            void* stream) {
  B2A_REQUIRE(x && lufs_out && ws && sos_h && stage_gain_h && chan_gain_h, B2A_E_INVALID, "lufs: null pointer");
  B2A_REQUIRE(B >= 1 && C >= 1 && T >= 1, B2A_E_INVALID, "lufs: empty input (B=%lld C=%d T=%lld)", (long long)B, C,
              (long long)T);
  B2A_REQUIRE(C <= 5, B2A_E_INVALID, "lufs: at most 5 channels have BS.1770 gains (got %d)", C);
  B2A_REQUIRE(T_padded >= T, B2A_E_INVALID, "lufs: T_padded < T");
  B2A_REQUIRE(T_padded < (int64_t)2147483647 - 2 * TILE, B2A_E_UNSUPPORTED, "lufs: rows longer than 2^31 samples");
  B2A_REQUIRE(B * C * ((T_padded + TILE - 1) / TILE) < (int64_t)2147483647, B2A_E_UNSUPPORTED, "lufs: too many tiles");
  B2A_REQUIRE(n_stage >= 1 && n_stage <= MAX_STAGES, B2A_E_UNSUPPORTED,
              "lufs: %d biquad stages (1..%d supported: K-weighting has 2)", n_stage, MAX_STAGES);
  B2A_REQUIRE(!gain_out || (target_db && (n_target == 1 || n_target == B)), B2A_E_INVALID,
              "lufs: gain_out needs target_db with 1 or B entries");
  Geometry g;
  B2A_REQUIRE(geometry(T_padded, rate, block_s, &g) == 0, B2A_E_UNSUPPORTED,
              "lufs: gating stride int(block_s*rate/4) must be >= 64 samples (rate=%g block_s=%g)", rate, block_s);
  if (n_stage == 1)
    return run<1>(x, B, C, T, T_padded, g, sos_h, stage_gain_h, rate, block_s, chan_gain_h, z_blocks, lufs_out,
                  loud_out, target_db, n_target, gain_out, ws, ws_bytes, stream);
  return run<2>(x, B, C, T, T_padded, g, sos_h, stage_gain_h, rate, block_s, chan_gain_h, z_blocks, lufs_out,
                loud_out, target_db, n_target, gain_out, ws, ws_bytes, stream);
}

extern "C" int b2a_gain_f32(const float* x, float* out, int64_t B, int64_t per_item, const float* gain,
                            void* stream) {
  B2A_REQUIRE(x && out && gain, B2A_E_INVALID, "gain: null pointer");
  B2A_REQUIRE(B >= 1 && per_item >= 1 && B <= 65535, B2A_E_INVALID, "gain: bad shape");
  int vec_ok = (((uintptr_t)x | (uintptr_t)out) % 16 == 0) && (per_item % 4 == 0);
  int64_t work = vec_ok ? per_item / 4 : per_item;
  int64_t want = (work + 255) / 256;
  // ~8 resident CTAs per SM in total across the batch; grid-stride inside
  int64_t cap = (int64_t)B2A_NUM_SMS * 8 / B + 1;
  unsigned gx = (unsigned)(want < cap ? want : cap);
  B2A_LAUNCH(gain_kernel, dim3(gx, (unsigned)B), dim3(256), 0, stream, x, out, per_item, gain, vec_ok);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}
