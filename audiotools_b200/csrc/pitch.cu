// pitch.cu -- length-preserving pitch shift of [rows, T] waveforms on sm_90a.
//
// Replaces EffectMixin.pitch_shift (ref:audiotools/core/effects.py:247-277), which moves the batch to the
// CPU and runs libsox `pitch -q <cents>` + `rate` row by row.  SoX's pitch effect is WSOLA time-scale
// modification followed by a rate change; NO numeric output of it is pinned anywhere in the reference
// (its tests only check batch[0] == single, ref:tests/core/test_effects.py:156-181), so this file defines
// the same construction natively and parity is stated through properties (tests/test_gpu_parity.py):
// exact length, pitch ratio 2^(n/12), batch == per-item, determinism.
//
//   r = 2^(semitones/12).
//   1. WSOLA search   frames of W samples, synthesis hop Hs = W/2, nominal analysis hop Hs/r; frame j starts at
//                     p_j = a_j + d_j, d_j in [-D, D) maximising the correlation (every 2nd sample, W/4 terms)
//                     of x[a_j + d ...] with the natural continuation x[p_{j-1} + Hs ...] of the previous frame.
//   2. overlap-add    s[u] = hann(u - J Hs) x[p_J + u - J Hs] + (1 - hann(u - J Hs)) x[p_{J-1} + u - (J-1) Hs],
//                     J = floor(u / Hs)   (periodic Hann at 50 % overlap sums to one) -> x stretched by r.
//   3. rate change    y[n] = sum_k w_k s[floor(n r) + k - half + 1]: windowed sinc, cutoff c = 0.95 min(1, 1/r),
//                     8 zero crossings each side, Hann window, weights normalised to sum 1 -> length T again.
//
// Kernel 1  wsola_search_kernel  one CTA (512 threads) per row.  Frames are sequential (each depends on the
//           previous choice); inside a frame the 2D x (W/4) correlation table is a register-tiled FIR: the
//           candidate window is staged in shared memory split by sample parity (the stride-2 correlation
//           then reads unit-stride streams) and by (index mod 8), a thread owns 8 consecutive candidates x a
//           slice of the taps with a sliding 16-sample register window (8 conflict-free loads + 2 broadcast
//           float4 tap loads per 64 FMAs), slices are summed through shared memory and the arg-max is a
//           shuffle tree.  The NEXT frame's window only depends on the nominal positions, so it
//           streams in with cp.async underneath the current frame's arithmetic.
// Kernel 2  wsola_ola_kernel     one thread per stretched sample (coalesced reads of x, write s once).
// Kernel 3  rate_kernel          one thread per output; the 2*half weights are generated in registers with
//           two Chebyshev recurrences (sin(pi c t) and the window's cos) instead of a phase table: a table
//           indexed by each lane's own fractional phase costs ~32 cache lines per load.
#include "b2a_common.h"

namespace b2a {
namespace pitch {

constexpr int ST = 512;  // search threads per CTA

struct Geo {
  int W, Hs, D, Lc;  // frame, synthesis hop, search radius, correlation taps (every 2nd sample)
  int J;             // frames
  int half;          // interpolation taps each side
  int H;             // left halo of the stretched row (half rounded up to 4)
  int rcap;          // capacity (samples) of one staged search region
  int64_t SL;        // floats per stretched row (halo + samples, multiple of 4)
  double r;          // pitch ratio = stretch factor
  float c, pic;      // cutoff, pi*c
  float cb, sb;      // cos, sin of pi*c        (sinc numerator recurrence)
  float cw, sw;      // cos, sin of pi/half     (window recurrence)
  float inv_half;
  float inv_Hs;       // 1 / Hs (the Hann argument is 2 t / W = t / Hs)
  int log2Hs;
  int identity;       // semitones == 0: the row is copied
};

// One launch serves rows with different shifts: every row belongs to a group (<= MAXG distinct shifts) and reads
// its group's geometry; buffers are laid out with the largest group's strides.
constexpr int MAXG = 8;
struct GeoTable {
  Geo g[MAXG];
  int n;
  int Jmax;            // stride of the nominal / position tables
  long long SLmax;     // stride of the stretched rows
};
__device__ __forceinline__ int group_of(const int* __restrict__ row_group, int row) {
  return row_group ? __ldg(row_group + row) : 0;
}

__device__ __forceinline__ void cp_async4(float* smem_dst, const float* gmem_src) {
#ifdef B2A_SIM
  *smem_dst = *gmem_src;
#else
  unsigned sa = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(sa), "l"(gmem_src) : "memory");
#endif
}
__device__ __forceinline__ void cp_async_wait_all() {
#ifndef B2A_SIM
  asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
#endif
}

// nominal analysis position of frame j (double arithmetic, once per call; every row shares the table)
__global__ void nominal_kernel(int* __restrict__ nom, const B2A_GRID_CONSTANT GeoTable tab) {
  const Geo& g = tab.g[blockIdx.y];
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < g.J) nom[(size_t)blockIdx.y * tab.Jmax + j] = (int)floor((double)j * (double)g.Hs / g.r + 0.5);
}

__device__ __forceinline__ float fast_rcp(float v) {
#ifdef B2A_SIM
  return 1.0f / v;
#else
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v));
  return r;
#endif
}

__host__ __device__ inline int search_row_stride(int rcap) { return (((rcap >> 4) + 3 + 31) & ~31) + 2; }

// Arg-max key: high word = the correlation as an order-preserving unsigned, low word = the tie-break (ties go to
// the smaller |offset|, then the smaller offset), so the larger 64-bit key wins and the result is deterministic.
__device__ __forceinline__ unsigned long long corr_key(float v, int d) {
  const unsigned b = __float_as_uint(v);
  const unsigned ord = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
  const unsigned tie = 0xffffffffu - (unsigned)(2 * abs(d) + (d > 0 ? 1 : 0));
  return ((unsigned long long)ord << 32) | tie;
}
__device__ __forceinline__ int key_offset(unsigned long long k) {
  const unsigned c = 0xffffffffu - (unsigned)(k & 0xffffffffu);
  const int m = (int)(c >> 1);
  return (c & 1) ? m : -m;
}
__device__ __forceinline__ unsigned long long warp_max_key(unsigned long long k) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long other = __shfl_xor_sync(0xffffffffu, k, o);
    k = other > k ? other : k;
  }
  return k;
}

// Region of frame j: covers its candidate window [a_j - D, a_j + D + span) and every possible continuation
// of frame j-1, [a_{j-1} - D + Hs, a_{j-1} + D + Hs + span).  lo is chosen so that a_j - D - lo is a multiple
// of 16: each parity stream of the candidate window then starts on a multiple of 8.
__device__ __forceinline__ void region_of(int aj, int ap, const Geo& g, int& lo, int& rn) {
  const int span = 2 * g.Lc;
  const int mn = min(aj - g.D, ap - g.D + g.Hs);
  const int mx = max(aj + g.D + span, ap + g.D + g.Hs + span);
  lo = aj - g.D - 16 * ((aj - g.D - mn + 15) >> 4);
  rn = min((mx - lo + 15) & ~15, g.rcap);
}

// Shared-memory image of a region: sample x[lo + i] has parity p = i & 1 and index m = i >> 1 in its parity
// stream; it is stored in row p*8 + (m & 7), column m >> 3.  A thread that owns 8 consecutive candidates of
// one parity then reads every window element as a unit-stride (conflict-free) 32-bit load across the warp.
__device__ __forceinline__ void stage_region(const float* __restrict__ xr, int T, int lo, int rn, float* buf, int RS,
                                             int tid) {
  // ST is a multiple of 16: a thread always writes the same row, 32 columns further each time
  float* dst = buf + (((tid & 1) << 3) + ((tid >> 1) & 7)) * RS + (tid >> 4);
  const float* src = xr + lo + tid;
  int u = lo + tid;
  for (int i = tid; i < rn; i += ST, dst += ST / 16, src += ST, u += ST) {
    if ((unsigned)u < (unsigned)T) cp_async4(dst, src); else *dst = 0.f;
  }
}

__global__ void __launch_bounds__(ST)
wsola_search_kernel(const float* __restrict__ x, int T, const B2A_GRID_CONSTANT GeoTable tab,
                    const int* __restrict__ row_group, const int* __restrict__ nom_all /*[n, Jmax]*/,
                    int* __restrict__ pos /*[rows, Jmax]*/) {
  B2A_DYN_SMEM(smem);
  const int grp = group_of(row_group, blockIdx.x);
  const Geo g = tab.g[grp];
  if (g.identity) return;
  const int* nom = nom_all + (size_t)grp * tab.Jmax;
  // layout (floats): [2 buffers][16 rows][RS] | part[8*ST] | tfb[Lc];  RS = 2 mod 32 (staging stores of 32
  // consecutive samples touch 16 rows x 2 columns: distinct banks)
  const int RS = search_row_stride(g.rcap);
  float* reg = reinterpret_cast<float*>(smem);
  float* part = reg + 32 * RS;
  float* tfb = part + 8 * ST;
  __shared__ unsigned long long wk[ST / 32];
  __shared__ int s_prev[2];
  const float* xr = x + (size_t)blockIdx.x * (size_t)T;
  int* pr = pos + (size_t)blockIdx.x * tab.Jmax;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int span = 2 * g.Lc;
  const int ne = g.D;       // candidates per parity
  const int G = ne >> 3;    // groups of 8 consecutive candidates per parity
  const int og = tid % (2 * G), kq = tid / (2 * G);
  const int parity = og / G, gi = og - parity * G;
  const int KS = min(ST / (2 * G), g.Lc >> 3);  // tap slices
  const int TS = g.Lc / KS;                     // taps per slice (multiple of 8)
  const bool active = kq < KS;
  if (tid == 0) { pr[0] = 0; s_prev[0] = 0; }
  if (g.J > 1) {
    int lo, rn;
    region_of(__ldg(nom + 1), __ldg(nom), g, lo, rn);
    stage_region(xr, T, lo, rn, reg + 16 * RS, RS, tid);  // buffer 1
  }
  for (int j = 1; j < g.J; ++j) {
    cp_async_wait_all();
    __syncthreads();  // region j landed; s_prev[(j-1)&1] visible; buffer (j+1)&1, part[] and tfb[] are free again
    const int prev = s_prev[(j - 1) & 1];
    const int a = __ldg(nom + j);
    const int cont = prev + g.Hs;  // natural continuation of frame j-1
    int lo, rn;
    region_of(a, __ldg(nom + j - 1), g, lo, rn);
    const float* buf = reg + (j & 1) * 16 * RS;
    int best = min(max(a, 0), max(T - g.W, 0));
    const bool search = cont + span <= T && a - g.D >= 0 && a + g.D + span <= T;  // uniform over the CTA
    if (search) {  // the template: tfb[i] = x[cont + 2 i]
      const int c = cont - lo;
      if (c >= 0 && c + span <= rn) {
        for (int i = tid; i < g.Lc; i += ST) {
          const int m = (c >> 1) + i;
          tfb[i] = buf[(((c & 1) << 3) + (m & 7)) * RS + (m >> 3)];
        }
      } else {  // continuation outside the staged region (only after a clamped frame)
        for (int i = tid; i < g.Lc; i += ST) tfb[i] = __ldg(xr + cont + 2 * i);
      }
    }
    if (j + 1 < g.J) {  // stream the next region in underneath this frame's correlations
      int lo2, rn2;
      region_of(__ldg(nom + j + 1), a, g, lo2, rn2);
      stage_region(xr, T, lo2, rn2, reg + ((j + 1) & 1) * 16 * RS, RS, tid);
    }
    if (search) {
      __syncthreads();  // tfb complete
      if (active) {
        const int s8 = (a - g.D - lo) >> 4;  // window start in units of 8 stream samples
        const float* rowp = buf + (parity << 3) * RS + s8 + gi + ((TS * kq) >> 3);
        const float4* tq = reinterpret_cast<const float4*>(tfb + TS * kq);
        const float* r0 = rowp, *r1 = r0 + RS, *r2 = r1 + RS, *r3 = r2 + RS;
        const float* r4 = r3 + RS, *r5 = r4 + RS, *r6 = r5 + RS, *r7 = r6 + RS;
        float w[8], v[8], acc[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = 0.f;
        w[0] = r0[0]; w[1] = r1[0]; w[2] = r2[0]; w[3] = r3[0]; w[4] = r4[0]; w[5] = r5[0]; w[6] = r6[0]; w[7] = r7[0];
#define B2A_CORR_STEP(WIN, NXT, I8)                                                                          \
  {                                                                                                          \
    NXT[0] = r0[(I8) + 1]; NXT[1] = r1[(I8) + 1]; NXT[2] = r2[(I8) + 1]; NXT[3] = r3[(I8) + 1];              \
    NXT[4] = r4[(I8) + 1]; NXT[5] = r5[(I8) + 1]; NXT[6] = r6[(I8) + 1]; NXT[7] = r7[(I8) + 1];              \
    const float4 ta = tq[2 * (I8)], tb = tq[2 * (I8) + 1];                                                   \
    const float t[8] = {ta.x, ta.y, ta.z, ta.w, tb.x, tb.y, tb.z, tb.w};                                     \
    _Pragma("unroll") for (int r = 0; r < 8; ++r) {                                                          \
      _Pragma("unroll") for (int u = 0; u < 8; ++u)                                                          \
          acc[r] = fmaf(t[u], (r + u < 8) ? WIN[r + u] : NXT[r + u - 8], acc[r]);                            \
    }                                                                                                        \
  }
        const int steps = TS >> 3;
        int i8 = 0;
#pragma unroll 1
        for (; i8 + 2 <= steps; i8 += 2) {  // ping-pong the two window halves: no register moves
          B2A_CORR_STEP(w, v, i8);
          B2A_CORR_STEP(v, w, i8 + 1);
        }
        if (i8 < steps) B2A_CORR_STEP(w, v, i8);
#undef B2A_CORR_STEP
        float* pq = part + kq * (2 * ne) + parity * ne + 8 * gi;
        *reinterpret_cast<float4*>(pq) = make_float4(acc[0], acc[1], acc[2], acc[3]);
        *reinterpret_cast<float4*>(pq + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
      }
      __syncthreads();
      unsigned long long key = 0ull;  // below every real key (NaN correlations never win: offset 0)
      if (tid < 2 * ne) {
        float v = 0.f;
        for (int q = 0; q < KS; ++q) v += part[q * (2 * ne) + tid];
        const int par = tid >= ne, e = tid - par * ne;
        if (v == v) key = corr_key(v, 2 * e + par - g.D);
      }
      key = warp_max_key(key);
      if (lane == 0) wk[warp] = key;
      __syncthreads();
      if (warp == 0) {
        key = warp_max_key(lane < ST / 32 ? wk[lane] : 0ull);
        best = a + (key ? key_offset(key) : 0);
      }
    }
    if (tid == 0) { pr[j] = best; s_prev[j & 1] = best; }
  }
}

// stretched row: sbuf[row][H + u] = s[u]; the H-sample halo in front is zero.  4 samples per thread (H, Hs and SL
// are multiples of 4, so the 4 samples share their two frames and the store is one aligned float4).
__global__ void __launch_bounds__(256)
wsola_ola_kernel(const float* __restrict__ x, const int* __restrict__ pos, float* __restrict__ sbuf, int T,
                 const B2A_GRID_CONSTANT GeoTable tab, const int* __restrict__ row_group) {
  const int row = blockIdx.y;
  const Geo g = tab.g[group_of(row_group, row)];
  const int i = 4 * (blockIdx.x * blockDim.x + threadIdx.x);
  if (g.identity || i >= g.SL) return;
  const int u = i - g.H;
  float v[4] = {0.f, 0.f, 0.f, 0.f};
  if (u >= 0) {
    const float* xr = x + (size_t)row * (size_t)T;
    const int* pr = pos + (size_t)row * tab.Jmax;
    const int J0 = u >> g.log2Hs, t0 = u - (J0 << g.log2Hs);
    const int i0 = J0 < g.J ? __ldg(pr + J0) + t0 : -8;                 // frame J0 reads x[i0 + q]
    const int i1 = J0 >= 1 ? __ldg(pr + J0 - 1) + t0 + g.Hs : -8;      // frame J0-1
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float h0 = 0.5f - 0.5f * cospif((float)(t0 + q) * g.inv_Hs);
      const float a = (J0 < g.J && i0 + q >= 0 && i0 + q < T) ? __ldg(xr + i0 + q) : 0.f;
      const float b = (J0 >= 1 && i1 + q >= 0 && i1 + q < T) ? __ldg(xr + i1 + q) : 0.f;
      v[q] = fmaf(1.0f - h0, b, h0 * a);
    }
  }
  *reinterpret_cast<float4*>(sbuf + (size_t)row * (size_t)tab.SLmax + i) = make_float4(v[0], v[1], v[2], v[3]);
}

__global__ void __launch_bounds__(256)
rate_kernel(const float* __restrict__ sbuf, const float* __restrict__ x, float* __restrict__ y, int T,
            const B2A_GRID_CONSTANT GeoTable tab, const int* __restrict__ row_group) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= T) return;
  const int row = blockIdx.y;
  const Geo g = tab.g[group_of(row_group, row)];
  if (g.identity) {
    y[(size_t)row * (size_t)T + n] = __ldg(x + (size_t)row * (size_t)T + n);
    return;
  }
  const double P = (double)n * g.r;  // read position in the stretched signal
  const int ip = (int)P;
  const float f = (float)(P - (double)ip);
  // tap k reads s[ip + k - half + 1] = sbuf[H + ip + k - half + 1]; its distance to P is t_k = t0 + k
  const float* sp = sbuf + (size_t)row * (size_t)tab.SLmax + ip + 1 + (g.H - g.half);
  const float t0 = (float)(1 - g.half) - f;
  float s0, c0, ws0, wc0;
  sincospif(g.c * t0, &s0, &c0);            // sin, cos(pi c t0)
  sincospif(t0 * g.inv_half, &ws0, &wc0);   // sin, cos(pi t0 / half)
  float sm = s0 * g.cb - c0 * g.sb;         // sin(pi c (t0 - 1))
  float cm = wc0 * g.cw + ws0 * g.sw;       // cos(pi (t0 - 1) / half)
  float sk = s0, ck = wc0;
  const float two_cb = 2.0f * g.cb, two_cw = 2.0f * g.cw;
  float acc = 0.f, wsum = 0.f;
  const int half = g.half;
  // taps 0 .. half-2 and half+1 .. 2 half-1 have |t| >= 1: sin(pi c t)/t straight from the recurrence
#define B2A_RATE_STEP()                                          \
  {                                                              \
    const float sn = fmaf(two_cb, sk, -sm), cn = fmaf(two_cw, ck, -cm); \
    sm = sk; sk = sn; cm = ck; ck = cn;                          \
  }
  float t = t0;
#pragma unroll 4
  for (int k = 0; k < half - 1; ++k) {
    const float w = fmaf(0.5f, ck, 0.5f) * (sk * fast_rcp(t));
    wsum += w;
    acc = fmaf(w, __ldg(sp + k), acc);
    t += 1.0f;
    B2A_RATE_STEP();
  }
  // the two taps around the read position (t = -f and 1 - f): where |t| is small the recurrence's absolute
  // error would be amplified by 1/t, so use the series of sin(z)/z there
#pragma unroll
  for (int k2 = 0; k2 < 2; ++k2) {
    const float tc = (float)k2 - f;
    const float z2 = (g.pic * tc) * (g.pic * tc);
    const float sinc = fabsf(tc) < 0.1f ? g.pic * fmaf(z2, fmaf(z2, 1.0f / 120.0f, -1.0f / 6.0f), 1.0f) : sk * fast_rcp(tc);
    const float w = fmaf(0.5f, ck, 0.5f) * sinc;
    wsum += w;
    acc = fmaf(w, __ldg(sp + half - 1 + k2), acc);
    B2A_RATE_STEP();
  }
  t = 2.0f - f;
#pragma unroll 4
  for (int k = half + 1; k < 2 * half; ++k) {
    const float w = fmaf(0.5f, ck, 0.5f) * (sk * fast_rcp(t));
    wsum += w;
    acc = fmaf(w, __ldg(sp + k), acc);
    t += 1.0f;
    B2A_RATE_STEP();
  }
#undef B2A_RATE_STEP
  y[(size_t)row * (size_t)T + n] = acc * fast_rcp(wsum);
}

// time stretch = the first two stages only: out[row][i] = s[i] (the stretched row without its halo)
__global__ void __launch_bounds__(256)
stretch_copy_kernel(const float* __restrict__ sbuf, const float* __restrict__ x, float* __restrict__ out, int T,
                    long long out_len, const B2A_GRID_CONSTANT GeoTable tab) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= out_len) return;
  const int row = blockIdx.y;
  const Geo& g = tab.g[0];
  float v;
  if (g.identity) v = i < T ? __ldg(x + (size_t)row * (size_t)T + i) : 0.f;
  else v = __ldg(sbuf + (size_t)row * (size_t)tab.SLmax + g.H + i);
  out[(size_t)row * (size_t)out_len + i] = v;
}

// min_len: the least number of stretched samples s[0 .. Ls) to produce (time_stretch's output length; 0 otherwise)
static int geometry(int64_t rows, int64_t T, int sr, float semitones, int64_t min_len, Geo* g) {
  (void)rows;
  const double r = pow(2.0, (double)semitones / 12.0);
  int W = 1;
  const double target = 0.046 * sr;
  while (W * 2 <= target * 1.4142135623730951) W *= 2;  // nearest power of two (in log scale)
  if (W < 64) W = 64;
  if (W > 2048) W = 2048;
  memset(g, 0, sizeof(*g));
  g->W = W; g->Hs = W / 2; g->D = W / 8; g->Lc = W / 4; g->r = r;
  g->J = (int)((double)T * r / g->Hs) + 2;
  const double c = 0.95 * (r > 1.0 ? 1.0 / r : 1.0);
  g->half = (int)ceil(8.0 / c);
  g->H = (g->half + 3) & ~3;
  int64_t Ls = (int64_t)ceil((double)T * r) + g->half + 2;  // samples s[0 .. Ls): what the rate change reads
  if (Ls < min_len) Ls = min_len;
  g->SL = (g->H + Ls + 3) / 4 * 4;
  const int drift = (int)ceil(fabs((double)g->Hs / r - (double)g->Hs)) + 1;
  g->rcap = (2 * g->D + 2 * g->Lc + drift + 48 + 63) / 64 * 64;
  const double PI = 3.14159265358979323846;
  g->c = (float)c; g->pic = (float)(PI * c);
  g->cb = (float)cos(PI * c); g->sb = (float)sin(PI * c);
  g->cw = (float)cos(PI / g->half); g->sw = (float)sin(PI / g->half);
  g->inv_half = (float)(1.0 / g->half);
  g->inv_Hs = 1.0f / (float)g->Hs;
  g->log2Hs = 0;
  while ((1 << g->log2Hs) < g->Hs) ++g->log2Hs;
  g->identity = (semitones == 0.0f);
  return 0;
}

static int build_table(int64_t rows, int64_t T, int sr, const float* semitones_h, int n_groups, GeoTable* tab,
                       int64_t min_len = 0) {
  memset(tab, 0, sizeof(*tab));
  tab->n = n_groups;
  for (int i = 0; i < n_groups; ++i) {
    geometry(rows, T, sr, semitones_h[i], min_len, &tab->g[i]);
    if (tab->g[i].J > tab->Jmax) tab->Jmax = tab->g[i].J;
    if (tab->g[i].SL > tab->SLmax) tab->SLmax = tab->g[i].SL;
  }
  return 0;
}
// workspace: positions [rows, Jmax] | nominal [n, Jmax] | (256 B aligned) stretched rows [rows, SLmax]
static size_t pos_bytes(int64_t rows, const GeoTable& t) {
  return ((size_t)(rows + t.n) * t.Jmax * 4 + 255) / 256 * 256;
}
static bool groups_ok(const float* semitones_h, int n_groups) {
  if (!semitones_h || n_groups < 1 || n_groups > MAXG) return false;
  for (int i = 0; i < n_groups; ++i)
    if (!(fabsf(semitones_h[i]) <= 24.f)) return false;
  return true;
}

}  // namespace pitch
}  // namespace b2a

using namespace b2a::pitch;

extern "C" size_t b2a_pitch_shift_multi_workspace_bytes(int64_t rows, int64_t T, int sr, const float* semitones_h,
                                                        int n_groups) {
  if (rows < 1 || T < 1 || sr < 1 || !groups_ok(semitones_h, n_groups)) return 0;
  GeoTable tab;
  build_table(rows, T, sr, semitones_h, n_groups, &tab);
  return pos_bytes(rows, tab) + (size_t)rows * (size_t)tab.SLmax * 4;
}

extern "C" int b2a_pitch_shift_multi_f32(const float* x, int64_t rows, int64_t T, int sr, const float* semitones_h,
                                         int n_groups, const int32_t* row_group, float* out, void* ws, size_t ws_bytes,
                                         void* stream) {
  B2A_REQUIRE(x && out && ws && semitones_h, B2A_E_INVALID, "pitch_shift: null pointer");
  B2A_REQUIRE(rows >= 1 && T >= 1 && sr >= 1, B2A_E_INVALID, "pitch_shift: bad argument");
  B2A_REQUIRE(n_groups >= 1 && n_groups <= MAXG, B2A_E_UNSUPPORTED, "pitch_shift: %d distinct shifts (max %d per call)",
              n_groups, MAXG);
  B2A_REQUIRE(groups_ok(semitones_h, n_groups), B2A_E_UNSUPPORTED, "pitch_shift: |semitones| > 24");
  B2A_REQUIRE(row_group || n_groups == 1, B2A_E_INVALID, "pitch_shift: row_group is required with several shifts");
  B2A_REQUIRE(rows * T < ((int64_t)1 << 40) && T < ((int64_t)1 << 28) && rows <= 65535, B2A_E_UNSUPPORTED,
              "pitch_shift: too large");
  B2A_REQUIRE(((uintptr_t)ws & 15) == 0, B2A_E_INVALID, "pitch_shift: workspace must be 16-byte aligned");
  B2A_REQUIRE(out != x, B2A_E_INVALID, "pitch_shift: in-place is not supported");
  GeoTable tab;
  build_table(rows, T, sr, semitones_h, n_groups, &tab);
  const size_t pb = pos_bytes(rows, tab);
  B2A_REQUIRE(ws_bytes >= pb + (size_t)rows * (size_t)tab.SLmax * 4, B2A_E_INVALID, "pitch_shift: workspace too small");
  int* pos = (int*)ws;
  int* nom = pos + (size_t)rows * tab.Jmax;
  float* sbuf = (float*)((char*)ws + pb);
  size_t smem = 0;
  for (int i = 0; i < n_groups; ++i) {
    const Geo& g = tab.g[i];
    const size_t b = (size_t)(32 * search_row_stride(g.rcap) + 8 * ST + g.Lc) * 4;
    if (b > smem) smem = b;
  }
  B2A_CUDA_OK(cudaFuncSetAttribute(wsola_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  B2A_LAUNCH(nominal_kernel, dim3((unsigned)((tab.Jmax + 255) / 256), (unsigned)n_groups), dim3(256), 0, stream, nom, tab);
  B2A_LAUNCH(wsola_search_kernel, dim3((unsigned)rows), dim3(ST), smem, stream, x, (int)T, tab, row_group,
             (const int*)nom, pos);
  B2A_LAUNCH(wsola_ola_kernel, dim3((unsigned)((tab.SLmax / 4 + 255) / 256), (unsigned)rows), dim3(256), 0, stream, x,
             (const int*)pos, sbuf, (int)T, tab, row_group);
  B2A_LAUNCH(rate_kernel, dim3((unsigned)((T + 255) / 256), (unsigned)rows), dim3(256), 0, stream, (const float*)sbuf, x,
             out, (int)T, tab, row_group);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" int b2a_pitch_shift_num_frames(int64_t T, int sr, float semitones) {
  if (T < 1 || sr < 1 || !(fabsf(semitones) <= 24.f)) return -1;
  Geo g;
  geometry(1, T, sr, semitones, 0, &g);
  return g.J;
}

/* EffectMixin.time_stretch (ref:audiotools/core/effects.py:279-309; SoX `tempo factor` there): the WSOLA stages of the
 * pitch shifter on their own -- speed the signal up by `factor` (duration / factor), pitch unchanged. */
static float stretch_semitones(double factor) { return (float)(12.0 * log2(1.0 / factor)); }

extern "C" int64_t b2a_time_stretch_out_len(int64_t T, double factor) {
  if (T < 1 || !(factor >= 0.25 && factor <= 4.0)) return -1;
  return (int64_t)floor((double)T / factor + 0.5);
}

// The stretched rows cover the whole output, round(T / factor) samples: r is 2^(semitones / 12) with the semitones
// rounded to float32, so T r alone can fall short of T / factor by more than the rate change's half + 2 samples of
// slack (by 20 samples at T = 2^28 - 1, factor 0.26875).  Frames past the last one read as 0 there.
static void stretch_table(int64_t rows, int64_t T, int sr, double factor, GeoTable* tab) {
  const float st = (factor == 1.0) ? 0.0f : stretch_semitones(factor);
  build_table(rows, T, sr, &st, 1, tab, b2a_time_stretch_out_len(T, factor));
}

extern "C" size_t b2a_time_stretch_workspace_bytes(int64_t rows, int64_t T, int sr, double factor) {
  if (rows < 1 || T < 1 || sr < 1 || !(factor >= 0.25 && factor <= 4.0)) return 0;
  GeoTable tab;
  stretch_table(rows, T, sr, factor, &tab);
  return pos_bytes(rows, tab) + (size_t)rows * (size_t)tab.SLmax * 4;
}

extern "C" int b2a_time_stretch_f32(const float* x, int64_t rows, int64_t T, int sr, double factor, float* out,
                                    void* ws, size_t ws_bytes, void* stream) {
  B2A_REQUIRE(x && out && ws, B2A_E_INVALID, "time_stretch: null pointer");
  B2A_REQUIRE(rows >= 1 && T >= 1 && sr >= 1, B2A_E_INVALID, "time_stretch: bad argument");
  B2A_REQUIRE(factor >= 0.25 && factor <= 4.0, B2A_E_UNSUPPORTED, "time_stretch: factor %g outside [0.25, 4]", factor);
  B2A_REQUIRE(rows * T < ((int64_t)1 << 40) && T < ((int64_t)1 << 28) && rows <= 65535, B2A_E_UNSUPPORTED,
              "time_stretch: too large");
  B2A_REQUIRE(((uintptr_t)ws & 15) == 0, B2A_E_INVALID, "time_stretch: workspace must be 16-byte aligned");
  const int64_t out_len = b2a_time_stretch_out_len(T, factor);
  GeoTable tab;
  stretch_table(rows, T, sr, factor, &tab);
  const size_t pb = pos_bytes(rows, tab);
  B2A_REQUIRE(ws_bytes >= pb + (size_t)rows * (size_t)tab.SLmax * 4, B2A_E_INVALID, "time_stretch: workspace too small");
  int* pos = (int*)ws;
  int* nom = pos + (size_t)rows * tab.Jmax;
  float* sbuf = (float*)((char*)ws + pb);
  const Geo& g = tab.g[0];
  B2A_REQUIRE(g.identity || g.H + out_len <= g.SL, B2A_E_INVALID, "time_stretch: internal length mismatch");
  if (!g.identity) {
    const size_t smem = (size_t)(32 * search_row_stride(g.rcap) + 8 * ST + g.Lc) * 4;
    B2A_CUDA_OK(cudaFuncSetAttribute(wsola_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    B2A_LAUNCH(nominal_kernel, dim3((unsigned)((tab.Jmax + 255) / 256), 1u), dim3(256), 0, stream, nom, tab);
    B2A_LAUNCH(wsola_search_kernel, dim3((unsigned)rows), dim3(ST), smem, stream, x, (int)T, tab, (const int*)nullptr,
               (const int*)nom, pos);
    B2A_LAUNCH(wsola_ola_kernel, dim3((unsigned)((tab.SLmax / 4 + 255) / 256), (unsigned)rows), dim3(256), 0, stream, x,
               (const int*)pos, sbuf, (int)T, tab, (const int*)nullptr);
  }
  B2A_LAUNCH(stretch_copy_kernel, dim3((unsigned)((out_len + 255) / 256), (unsigned)rows), dim3(256), 0, stream,
             (const float*)sbuf, x, out, (int)T, (long long)out_len, tab);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}
