// iir.cu -- per-item IIR biquad cascades of a batch (K19 in DESIGN.md): scipy.signal.sosfilt with zero initial state.
//
//   sos [sos_items, S, 6] float32, rows b0 b1 b2 a0 a1 a2; the kernels use b / a0 and a / a0 in float32 (exact when
//   a0 = 1, which is what Engine.sos_filter passes).  Item b uses set b when sos_items = B, else set 0, for all its
//   channels.  Each section is the transposed direct form II of sosfilt, sections in order:
//     y = b0 u + z1;  z1 = b1 u - a1 y + z2;  z2 = b2 u - a2 y      (u: the section's input, y: its output)
//   run in double on the float32 samples and coefficients; y is rounded to float32 once.  A float32 recursion loses up
//   to ~1e5 u near z = 1 (low frequencies, high Q), and splitting it into chunks changes that error unpredictably (a
//   chunk's zero-state response and its carried start state nearly cancel wherever a resonance is excited at the
//   chunk's start), so every stage that carries state does it in double.
//   x is float(gain[b] x) when a gain is given; reverse reads and writes every row back to front.
//   A section that fails the triangle test |a2| < 1 and |a1| < 1 + a2 (a pole on or outside the unit circle) makes its
//   item's output all NaN.  A NaN or inf sample makes its row non-finite from that sample on.
//
// The cascade's state s = (z1, z2) of every section is 2S numbers.  With the input set to 0 one sample maps s to A s,
// and a chunk of CHUNK samples maps it to M = A^CHUNK.  Three launches, no host sync, exact carries (no warm-up):
//   chunk_state_kernel   a warp per (row, 32 consecutive chunks), a lane per chunk: the recursion over the chunk
//                        from zero state gives the chunk's end state e_k.  Samples travel through a 32 x 32
//                        shared tile per warp, so every global access is a coalesced row of 32 floats.
//   carry_kernel         a warp per row: A from the item's coefficients in double, M and M^2, M^4, M^8, M^16 by
//                        squaring, then the affine scan s_{k+1} = M s_k + e_k, s_0 = 0, 32 chunks at a time as a
//                        warp scan in double; writes every chunk's start state s_k.
//   filter_kernel        the layout of the first kernel: the recursion over the chunk from s_k writes y.
// Nothing depends on the launch geometry or on other items: reruns and batch-versus-single calls are bit-identical.
#include "b2a_common.h"

namespace b2a {
namespace iir {

constexpr int CHUNK = 1024;   // samples of a row per chunk (one lane's sequential run); tests cover T = CHUNK +- 1
constexpr int TILE = 32;      // samples per lane per shared-memory tile
constexpr int WARPS = 8;      // warps per CTA of the chunk kernels
constexpr int SMAX = 8;       // largest number of sections

template <int S>
struct Coef {
  double b0[S], b1[S], b2[S], a1[S], a2[S];  // the float32 coefficients, exactly
  bool stable;
};

template <int S>
__device__ __forceinline__ Coef<S> load_coef(const float* __restrict__ sos) {
  Coef<S> c;
  c.stable = true;
#pragma unroll
  for (int s = 0; s < S; ++s) {
    const float* r = sos + 6 * s;
    const float a0 = __ldg(r + 3), a1 = __ldg(r + 4) / a0, a2 = __ldg(r + 5) / a0;
    c.b0[s] = __ldg(r) / a0, c.b1[s] = __ldg(r + 1) / a0, c.b2[s] = __ldg(r + 2) / a0;
    c.a1[s] = a1, c.a2[s] = a2;
    // written so that a NaN coefficient fails it
    c.stable = c.stable && fabsf(a2) < 1.f && fabsf(a1) < 1.f + a2;
  }
  return c;
}

// One sample through the cascade in double; z holds (z1, z2) of every section
template <int S>
__device__ __forceinline__ double step(const Coef<S>& c, double (&z)[2 * S], double u) {
#pragma unroll
  for (int s = 0; s < S; ++s) {
    const double y = fma(c.b0[s], u, z[2 * s]);
    z[2 * s] = fma(-c.a1[s], y, fma(c.b1[s], u, z[2 * s + 1]));
    z[2 * s + 1] = fma(-c.a2[s], y, c.b2[s] * u);
    u = y;
  }
  return u;
}

// Walk the warp's chunks tile by tile: lane l runs chunk g * 32 + l of row `row` from state z.  WRITE: y replaces the
// tile and goes to out.  Flat indices are 64-bit.
template <int S, bool WRITE>
__device__ __forceinline__ void run_chunks(const float* x, float* out, int64_t row_off, int64_t T, int64_t first,
                                           float g0, bool reverse, const Coef<S>& c, double (&z)[2 * S], float* tile) {
  const int lane = threadIdx.x & 31;
  const int64_t len = T < CHUNK ? T : CHUNK;
  const int n_tiles = (int)((len + TILE - 1) / TILE);
  for (int t = 0; t < n_tiles; ++t) {
    for (int r = 0; r < 32; ++r) {
      const int64_t n = first + (int64_t)r * CHUNK + t * TILE + lane;
      tile[r * (TILE + 1) + lane] = n < T ? x[row_off + (reverse ? T - 1 - n : n)] * g0 : 0.f;
    }
    __syncwarp();
    float* mine = tile + lane * (TILE + 1);
#pragma unroll 4
    for (int k = 0; k < TILE; ++k) {
      const double y = step<S>(c, z, (double)mine[k]);
      if (WRITE) mine[k] = (float)y;
    }
    __syncwarp();
    if (WRITE) {
      for (int r = 0; r < 32; ++r) {
        const int64_t n = first + (int64_t)r * CHUNK + t * TILE + lane;
        if (n < T) out[row_off + (reverse ? T - 1 - n : n)] = tile[r * (TILE + 1) + lane];
      }
      __syncwarp();
    }
  }
}

// ws_e [rows, n_chunks, 2S]: end state of every chunk from zero state.
template <int S>
__global__ void __launch_bounds__(WARPS * 32) chunk_state_kernel(const float* __restrict__ x,
                                                                 const float* __restrict__ gain, int C, int64_t T,
                                                                 const float* __restrict__ sos, int64_t sos_items,
                                                                 int64_t n_chunks, int64_t work, int reverse,
                                                                 double* __restrict__ ws_e) {
  __shared__ float s_tile[WARPS][32 * (TILE + 1)];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t n_groups = (n_chunks + 31) / 32;
  for (int64_t w = (int64_t)blockIdx.x * WARPS + wid; w < work; w += (int64_t)gridDim.x * WARPS) {
    const int64_t row = w / n_groups, g = w - row * n_groups, b = row / C;
    const Coef<S> c = load_coef<S>(sos + (sos_items > 1 ? b : 0) * 6 * S);
    const float g0 = gain ? __ldg(gain + b) : 1.f;
    double z[2 * S];
#pragma unroll
    for (int i = 0; i < 2 * S; ++i) z[i] = 0.0;
    run_chunks<S, false>(x, nullptr, row * T, T, g * 32 * CHUNK, g0, reverse, c, z, s_tile[wid]);
    const int64_t k = g * 32 + lane;
    if (k < n_chunks) {
#pragma unroll
      for (int i = 0; i < 2 * S; ++i) ws_e[(row * n_chunks + k) * 2 * S + i] = z[i];
    }
  }
}

// v += P w for an N x N row-major matrix in shared memory (every lane reads the same word: a broadcast)
template <int N>
__device__ __forceinline__ void matvec_add(const double* P, const double (&w)[N], double (&v)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) {
    double a = 0.0;
#pragma unroll
    for (int j = 0; j < N; ++j) a = fma(P[i * N + j], w[j], a);
    v[i] += a;
  }
}

// dst = src * src for N x N matrices in shared memory, by the 32 lanes of the warp
template <int N>
__device__ __forceinline__ void square(const double* src, double* dst) {
  const int lane = threadIdx.x & 31;
  for (int o = lane; o < N * N; o += 32) {
    const int i = o / N, j = o - i * N;
    double a = 0.0;
#pragma unroll
    for (int k = 0; k < N; ++k) a = fma(src[i * N + k], src[k * N + j], a);
    dst[o] = a;
  }
  __syncwarp();
}

// One warp (one CTA) per row.  ws_s [rows, n_chunks, 2S]: the start state of every chunk.
template <int S>
__global__ void __launch_bounds__(32) carry_kernel(const float* __restrict__ sos, int64_t sos_items, int C,
                                                   int64_t rows, int64_t n_chunks, const double* __restrict__ ws_e,
                                                   double* __restrict__ ws_s) {
  constexpr int N = 2 * S;
  __shared__ double s_pow[6][N * N];  // M, M^2, M^4, M^8, M^16; [5] scratch
  const int lane = threadIdx.x;
  for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
    const int64_t b = row / C;
    const float* so = sos + (sos_items > 1 ? b : 0) * 6 * S;
    if (n_chunks > 1) {
      // A, row by row: Y is the previous section's output as a linear form of the state (0 before section 0)
      if (lane == 0) {
        double Y[N], Ys[N];
        for (int j = 0; j < N; ++j) Y[j] = 0.0;
        for (int s = 0; s < S; ++s) {
          const float a0 = so[6 * s + 3];
          const double b0 = (double)(so[6 * s] / a0), b1 = (double)(so[6 * s + 1] / a0),
                       b2 = (double)(so[6 * s + 2] / a0), a1 = (double)(so[6 * s + 4] / a0),
                       a2 = (double)(so[6 * s + 5] / a0);
          for (int j = 0; j < N; ++j) Ys[j] = b0 * Y[j] + (j == 2 * s ? 1.0 : 0.0);
          for (int j = 0; j < N; ++j) {
            s_pow[0][(2 * s) * N + j] = b1 * Y[j] - a1 * Ys[j] + (j == 2 * s + 1 ? 1.0 : 0.0);
            s_pow[0][(2 * s + 1) * N + j] = b2 * Y[j] - a2 * Ys[j];
          }
          for (int j = 0; j < N; ++j) Y[j] = Ys[j];
        }
      }
      __syncwarp();
      // A^CHUNK: log2(CHUNK) squarings, alternating between slots 0 and 5
      int cur = 0;
      for (int p = 1; p < CHUNK; p *= 2) {
        square<N>(s_pow[cur], s_pow[5 - cur]);
        cur = 5 - cur;
      }
      if (cur != 0) {
        for (int o = lane; o < N * N; o += 32) s_pow[0][o] = s_pow[cur][o];
        __syncwarp();
      }
      for (int p = 1; p < 5; ++p) square<N>(s_pow[p - 1], s_pow[p]);
    }
    if (lane == 0) {
#pragma unroll
      for (int i = 0; i < N; ++i) ws_s[row * n_chunks * N + i] = 0.0;  // s_0
    }
    double carry[N];  // start state of the batch's first chunk
#pragma unroll
    for (int i = 0; i < N; ++i) carry[i] = 0.0;
    for (int64_t base = 0; base + 1 < n_chunks; base += 32) {  // the last chunk's end state is not needed
      const int64_t k = base + lane;
      double v[N], w[N];
#pragma unroll
      for (int i = 0; i < N; ++i) v[i] = k < n_chunks ? ws_e[(row * n_chunks + k) * N + i] : 0.0;
      if (lane == 0 && base > 0) matvec_add<N>(s_pow[0], carry, v);
      // inclusive scan: lane l ends with the end state of chunk base + l, i.e. the start state of chunk base + l + 1
#pragma unroll
      for (int p = 0; p < 5; ++p) {
        const int o = 1 << p;
#pragma unroll
        for (int i = 0; i < N; ++i) w[i] = __shfl_up_sync(0xffffffffu, v[i], o);
        if (lane >= o) matvec_add<N>(s_pow[p], w, v);
      }
      if (k + 1 < n_chunks) {
#pragma unroll
        for (int i = 0; i < N; ++i) ws_s[(row * n_chunks + k + 1) * N + i] = v[i];
      }
#pragma unroll
      for (int i = 0; i < N; ++i) carry[i] = __shfl_sync(0xffffffffu, v[i], 31);
    }
    __syncwarp();  // the next row overwrites s_pow
  }
}

template <int S>
__global__ void __launch_bounds__(WARPS * 32) filter_kernel(const float* x, const float* __restrict__ gain, int C,
                                                            int64_t T, const float* __restrict__ sos,
                                                            int64_t sos_items, int64_t n_chunks, int64_t work,
                                                            int reverse, const double* __restrict__ ws_s, float* out) {
  __shared__ float s_tile[WARPS][32 * (TILE + 1)];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t n_groups = (n_chunks + 31) / 32;
  for (int64_t w = (int64_t)blockIdx.x * WARPS + wid; w < work; w += (int64_t)gridDim.x * WARPS) {
    const int64_t row = w / n_groups, g = w - row * n_groups, b = row / C;
    const Coef<S> c = load_coef<S>(sos + (sos_items > 1 ? b : 0) * 6 * S);
    if (!c.stable) {  // warp-uniform: the whole item is NaN
      const int64_t lo = g * 32 * CHUNK, hi = lo + 32 * CHUNK < T ? lo + 32 * CHUNK : T;
      for (int64_t n = lo + lane; n < hi; n += 32) out[row * T + n] = __int_as_float(0x7fffffff);
      continue;
    }
    const float g0 = gain ? __ldg(gain + b) : 1.f;
    const int64_t k = g * 32 + lane;
    double z[2 * S];
#pragma unroll
    for (int i = 0; i < 2 * S; ++i) z[i] = k < n_chunks ? __ldg(ws_s + (row * n_chunks + k) * 2 * S + i) : 0.0;
    run_chunks<S, true>(x, out, row * T, T, g * 32 * CHUNK, g0, reverse, c, z, s_tile[wid]);
  }
}

}  // namespace iir
}  // namespace b2a

using namespace b2a::iir;

static int64_t iir_chunks(int64_t T) { return (T + CHUNK - 1) / CHUNK; }

extern "C" size_t b2a_sos_filter_workspace_bytes(int64_t B, int C, int64_t T, int S) {
  if (B < 1 || C < 1 || T < 1 || S < 1 || S > SMAX || T > INT64_MAX / 8 / B / C) return 0;
  return (size_t)(2 * B * C * iir_chunks(T) * 2 * S) * sizeof(double);
}

template <int S>
static int sos_launch(const float* x, const float* gain, int64_t B, int C, int64_t T, const float* sos,
                      int64_t sos_items, int reverse, float* out, float* ws, void* stream) {
  const int64_t rows = B * C, n_chunks = iir_chunks(T), work = rows * ((n_chunks + 31) / 32);
  double* ws_e = reinterpret_cast<double*>(ws);
  double* ws_s = ws_e + rows * n_chunks * 2 * S;
  const int64_t g13 = (work + WARPS - 1) / WARPS;
  const unsigned grid13 = (unsigned)(g13 < INT32_MAX ? g13 : INT32_MAX);
  const unsigned grid2 = (unsigned)(rows < INT32_MAX ? rows : INT32_MAX);
  B2A_LAUNCH(chunk_state_kernel<S>, dim3(grid13), dim3(WARPS * 32), 0, stream, x, gain, C, T, sos, sos_items, n_chunks,
             work, reverse, ws_e);
  B2A_CUDA_OK(cudaGetLastError());
  B2A_LAUNCH(carry_kernel<S>, dim3(grid2), dim3(32), 0, stream, sos, sos_items, C, rows, n_chunks, ws_e, ws_s);
  B2A_CUDA_OK(cudaGetLastError());
  B2A_LAUNCH(filter_kernel<S>, dim3(grid13), dim3(WARPS * 32), 0, stream, x, gain, C, T, sos, sos_items, n_chunks, work,
             reverse, ws_s, out);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" int b2a_sos_filter_f32(const float* x, const float* gain, int64_t B, int C, int64_t T, const float* sos,
                                  int64_t sos_items, int S, int reverse, float* out, void* ws, void* stream) {
  B2A_REQUIRE(x && sos && out && ws, B2A_E_INVALID, "sos_filter: null pointer");
  B2A_REQUIRE(B >= 1 && C >= 1 && T >= 1, B2A_E_INVALID, "sos_filter: bad shape B=%lld C=%d T=%lld", (long long)B, C,
              (long long)T);
  B2A_REQUIRE(T <= INT64_MAX / 8 / B / C, B2A_E_INVALID, "sos_filter: B * C * T overflows");
  B2A_REQUIRE(S >= 1 && S <= SMAX, B2A_E_INVALID, "sos_filter: %d sections; 1 .. %d are supported", S, SMAX);
  B2A_REQUIRE(sos_items == 1 || sos_items == B, B2A_E_INVALID,
              "sos_filter: sos_items must be 1 or B=%lld, got %lld", (long long)B, (long long)sos_items);
  float* w = static_cast<float*>(ws);
  switch (S) {
    case 1: return sos_launch<1>(x, gain, B, C, T, sos, sos_items, reverse, out, w, stream);
    case 2: return sos_launch<2>(x, gain, B, C, T, sos, sos_items, reverse, out, w, stream);
    case 3: return sos_launch<3>(x, gain, B, C, T, sos, sos_items, reverse, out, w, stream);
    case 4: return sos_launch<4>(x, gain, B, C, T, sos, sos_items, reverse, out, w, stream);
    case 5: return sos_launch<5>(x, gain, B, C, T, sos, sos_items, reverse, out, w, stream);
    case 6: return sos_launch<6>(x, gain, B, C, T, sos, sos_items, reverse, out, w, stream);
    case 7: return sos_launch<7>(x, gain, B, C, T, sos, sos_items, reverse, out, w, stream);
    default: return sos_launch<8>(x, gain, B, C, T, sos, sos_items, reverse, out, w, stream);
  }
}
