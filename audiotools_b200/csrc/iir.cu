// iir.cu -- per-item IIR biquad cascades of a batch (K19 in DESIGN.md): scipy.signal.sosfilt with zero or given
// initial state, and scipy.signal.sosfiltfilt (method "pad") with its gradient.
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
// and a chunk of CHUNK samples maps it to M = A^CHUNK.  A pass is three launches, no host sync, exact carries (no
// warm-up):
//   chunk_state_kernel   a warp per (row, 32 consecutive chunks), a lane per chunk: the recursion over the chunk
//                        from zero state gives the chunk's end state e_k.  Samples travel through a 32 x 32
//                        shared tile per warp, so every global access is a coalesced row of 32 floats.
//   carry_kernel         a warp per row: A from the item's coefficients in double, M and M^2, M^4, M^8, M^16 by
//                        squaring, then the affine scan s_{k+1} = M s_k + e_k from the start state s_0, 32 chunks at
//                        a time as a warp scan in double; writes every chunk's start state s_k.
//   filter_kernel        the layout of the first kernel: the recursion over the chunk from s_k writes y.
// A pass walks a virtual row v[m], m in [0, L) (struct Pass): the samples of x, or of the intermediate between the two
// passes of sosfiltfilt, read forwards or backwards, with scipy's edge extension applied in the loads.  s_0 is 0, a
// given zi, or sosfilt_zi(sos) v[0] (read on the device).  The filter kernel can also write the state after v[L - 1]
// (zf) and, per warp, G sum(v) - sum(y) (G: the cascade's DC gain), the rank-one term of the sosfiltfilt backward.
// Nothing depends on the launch geometry or on other items: reruns and batch-versus-single calls are bit-identical.
//
// The loudness backward (b2a_lufs_backward_f32, K21) runs two passes of the K-weighting on the LOUDNESS layout: the
// forward pass over a row of x zero-extended to Lmax samples stores u = wt[row] * m[e] * y (m[e]: the gating blocks
// kept by the forward that contain sample e) into the intermediate, and the reverse pass over the intermediate stores
// its first T samples (the adjoint of the zero extension) into grad_x.
#include "b2a_common.h"
#include "iir_internal.h"

namespace b2a {
namespace iir {

constexpr int CHUNK = 1024;   // samples of a row per chunk (one lane's sequential run); tests cover T = CHUNK +- 1
constexpr int TILE = 32;      // samples per lane per shared-memory tile
constexpr int WARPS = 8;      // warps per CTA of the chunk kernels
constexpr int SMAX = 8;       // largest number of sections

// padtype of b2a_sos_filtfilt_f32 (b2a.h); PAD_ZERO (outside [0, T) reads 0) is the backward's crop adjoint
enum { PAD_NONE = 0, PAD_ODD = 1, PAD_EVEN = 2, PAD_CONST = 3, PAD_ZERO = 4 };

// Row layouts of a pass: rows of x as they are (sosfilt); rows padded by the edge extension or read from the
// intermediate (sosfiltfilt); the loudness backward's rows (a row of x zero-extended to Lmax samples, or a row of the
// intermediate, with the gating weight applied on the store of the forward pass)
enum { ROWS = 0, EXTENDED = 1, LOUDNESS = 2 };

// One pass of the cascade over every row.  Row r of length L = T + 2 pl: m in [0, L) is the extended position
// e = (reverse ? L - 1 - m : m) - pl in [-pl, T + pl).  A source or destination row is either a row of T samples (x /
// out: e outside [0, T) is extended on load by padtype and dropped on store) or the intermediate, Lmax samples per row
// (index e + pl).
struct Pass {
  const float* src;         // [rows, T] or the intermediate
  const float* gain;        // [B] or null; scales rows of x only
  float* dst;               // [rows, T] or the intermediate
  const float* sos;
  int64_t sos_items;
  int C;
  int64_t T, Lmax;          // samples of a row of x; row stride of the intermediate, T + 2 max(pl)
  int64_t n_chunks, work;   // chunks of Lmax; warps of the chunk kernels
  int src_mid, dst_mid, reverse, padtype;
  int64_t padlen;           // >= 0, or < 0: scipy's default for the item's sections
  const double* zi;         // [S, rows, 2] start states, or null
  int zi_unit;              // start from sosfilt_zi(sos) v[0]
  double* zf;               // [S, rows, 2]: the state after v[L - 1], or null
  double* part;             // [rows, n_groups]: G sum(v) - sum(y) over a warp's chunks, or null
  const double* add_first;  // [rows, n_groups]: their sum is added to v[0], or null
  const double* wt;         // LOUDNESS: [rows] weight of the store, or null (no weight)
  const int* kept;          // LOUDNESS: [B, nblk + 1] running count of the kept gating blocks
  int nblk, blk_stride, blk_len;
};

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

// scipy's default padlen, 3 (2S + 1 - min(#{b2 == 0}, #{a2 == 0})), or the given one
__device__ __forceinline__ int64_t row_padlen(const float* so, int S, int64_t padlen) {
  if (padlen >= 0) return padlen;
  int nb = 0, na = 0;
  for (int s = 0; s < S; ++s) {
    const float a0 = so[6 * s + 3];
    nb += so[6 * s + 2] / a0 == 0.f;
    na += so[6 * s + 5] / a0 == 0.f;
  }
  return 3 * (2 * S + 1 - (nb < na ? nb : na));
}

// One row of a pass: pointers at the row, its padding and length
struct Row {
  const float* src;
  float* dst;
  int64_t T, L, pl;
  float g, first, last;  // gain; the gained first and last samples of a row of x (the extension's edges)
  int src_mid, dst_mid, reverse, padtype;
  double w;              // LOUDNESS: the row's weight (kept != null)
  const int* kept;       // LOUDNESS: the item's running count of kept blocks, or null
  int nblk, bs, bk;      // LOUDNESS: blocks, their stride and length in samples
};

__device__ __forceinline__ Row make_row(const Pass& p, int S, int64_t row, int64_t b) {
  Row r;
  const int64_t pl = row_padlen(p.sos + (p.sos_items > 1 ? b : 0) * 6 * S, S, p.padlen);
  r.src = p.src + row * (p.src_mid ? p.Lmax : p.T);
  r.dst = p.dst ? p.dst + row * (p.dst_mid ? p.Lmax : p.T) : nullptr;
  r.T = p.T, r.pl = pl, r.L = p.T + 2 * pl;
  r.g = p.gain ? __ldg(p.gain + b) : 1.f;
  r.first = p.src_mid ? 0.f : r.src[0] * r.g;
  r.last = p.src_mid ? 0.f : r.src[p.T - 1] * r.g;
  r.src_mid = p.src_mid, r.dst_mid = p.dst_mid, r.reverse = p.reverse, r.padtype = p.padtype;
  return r;
}

// make_row, and for LOUDNESS the virtual length Lmax and the store's weight
template <int LAY>
__device__ __forceinline__ Row make_row_as(const Pass& p, int S, int64_t row, int64_t b) {
  Row r = make_row(p, S, row, b);
  if (LAY == LOUDNESS) {
    r.L = p.Lmax;
    r.kept = p.wt ? p.kept + b * (p.nblk + 1) : nullptr;
    r.w = p.wt ? p.wt[row] : 0.0;
    r.nblk = p.nblk, r.bs = p.blk_stride, r.bk = p.blk_len;
  }
  return r;
}

// LOUDNESS: the number of kept blocks [i stride, i stride + len), 0 <= i < nblk, that contain sample e
__device__ __forceinline__ int kept_blocks(const Row& r, int64_t e) {
  const int64_t hi = e / r.bs < r.nblk - 1 ? e / r.bs : r.nblk - 1, lo = e < r.bk ? 0 : (e - r.bk) / r.bs + 1;
  return hi >= lo ? r.kept[hi + 1] - r.kept[lo] : 0;
}

// v[m]: 0 past the row's end.  ROWS: a row of x without padding (pl = 0, L = T), the zero-state filter's own index
// expression.  EXTENDED: one predicated load and selects, no divergent branch, so a tile's 32 loads issue together.
// LOUDNESS: a row of x reads 0 from T on.
template <int LAY>
__device__ __forceinline__ float load(const Row& r, int64_t m) {
  if (LAY == ROWS) return m < r.L ? r.src[r.reverse ? r.L - 1 - m : m] * r.g : 0.f;
  if (LAY == LOUDNESS) {
    const int64_t e = r.reverse ? r.L - 1 - m : m;
    return m < r.L && (r.src_mid || e < r.T) ? r.src[e] * r.g : 0.f;
  }
  const int64_t e = (r.reverse ? r.L - 1 - m : m) - r.pl;
  const bool inside = r.src_mid || (e >= 0 && e < r.T);
  const bool mirror = r.padtype == PAD_ODD || r.padtype == PAD_EVEN;
  const int64_t i = r.src_mid ? e + r.pl : e < 0 ? -e : e >= r.T ? 2 * (r.T - 1) - e : e;
  const float v = m < r.L && (inside || mirror) ? r.src[i] * (r.src_mid ? 1.f : r.g) : 0.f;
  if (inside || m >= r.L) return v;
  const float edge = e < 0 ? r.first : r.last;
  return r.padtype == PAD_ODD ? 2.f * edge - v : r.padtype == PAD_EVEN ? v : r.padtype == PAD_CONST ? edge : 0.f;
}

template <int LAY>
__device__ __forceinline__ void store(const Row& r, int64_t m, float y) {
  if (LAY == ROWS) {
    if (m < r.L) r.dst[r.reverse ? r.L - 1 - m : m] = y;
    return;
  }
  if (LAY == LOUDNESS) {
    const int64_t e = r.reverse ? r.L - 1 - m : m;
    if (m < r.L && (r.dst_mid || e < r.T)) r.dst[e] = r.kept ? (float)((double)y * r.w * kept_blocks(r, e)) : y;
    return;
  }
  const int64_t e = (r.reverse ? r.L - 1 - m : m) - r.pl;
  if (m < r.L && (r.dst_mid || (e >= 0 && e < r.T))) r.dst[r.dst_mid ? e + r.pl : e] = y;
}

// The sum of a row's n warp partials, the same order in every warp that asks
__device__ __forceinline__ double warp_sum(const double* v, int64_t n) {
  const int lane = threadIdx.x & 31;
  double a = 0.0;
  for (int64_t i = lane; i < n; i += 32) a += v[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  return a;
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

// What the filter kernel gathers besides y (EXTRA): the state after v[L - 1] and the sums of v and y over m < L
struct Extra {
  double* zf;           // this row's zf (section stride zf_stride), or null
  int64_t zf_stride;
  double sum_v, sum_y;
};

// Walk the warp's chunks tile by tile: lane l runs chunk g * 32 + l of the row from state z.  WRITE: y replaces the
// tile and is stored.  add0 (when `add`) is added to v[0].  Flat indices are 64-bit.
template <int S, bool WRITE, int LAY, bool EXTRA>
__device__ __forceinline__ void run_chunks(const Row& rw, int64_t first, bool add, double add0, const Coef<S>& c,
                                           double (&z)[2 * S], float* tile, Extra& ex) {
  const int lane = threadIdx.x & 31;
  const int64_t len = rw.L < CHUNK ? rw.L : CHUNK;
  const int n_tiles = (int)((len + TILE - 1) / TILE);
  for (int t = 0; t < n_tiles; ++t) {
    for (int r = 0; r < 32; ++r) {
      const int64_t n = first + (int64_t)r * CHUNK + t * TILE + lane;
      float v = load<LAY>(rw, n);
      if (LAY == EXTENDED && add && n == 0) v = (float)((double)v + add0);
      tile[r * (TILE + 1) + lane] = v;
    }
    __syncwarp();
    float* mine = tile + lane * (TILE + 1);
    const int64_t base = first + (int64_t)lane * CHUNK + t * TILE;  // position of mine[0]
#pragma unroll 4
    for (int k = 0; k < TILE; ++k) {
      const double u = (double)mine[k];
      const double y = step<S>(c, z, u);
      if (WRITE) mine[k] = (float)y;
      if (EXTRA) {
        if (base + k < rw.L) ex.sum_v += u, ex.sum_y += y;
        if (ex.zf && base + k == rw.L - 1) {
#pragma unroll
          for (int i = 0; i < 2 * S; ++i) ex.zf[(i >> 1) * ex.zf_stride + (i & 1)] = z[i];
        }
      }
    }
    __syncwarp();
    if (WRITE) {
      for (int r = 0; r < 32; ++r) {
        const int64_t n = first + (int64_t)r * CHUNK + t * TILE + lane;
        store<LAY>(rw, n, tile[r * (TILE + 1) + lane]);
      }
      __syncwarp();
    }
  }
}

// ws_e [rows, n_chunks, 2S]: end state of every chunk from zero state.
template <int S, int LAY>
__global__ void __launch_bounds__(WARPS * 32) chunk_state_kernel(const Pass p, double* __restrict__ ws_e) {
  __shared__ float s_tile[WARPS][32 * (TILE + 1)];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t n_chunks = p.n_chunks, n_groups = (n_chunks + 31) / 32;
  for (int64_t w = (int64_t)blockIdx.x * WARPS + wid; w < p.work; w += (int64_t)gridDim.x * WARPS) {
    const int64_t row = w / n_groups, g = w - row * n_groups, b = row / p.C;
    const Coef<S> c = load_coef<S>(p.sos + (p.sos_items > 1 ? b : 0) * 6 * S);
    const Row rw = make_row_as<LAY>(p, S, row, b);
    const bool add = p.add_first && g == 0;
    const double add0 = add ? warp_sum(p.add_first + row * n_groups, n_groups) : 0.0;
    double z[2 * S];
#pragma unroll
    for (int i = 0; i < 2 * S; ++i) z[i] = 0.0;
    Extra ex{};
    run_chunks<S, false, LAY, false>(rw, g * 32 * CHUNK, add, add0, c, z, s_tile[wid], ex);
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

// s_0 of a row: the given zi, or sosfilt_zi(sos) v[0] -- each section's lfilter_zi, (I - A_s)^-1 B_s in closed form,
// times the DC gains of the sections before it, in double from the float32 coefficients
template <int S>
__device__ __forceinline__ void start_state(const Pass& p, int64_t row, int64_t b, int64_t rows, double (&s0)[2 * S]) {
  if (p.zi) {
#pragma unroll
    for (int i = 0; i < 2 * S; ++i) s0[i] = p.zi[((i >> 1) * rows + row) * 2 + (i & 1)];
    return;
  }
  const float* so = p.sos + (p.sos_items > 1 ? b : 0) * 6 * S;
  const double v = (double)load<EXTENDED>(make_row(p, S, row, b), 0);
  double scale = v;
#pragma unroll
  for (int s = 0; s < S; ++s) {
    const float a0 = so[6 * s + 3];
    const double b0 = (double)(so[6 * s] / a0), b1 = (double)(so[6 * s + 1] / a0), b2 = (double)(so[6 * s + 2] / a0),
                 a1 = (double)(so[6 * s + 4] / a0), a2 = (double)(so[6 * s + 5] / a0);
    const double B1 = b1 - a1 * b0, B2 = b2 - a2 * b0, z1 = (B1 + B2) / (1.0 + a1 + a2);
    s0[2 * s] = scale * z1;
    s0[2 * s + 1] = scale * (B2 - a2 * z1);
    scale *= (b0 + b1 + b2) / (1.0 + a1 + a2);
  }
}

// One warp (one CTA) per row.  ws_s [rows, n_chunks, 2S]: the start state of every chunk.
template <int S>
__global__ void __launch_bounds__(32) carry_kernel(const Pass p, const double* __restrict__ ws_e,
                                                   double* __restrict__ ws_s) {
  constexpr int N = 2 * S;
  __shared__ double s_pow[6][N * N];  // M, M^2, M^4, M^8, M^16; [5] scratch
  const int lane = threadIdx.x;
  const int64_t rows = p.work / ((p.n_chunks + 31) / 32), n_chunks = p.n_chunks;
  const bool has_s0 = p.zi || p.zi_unit;
  for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
    const int64_t b = row / p.C;
    const float* so = p.sos + (p.sos_items > 1 ? b : 0) * 6 * S;
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
      for (int p2 = 1; p2 < CHUNK; p2 *= 2) {
        square<N>(s_pow[cur], s_pow[5 - cur]);
        cur = 5 - cur;
      }
      if (cur != 0) {
        for (int o = lane; o < N * N; o += 32) s_pow[0][o] = s_pow[cur][o];
        __syncwarp();
      }
      for (int q = 1; q < 5; ++q) square<N>(s_pow[q - 1], s_pow[q]);
    }
    double carry[N];  // start state of the batch's first chunk
#pragma unroll
    for (int i = 0; i < N; ++i) carry[i] = 0.0;
    if (has_s0) start_state<S>(p, row, b, rows, carry);
    if (lane == 0) {
#pragma unroll
      for (int i = 0; i < N; ++i) ws_s[row * n_chunks * N + i] = carry[i];  // s_0
    }
    for (int64_t base = 0; base + 1 < n_chunks; base += 32) {  // the last chunk's end state is not needed
      const int64_t k = base + lane;
      double v[N], w[N];
#pragma unroll
      for (int i = 0; i < N; ++i) v[i] = k < n_chunks ? ws_e[(row * n_chunks + k) * N + i] : 0.0;
      if (lane == 0 && (base > 0 || has_s0)) matvec_add<N>(s_pow[0], carry, v);
      // inclusive scan: lane l ends with the end state of chunk base + l, i.e. the start state of chunk base + l + 1
#pragma unroll
      for (int q = 0; q < 5; ++q) {
        const int o = 1 << q;
#pragma unroll
        for (int i = 0; i < N; ++i) w[i] = __shfl_up_sync(0xffffffffu, v[i], o);
        if (lane >= o) matvec_add<N>(s_pow[q], w, v);
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

template <int S, int LAY, bool EXTRA>
__global__ void __launch_bounds__(WARPS * 32) filter_kernel(const Pass p, const double* __restrict__ ws_s) {
  __shared__ float s_tile[WARPS][32 * (TILE + 1)];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t n_chunks = p.n_chunks, n_groups = (n_chunks + 31) / 32, rows = p.work / n_groups;
  for (int64_t w = (int64_t)blockIdx.x * WARPS + wid; w < p.work; w += (int64_t)gridDim.x * WARPS) {
    const int64_t row = w / n_groups, g = w - row * n_groups, b = row / p.C;
    const Coef<S> c = load_coef<S>(p.sos + (p.sos_items > 1 ? b : 0) * 6 * S);
    const Row rw = make_row_as<LAY>(p, S, row, b);
    const int64_t lo = g * 32 * CHUNK, hi = lo + 32 * CHUNK < rw.L ? lo + 32 * CHUNK : rw.L;
    if (!c.stable) {  // warp-uniform: the whole item is NaN
      const float nan = __int_as_float(0x7fffffff);
      for (int64_t m = lo + lane; m < hi; m += 32) store<LAY>(rw, m, nan);
      if (EXTRA && lane == 0) {
        if (p.zf && rw.L - 1 >= lo && rw.L - 1 < hi) {
          for (int i = 0; i < 2 * S; ++i) p.zf[((i >> 1) * rows + row) * 2 + (i & 1)] = (double)nan;
        }
        if (p.part) p.part[row * n_groups + g] = (double)nan;
      }
      continue;
    }
    const bool add = p.add_first && g == 0;
    const double add0 = add ? warp_sum(p.add_first + row * n_groups, n_groups) : 0.0;
    const int64_t k = g * 32 + lane;
    double z[2 * S];
#pragma unroll
    for (int i = 0; i < 2 * S; ++i) z[i] = k < n_chunks ? __ldg(ws_s + (row * n_chunks + k) * 2 * S + i) : 0.0;
    Extra ex{p.zf ? p.zf + row * 2 : nullptr, rows * 2, 0.0, 0.0};
    run_chunks<S, true, LAY, EXTRA>(rw, lo, add, add0, c, z, s_tile[wid], ex);
    if (EXTRA && p.part) {
      double sv = ex.sum_v, sy = ex.sum_y;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        sv += __shfl_xor_sync(0xffffffffu, sv, o);
        sy += __shfl_xor_sync(0xffffffffu, sy, o);
      }
      double G = 1.0;  // the cascade's gain at DC, as start_state's scale
#pragma unroll
      for (int s = 0; s < S; ++s) G *= (c.b0[s] + c.b1[s] + c.b2[s]) / (1.0 + c.a1[s] + c.a2[s]);
      if (lane == 0) p.part[row * n_groups + g] = G * sv - sy;
    }
  }
}

// The sosfiltfilt backward's last step: grad_x = gain E^T f, E the edge extension, f the intermediate with the sum of
// `part` added to its first sample (f = K^T ..., K = H + c e_0^T)
__global__ void __launch_bounds__(256) fold_kernel(const Pass p, int S, const double* __restrict__ part,
                                                   const float* __restrict__ f, float* __restrict__ gx) {
  const int64_t n_groups = (p.n_chunks + 31) / 32, rows = p.work / n_groups, T = p.T, total = rows * T;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / T, n = i - row * T, b = row / p.C;
    const int64_t pl = row_padlen(p.sos + (p.sos_items > 1 ? b : 0) * 6 * S, S, p.padlen);
    const float* fr = f + row * p.Lmax;
    const double* pr = part + row * n_groups;
    auto F = [&](int64_t j) -> double {
      double v = (double)fr[j];
      if (j == 0) {
        for (int64_t q = 0; q < n_groups; ++q) v += pr[q];
      }
      return v;
    };
    double acc = F(pl + n);
    if (pl > 0) {
      if (p.padtype == PAD_ODD || p.padtype == PAD_EVEN) {  // the mirrored samples
        const double sgn = p.padtype == PAD_ODD ? -1.0 : 1.0;
        if (n >= 1 && n <= pl) acc += sgn * F(pl - n);
        if (T - 1 - n >= 1 && T - 1 - n <= pl) acc += sgn * F(2 * T - 2 + pl - n);
      }
      if (p.padtype == PAD_ODD || p.padtype == PAD_CONST) {  // the edge sample, 2 x[0] (odd) or x[0] (constant)
        const double wt = p.padtype == PAD_ODD ? 2.0 : 1.0;
        if (n == 0) {
          for (int64_t q = 1; q <= pl; ++q) acc += wt * F(pl - q);
        }
        if (n == T - 1) {
          for (int64_t q = 1; q <= pl; ++q) acc += wt * F(pl + T - 1 + q);
        }
      }
    }
    gx[i] = (float)(acc * (double)(p.gain ? __ldg(p.gain + b) : 1.f));
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

// The three launches of one pass; ws_e / ws_s: [rows, n_chunks, 2S] doubles each
// LAY: ROWS (rows of x as they are: sosfilt), EXTENDED (sosfiltfilt) or LOUDNESS
template <int S, int LAY>
static int run_pass(const Pass& p, double* ws_e, double* ws_s, void* stream) {
  const int64_t rows = p.work / ((p.n_chunks + 31) / 32);
  const int64_t g13 = (p.work + WARPS - 1) / WARPS;
  const unsigned grid13 = (unsigned)(g13 < INT32_MAX ? g13 : INT32_MAX);
  const unsigned grid2 = (unsigned)(rows < INT32_MAX ? rows : INT32_MAX);
  void (*chunk_state)(const Pass, double*) = chunk_state_kernel<S, LAY>;
  B2A_LAUNCH(chunk_state, dim3(grid13), dim3(WARPS * 32), 0, stream, p, ws_e);
  B2A_CUDA_OK(cudaGetLastError());
  B2A_LAUNCH(carry_kernel<S>, dim3(grid2), dim3(32), 0, stream, p, ws_e, ws_s);
  B2A_CUDA_OK(cudaGetLastError());
  void (*filter)(const Pass, const double*) =
      p.zf || p.part ? filter_kernel<S, LAY, true> : filter_kernel<S, LAY, false>;
  B2A_LAUNCH(filter, dim3(grid13), dim3(WARPS * 32), 0, stream, p, ws_s);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

template <int LAY>
static int pass_launch(int S, const Pass& p, double* ws_e, double* ws_s, void* stream) {
  switch (S) {
    case 1: return run_pass<1, LAY>(p, ws_e, ws_s, stream);
    case 2: return run_pass<2, LAY>(p, ws_e, ws_s, stream);
    case 3: return run_pass<3, LAY>(p, ws_e, ws_s, stream);
    case 4: return run_pass<4, LAY>(p, ws_e, ws_s, stream);
    case 5: return run_pass<5, LAY>(p, ws_e, ws_s, stream);
    case 6: return run_pass<6, LAY>(p, ws_e, ws_s, stream);
    case 7: return run_pass<7, LAY>(p, ws_e, ws_s, stream);
    default: return run_pass<8, LAY>(p, ws_e, ws_s, stream);
  }
}

// A pass over rows of T samples padded by up to pmax on either side: everything but the buffers
static Pass make_pass(int64_t B, int C, int64_t T, int64_t pmax, const float* sos, int64_t sos_items) {
  Pass p{};
  p.sos = sos, p.sos_items = sos_items, p.C = C, p.T = T, p.Lmax = T + 2 * pmax;
  p.n_chunks = iir_chunks(p.Lmax);
  p.work = B * C * ((p.n_chunks + 31) / 32);
  return p;
}

static int check_args(const char* name, const void* x, const float* sos, const void* out, const void* ws, int64_t B,
                      int C, int64_t T, int S, int64_t sos_items) {
  B2A_REQUIRE(x && sos && out && ws, B2A_E_INVALID, "%s: null pointer", name);
  B2A_REQUIRE(B >= 1 && C >= 1 && T >= 1, B2A_E_INVALID, "%s: bad shape B=%lld C=%d T=%lld", name, (long long)B, C,
              (long long)T);
  B2A_REQUIRE(T <= INT64_MAX / 8 / B / C, B2A_E_INVALID, "%s: B * C * T overflows", name);
  B2A_REQUIRE(S >= 1 && S <= SMAX, B2A_E_INVALID, "%s: %d sections; 1 .. %d are supported", name, S, SMAX);
  B2A_REQUIRE(sos_items == 1 || sos_items == B, B2A_E_INVALID, "%s: sos_items must be 1 or B=%lld, got %lld", name,
              (long long)B, (long long)sos_items);
  return B2A_OK;
}

extern "C" int b2a_sos_filter_f32(const float* x, const float* gain, int64_t B, int C, int64_t T, const float* sos,
                                  int64_t sos_items, int S, int reverse, float* out, void* ws, void* stream) {
  const int rc = check_args("sos_filter", x, sos, out, ws, B, C, T, S, sos_items);
  if (rc != B2A_OK) return rc;
  Pass p = make_pass(B, C, T, 0, sos, sos_items);
  p.src = x, p.gain = gain, p.dst = out, p.reverse = reverse;
  double* ws_e = static_cast<double*>(ws);
  return pass_launch<ROWS>(S, p, ws_e, ws_e + B * C * p.n_chunks * 2 * S, stream);
}

extern "C" int b2a_sos_filter_zi_f32(const float* x, const float* gain, int64_t B, int C, int64_t T, const float* sos,
                                     int64_t sos_items, int S, const double* zi, float* out, double* zf, void* ws,
                                     void* stream) {
  const int rc = check_args("sos_filter_zi", x, sos, out, ws, B, C, T, S, sos_items);
  if (rc != B2A_OK) return rc;
  B2A_REQUIRE(zi, B2A_E_INVALID, "sos_filter_zi: null pointer");
  Pass p = make_pass(B, C, T, 0, sos, sos_items);
  p.src = x, p.gain = gain, p.dst = out, p.zi = zi, p.zf = zf;
  double* ws_e = static_cast<double*>(ws);
  return pass_launch<ROWS>(S, p, ws_e, ws_e + B * C * p.n_chunks * 2 * S, stream);
}

// Largest padding of a call: none, the given padlen, or scipy's default at its largest, 3 (2S + 1); -1 when invalid
static int64_t filtfilt_pmax(int S, int padtype, int64_t padlen) {
  if (padtype < PAD_NONE || padtype > PAD_CONST) return -1;
  if (padtype == PAD_NONE) return 0;
  return padlen >= 0 ? padlen : 3 * (2 * S + 1);
}

// Workspace of sosfiltfilt and its backward, doubles first: ws_e, ws_s [rows, n_chunks, 2S], two partial arrays
// [rows, n_groups], then the intermediate [rows, Lmax] floats
struct FiltFiltWs {
  double *e, *s, *part_a, *part_b;
  float* mid;
  size_t bytes;
};

static FiltFiltWs filtfilt_ws(const Pass& p, int S, int64_t rows, void* ws) {
  FiltFiltWs w;
  const int64_t n_groups = (p.n_chunks + 31) / 32, states = rows * p.n_chunks * 2 * S;
  double* d = static_cast<double*>(ws);
  w.e = d, w.s = d + states, w.part_a = d + 2 * states, w.part_b = w.part_a + rows * n_groups;
  w.mid = reinterpret_cast<float*>(w.part_b + rows * n_groups);
  w.bytes = (size_t)(2 * states + 2 * rows * n_groups) * sizeof(double) + (size_t)(rows * p.Lmax) * sizeof(float);
  return w;
}

extern "C" size_t b2a_sos_filtfilt_workspace_bytes(int64_t B, int C, int64_t T, int S, int padtype, int64_t padlen) {
  const int64_t pmax = filtfilt_pmax(S, padtype, padlen);
  if (B < 1 || C < 1 || T < 1 || S < 1 || S > SMAX || pmax < 0 || T > INT64_MAX / 32 / B / C || T <= pmax) return 0;
  return filtfilt_ws(make_pass(B, C, T, pmax, nullptr, 1), S, B * C, nullptr).bytes;
}

static int filtfilt_check(const char* name, const float* x, const float* sos, const float* out, const void* ws,
                          int64_t B, int C, int64_t T, int S, int64_t sos_items, int padtype, int64_t padlen) {
  const int rc = check_args(name, x, sos, out, ws, B, C, T, S, sos_items);
  if (rc != B2A_OK) return rc;
  B2A_REQUIRE(T <= INT64_MAX / 32 / B / C, B2A_E_INVALID, "%s: B * C * T overflows", name);
  const int64_t pmax = filtfilt_pmax(S, padtype, padlen);
  B2A_REQUIRE(pmax >= 0, B2A_E_INVALID, "%s: padtype %d; 0 (none), 1 (odd), 2 (even) or 3 (constant)", name, padtype);
  B2A_REQUIRE(T > pmax, B2A_E_INVALID, "%s: T=%lld must exceed the padding %lld", name, (long long)T, (long long)pmax);
  return B2A_OK;
}

extern "C" int b2a_sos_filtfilt_f32(const float* x, const float* gain, int64_t B, int C, int64_t T, const float* sos,
                                    int64_t sos_items, int S, int padtype, int64_t padlen, float* out, void* ws,
                                    void* stream) {
  const int rc = filtfilt_check("sos_filtfilt", x, sos, out, ws, B, C, T, S, sos_items, padtype, padlen);
  if (rc != B2A_OK) return rc;
  const int64_t pmax = filtfilt_pmax(S, padtype, padlen);
  Pass p = make_pass(B, C, T, pmax, sos, sos_items);
  const FiltFiltWs w = filtfilt_ws(p, S, B * C, ws);
  p.padtype = padtype, p.padlen = padtype == PAD_NONE ? 0 : padlen, p.zi_unit = 1;
  // forward over the extended row into the intermediate, from sosfilt_zi * ext[0]
  p.src = x, p.gain = gain, p.dst = w.mid, p.dst_mid = 1;
  int r = pass_launch<EXTENDED>(S, p, w.e, w.s, stream);
  if (r != B2A_OK) return r;
  // backwards over the intermediate, from sosfilt_zi * its last sample, cropped into out
  p.src = w.mid, p.src_mid = 1, p.gain = nullptr, p.dst = out, p.dst_mid = 0, p.reverse = 1;
  return pass_launch<EXTENDED>(S, p, w.e, w.s, stream);
}

extern "C" int b2a_sos_filtfilt_backward_f32(const float* grad_y, const float* gain, int64_t B, int C, int64_t T,
                                             const float* sos, int64_t sos_items, int S, int padtype, int64_t padlen,
                                             float* grad_x, void* ws, void* stream) {
  const int rc = filtfilt_check("sos_filtfilt_backward", grad_y, sos, grad_x, ws, B, C, T, S, sos_items, padtype,
                                padlen);
  if (rc != B2A_OK) return rc;
  const int64_t pmax = filtfilt_pmax(S, padtype, padlen);
  Pass p = make_pass(B, C, T, pmax, sos, sos_items);
  const FiltFiltWs w = filtfilt_ws(p, S, B * C, ws);
  p.padlen = padtype == PAD_NONE ? 0 : padlen;
  // H P^T g into the intermediate (the crop's adjoint pads with zeros), and r1 = G sum(g) - sum(H P^T g)
  p.src = grad_y, p.padtype = PAD_ZERO, p.dst = w.mid, p.dst_mid = 1, p.part = w.part_a;
  int r = pass_launch<EXTENDED>(S, p, w.e, w.s, stream);
  if (r != B2A_OK) return r;
  // H^T (w + r1 e_last), in place, and r2 = G sum(w') - sum(H^T w')
  p.src = w.mid, p.src_mid = 1, p.reverse = 1, p.add_first = w.part_a, p.part = w.part_b;
  r = pass_launch<EXTENDED>(S, p, w.e, w.s, stream);
  if (r != B2A_OK) return r;
  // grad_x = gain E^T (f + r2 e_0)
  p.padtype = padtype, p.gain = gain;
  const int64_t total = B * C * T, blocks = (total + 255) / 256;
  B2A_LAUNCH(fold_kernel, dim3((unsigned)(blocks < 65536 * 16 ? blocks : 65536 * 16)), dim3(256), 0, stream, p, S,
             w.part_b, w.mid, grad_x);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

// ---- the loudness backward's two passes (iir_internal.h)
namespace b2a {
namespace iir {

size_t loudness_adjoint_workspace_bytes(int64_t rows, int64_t Tp, int S) {
  return (size_t)(2 * rows * iir_chunks(Tp) * 2 * S) * sizeof(double) + (size_t)(rows * Tp) * sizeof(float);
}

int loudness_adjoint(const float* x, const float* gain, int64_t B, int C, int64_t T, int64_t Tp, const float* sos,
                     int S, const double* wt, const int* kept, int nblk, int blk_stride, int blk_len, float* grad_x,
                     void* ws, void* stream) {
  B2A_REQUIRE(S == 1 || S == 2, B2A_E_UNSUPPORTED, "lufs_backward: %d sections (1 or 2)", S);
  Pass p = make_pass(B, C, T, 0, sos, 1);
  p.Lmax = Tp, p.n_chunks = iir_chunks(Tp), p.work = B * C * ((p.n_chunks + 31) / 32);
  p.kept = kept, p.nblk = nblk, p.blk_stride = blk_stride, p.blk_len = blk_len;
  const int64_t states = B * C * p.n_chunks * 2 * S;
  double* ws_e = static_cast<double*>(ws);
  float* u = reinterpret_cast<float*>(ws_e + 2 * states);
  // u = wt m K x over the zero-extended row, into the intermediate
  p.src = x, p.gain = gain, p.dst = u, p.dst_mid = 1, p.wt = wt;
  int r = S == 1 ? run_pass<1, LOUDNESS>(p, ws_e, ws_e + states, stream)
                 : run_pass<2, LOUDNESS>(p, ws_e, ws_e + states, stream);
  if (r != B2A_OK) return r;
  // grad_x = the first T samples of K^T u
  p.src = u, p.src_mid = 1, p.gain = nullptr, p.dst = grad_x, p.dst_mid = 0, p.reverse = 1, p.wt = nullptr;
  return S == 1 ? run_pass<1, LOUDNESS>(p, ws_e, ws_e + states, stream)
                : run_pass<2, LOUDNESS>(p, ws_e, ws_e + states, stream);
}

}  // namespace iir
}  // namespace b2a
