// specmask.cu -- in-place operations on a complex STFT [rows, F, N] for the SpectralTransform family, sm_90a.
//
// The reference expresses every one of them through |X|, angle(X), masked_fill and mag * exp(1j * phase)
// (ref:audiotools/core/dsp.py:217-370): about a dozen elementwise passes over the spectrogram each.  Here:
//   band_mask_kernel   mask_frequencies / mask_timesteps (:217-306).  Cells outside the band are unchanged by the
//                      reference's polar round trip (up to its rounding), so the kernel touches ONLY masked cells:
//                      it evaluates lo[item] <= axis_val < hi[item] in float32 exactly as the reference does
//                      (axis_val = the reference's own torch.linspace values, passed in) and stores the constant
//                      fill = val * exp(1j * val).  No loads of the spectrogram; one CTA per (row, bin) line.
//   rotate_kernel      shift_phase (:335-351): X *= exp(1j * shift), shift per item or per cell -- one read, one write.
//   maxpow_kernel +    mask_low_magnitudes (:308-333): log_magnitude()'s top_db floor needs the global maximum of
//   mask_low_kernel    |X|^2 (one read-only pass, atomicMax on the bit pattern), then cells whose
//                      10 log10(max(|X|^2, 1e-10)) (floored at max - 80 dB) is below the item's cut-off get
//                      magnitude `val` and keep their phase; only those cells are written.
// The gradient path (a spectrogram that requires a gradient) cannot write in place: autograd may have saved the input
// for another node.  Its forwards write a new tensor (one read, one write per cell) and its backwards recompute the
// mask decision from the saved X with the forward's own arithmetic:
//   band_mask_out_kernel<false> / <true>   out = band ? fill : X  /  gX = band || X == 0 ? 0 : g
//   mask_low_out_kernel, mask_low_bwd_kernel  unmasked: g (0 at X == 0); masked: val (g - Re(g conj u) u) / |X|,
//                      u = X / |X| (the phase's derivative, evaluated in float64; 0 at X == 0 and for val == 0)
//   gate_apply_kernel  reads the booleans from one tensor (X) and multiplies another (X forward, g backward)
#include "b2a_common.h"

namespace b2a {
namespace specmask {

__global__ void __launch_bounds__(256)
band_mask_kernel(float2* __restrict__ spec, int F, int N, const float* __restrict__ axis_vals,
                 const float* __restrict__ lo, const float* __restrict__ hi, int rows_per_item, int axis, float2 fill) {
  const int line = blockIdx.x;  // row * F + f
  const int row = line / F, f = line - row * F;
  const int item = row / rows_per_item;
  const float l = __ldg(lo + item), h = __ldg(hi + item);
  float2* p = spec + (size_t)line * N;
  if (axis == 0) {
    const float v = __ldg(axis_vals + f);
    if (!(l <= v && v < h)) return;  // CTA-uniform: the whole line is outside the band
    for (int n = threadIdx.x; n < N; n += blockDim.x) p[n] = fill;
  } else {
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
      const float v = __ldg(axis_vals + n);
      if (l <= v && v < h) p[n] = fill;
    }
  }
}

// BWD false: out = in band ? fill : spec.  BWD true: out = in band || spec == 0 ? 0 : g (fill is 0).  The band test is
// band_mask_kernel's; a line inside a frequency band reads nothing.
template <bool BWD>
__global__ void __launch_bounds__(256)
band_mask_out_kernel(const float2* __restrict__ g, const float2* __restrict__ spec, float2* __restrict__ out, int F,
                     int N, const float* __restrict__ axis_vals, const float* __restrict__ lo,
                     const float* __restrict__ hi, int rows_per_item, int axis, float2 fill) {
  const int line = blockIdx.x;  // row * F + f
  const int row = line / F, f = line - row * F;
  const int item = row / rows_per_item;
  const float l = __ldg(lo + item), h = __ldg(hi + item);
  const size_t base = (size_t)line * N;
  bool line_in = false;
  if (axis == 0) {
    const float v = __ldg(axis_vals + f);
    line_in = l <= v && v < h;  // CTA-uniform
  }
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    bool in = line_in;
    if (axis != 0) {
      const float v = __ldg(axis_vals + n);
      in = l <= v && v < h;
    }
    float2 r = fill;
    if (!in) {
      r = spec[base + n];
      if (BWD) r = (r.x == 0.f && r.y == 0.f) ? make_float2(0.f, 0.f) : g[base + n];
    }
    out[base + n] = r;
  }
}

// mode 0: shift[item]; mode 1: shift[cell]
__global__ void __launch_bounds__(256)
rotate_kernel(float2* __restrict__ spec, long long total, long long cells_per_item, const float* __restrict__ shift,
              int mode) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const float s = mode ? __ldg(shift + i) : __ldg(shift + i / cells_per_item);
    float sn, cs;
    sincosf(s, &sn, &cs);
    const float2 z = spec[i];
    spec[i] = make_float2(z.x * cs - z.y * sn, z.x * sn + z.y * cs);
  }
}

__device__ __forceinline__ float power_of(float2 z) {
  const float mag = hypotf(z.x, z.y);  // torch.abs(complex64)
  return mag * mag;                    // .pow(2)
}

// max(a, b) as torch.maximum and clamp compute it: NaN if either is NaN (fmaxf would drop the NaN).  Equal to fmaxf
// for any other pair.
__device__ __forceinline__ float max_nan(float a, float b) { return (a != a || b != b) ? a + b : fmaxf(a, b); }

// The maximum of |X|^2 as an unsigned max of bit patterns: |X|^2 is +0 or positive, and those order like their bits.
// Every NaN pattern, of either sign, ranks above +inf's 0x7f800000, so a NaN anywhere in the batch wins, as in
// log_spec.max(); it is stored as the positive quiet NaN 0x7fffffff.
__global__ void __launch_bounds__(256)
maxpow_kernel(const float2* __restrict__ spec, long long total, unsigned* __restrict__ max_bits) {
  unsigned m = 0u;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    m = max(m, __float_as_uint(power_of(spec[i])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ unsigned sm[8];
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) m = max(m, sm[w]);
    atomicMax(max_bits, m > 0x7f800000u ? 0x7fffffffu : m);
  }
}

// log_magnitude()'s top_db floor from the maximum maxpow_kernel found (NaN when the batch holds a NaN)
__device__ __forceinline__ float mask_low_floor(const unsigned* max_bits, float amin2, float top_db) {
  return 10.0f * log10f(max_nan(__uint_as_float(*max_bits), amin2)) - top_db;
}

// the mask decision of mask_low_magnitudes, shared by the forwards and the backward.  torch.maximum(log_spec, NaN) is
// NaN and NaN < cut is false: a NaN floor masks nothing.  A NaN cell makes the floor NaN (it enters the batch's
// maximum), so the cell's own power needs no test, and the floor's is the same for every cell of a launch.
__device__ __forceinline__ bool mask_low_cell(float2 z, float floor_db, float cut, float amin2) {
  float db = 10.0f * log10f(fmaxf(power_of(z), amin2));
  db = fmaxf(db, floor_db);
  return db < cut && floor_db == floor_db;
}

// magnitude := val, phase kept: val * exp(1j * atan2(im, re))
__device__ __forceinline__ float2 keep_phase(float2 z, float val) {
  const float ph = atan2f(z.y, z.x);
  float sn, cs;
  sincosf(ph, &sn, &cs);
  return make_float2(val * cs, val * sn);
}

__global__ void __launch_bounds__(256)
mask_low_kernel(float2* __restrict__ spec, long long total, long long cells_per_item, const float* __restrict__ cutoff,
                const unsigned* __restrict__ max_bits, float amin2, float top_db, float val) {
  const float floor_db = mask_low_floor(max_bits, amin2, top_db);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const float2 z = spec[i];
    if (mask_low_cell(z, floor_db, __ldg(cutoff + i / cells_per_item), amin2)) spec[i] = keep_phase(z, val);
  }
}

__global__ void __launch_bounds__(256)
mask_low_out_kernel(const float2* __restrict__ spec, float2* __restrict__ out, long long total, long long cells_per_item,
                    const float* __restrict__ cutoff, const unsigned* __restrict__ max_bits, float amin2, float top_db,
                    float val) {
  const float floor_db = mask_low_floor(max_bits, amin2, top_db);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const float2 z = spec[i];
    out[i] = mask_low_cell(z, floor_db, __ldg(cutoff + i / cells_per_item), amin2) ? keep_phase(z, val) : z;
  }
}

__global__ void __launch_bounds__(256)
mask_low_bwd_kernel(const float2* __restrict__ g, const float2* __restrict__ spec, float2* __restrict__ gx,
                    long long total, long long cells_per_item, const float* __restrict__ cutoff,
                    const unsigned* __restrict__ max_bits, float amin2, float top_db, float val) {
  const float floor_db = mask_low_floor(max_bits, amin2, top_db);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const float2 z = spec[i];
    float2 r = make_float2(0.f, 0.f);  // X == 0: |X| and angle(X) both backpropagate 0
    if (z.x != 0.f || z.y != 0.f) {
      const float2 gi = g[i];
      if (!mask_low_cell(z, floor_db, __ldg(cutoff + i / cells_per_item), amin2)) {
        r = gi;
      } else if (val != 0.f) {
        // val * exp(1j angle X): the tangential part of g scaled by val / |X|, i.e. val Im(g conj X) / |X|^3 * (1j X).
        // In float64: the factor 1 / |X| amplifies every float32 rounding of the small cells, and only masked cells
        // with a non-zero fill take this branch.
        const double x = z.x, y = z.y;
        const double p = x * x + y * y;
        const double s = (double)val * ((double)gi.y * x - (double)gi.x * y) / (p * sqrt(p));
        r = make_float2((float)(-s * y), (float)(s * x));
      }
    }
    gx[i] = r;
  }
}


// ---------------------------------------------------------------------------------------------
// Spectral noise gate (ref:audiotools/ml/layers/spectral_gate.py:60-129; the reference: |X| -> dB -> mean/std over time
// -> compare -> conv2d(7 x 11 triangle) -> 1 - amount * mask -> multiply: eight tensor passes + cuDNN).
//   gate_stats_kernel  per (noise row, bin): thresh = mean_t(db) + n_std * std_t(db) (unbiased, torch.std), with
//                      db = 20 log10(max(|X|, 1e-4)); one warp per line, frames contiguous.
//   gate_apply_kernel  out = Y * (1 - amount[item] * S),  S = the zero-padded 2-D smoothing of the boolean
//                      (db(X) < thresh[bin]) with the SEPARABLE kernel rf (x) rt / sum: a CTA stages the booleans of a
//                      (TF + 2 hf) x (TT + 2 ht) tile, smooths along time, then along frequency, and writes the
//                      product -- one read and one write of the spectrogram (out of place: neighbours read |X|).
//                      Y = X in the forward; Y = g in the backward (S is a constant of the gradient: the reference
//                      builds it from a comparison), which reads X again and the saved thresholds.
// ---------------------------------------------------------------------------------------------
// clamp(1e-4) keeps a NaN: a NaN cell of the signal is never below its threshold, and one in the noise makes its
// bin's threshold NaN, so that bin is never gated
__device__ __forceinline__ float gate_db(float2 z) { return 20.0f * log10f(max_nan(hypotf(z.x, z.y), 1e-4f)); }

__global__ void __launch_bounds__(256)
gate_stats_kernel(const float2* __restrict__ nz, int lines, int N, float n_std, float* __restrict__ thresh) {
  const int line = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;  // one warp per (row, bin) line
  if (line >= lines) return;
  const float2* p = nz + (size_t)line * N;
  float a = 0.f;
  for (int n = lane; n < N; n += 32) a += gate_db(p[n]);
  const float mean = warp_sum(a) / (float)N;
  float q = 0.f;
  for (int n = lane; n < N; n += 32) { const float d = gate_db(p[n]) - mean; q = fmaf(d, d, q); }
  q = warp_sum(q);
  if (lane == 0) thresh[line] = mean + sqrtf(q / (float)(N - 1)) * n_std;  // unbiased; N == 1 -> nan, as torch.std
}

constexpr int GT_F = 16, GT_T = 64, G_MAXH = 8;  // tile, largest half-width of either smoothing vector

struct GateParams {
  const float2* spec;    // X: the booleans
  const float2* mul;     // the tensor multiplied (X, or the output gradient)
  float2* out;
  const float* thresh;   // [nz_rows, F]
  const float* amount;   // [rows / rows_per_item]
  int F, N, rows_per_item, nz_rows, hf, ht;
  float rf[2 * G_MAXH + 1], rt[2 * G_MAXH + 1];  // smoothing vectors, already divided by the 2-D sum (rf only)
};

__global__ void __launch_bounds__(256) gate_apply_kernel(GateParams p) {
  __shared__ float sb[GT_F + 2 * G_MAXH][GT_T + 2 * G_MAXH + 1];  // booleans with halo
  __shared__ float st[GT_F + 2 * G_MAXH][GT_T + 1];               // smoothed along time
  const int tid = threadIdx.x;
  const int row = blockIdx.z, f0 = blockIdx.y * GT_F, t0 = blockIdx.x * GT_T;
  const float2* sp = p.spec + (size_t)row * p.F * (size_t)p.N;
  const float* th = p.thresh + (size_t)(p.nz_rows == 1 ? 0 : row) * p.F;
  const int HF = GT_F + 2 * p.hf, HT = GT_T + 2 * p.ht;
  for (int i = tid; i < HF * HT; i += 256) {
    const int a = i / HT, b = i - a * HT;
    const int f = f0 + a - p.hf, t = t0 + b - p.ht;
    float m = 0.f;  // conv2d zero padding
    if (f >= 0 && f < p.F && t >= 0 && t < p.N) m = (gate_db(sp[(size_t)f * p.N + t]) < __ldg(th + f)) ? 1.f : 0.f;
    sb[a][b] = m;
  }
  __syncthreads();
  for (int i = tid; i < HF * GT_T; i += 256) {
    const int a = i / GT_T, b = i - a * GT_T;
    float acc = 0.f;
    for (int d = 0; d <= 2 * p.ht; ++d) acc = fmaf(p.rt[d], sb[a][b + d], acc);
    st[a][b] = acc;
  }
  __syncthreads();
  const float amt = __ldg(p.amount + row / p.rows_per_item);
  float2* op = p.out + (size_t)row * p.F * (size_t)p.N;
  for (int i = tid; i < GT_F * GT_T; i += 256) {
    const int a = i / GT_T, b = i - a * GT_T;
    const int f = f0 + a, t = t0 + b;
    if (f >= p.F || t >= p.N) continue;
    float acc = 0.f;
    for (int d = 0; d <= 2 * p.hf; ++d) acc = fmaf(p.rf[d], st[a + d][b], acc);
    const float g = 1.0f - acc * amt;
    const float2 z = p.mul[((size_t)row * p.F + f) * (size_t)p.N + t];
    op[(size_t)f * p.N + t] = make_float2(z.x * g, z.y * g);
  }
}

static unsigned grid_for(long long total) {
  long long blocks = (total + 255) / 256;
  const long long cap = (long long)B2A_NUM_SMS * 16;
  return (unsigned)(blocks < cap ? blocks : cap);
}

}  // namespace specmask
}  // namespace b2a

using namespace b2a::specmask;

extern "C" int b2a_spec_band_mask_f32(float* spec, int64_t rows, int F, int N, const float* axis_vals, const float* lo,
                                      const float* hi, int rows_per_item, int axis, float fill_re, float fill_im,
                                      void* stream) {
  B2A_REQUIRE(spec && axis_vals && lo && hi, B2A_E_INVALID, "spec_band_mask: null pointer");
  B2A_REQUIRE(rows >= 1 && F >= 1 && N >= 1 && rows_per_item >= 1 && (axis == 0 || axis == 1), B2A_E_INVALID,
              "spec_band_mask: bad argument");
  B2A_REQUIRE(((uintptr_t)spec & 7) == 0, B2A_E_INVALID, "spec_band_mask: spectra must be 8-byte aligned");
  B2A_REQUIRE(rows * F < (int64_t)2147483647, B2A_E_UNSUPPORTED, "spec_band_mask: too many lines");
  B2A_LAUNCH(band_mask_kernel, dim3((unsigned)(rows * F)), dim3(N >= 256 ? 256 : 64), 0, stream,
             reinterpret_cast<float2*>(spec), F, N, axis_vals, lo, hi, rows_per_item, axis, make_float2(fill_re, fill_im));
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

// the checks and the launch of both out-of-place band-mask passes
static int band_mask_out(bool bwd, const float* g, const float* spec, float* out, int64_t rows, int F, int N,
                         const float* axis_vals, const float* lo, const float* hi, int rows_per_item, int axis,
                         float2 fill, void* stream) {
  B2A_REQUIRE(spec && out && axis_vals && lo && hi && (g || !bwd), B2A_E_INVALID, "spec_band_mask: null pointer");
  B2A_REQUIRE(rows >= 1 && F >= 1 && N >= 1 && rows_per_item >= 1 && (axis == 0 || axis == 1), B2A_E_INVALID,
              "spec_band_mask: bad argument");
  B2A_REQUIRE((((uintptr_t)spec | (uintptr_t)out | (uintptr_t)g) & 7) == 0, B2A_E_INVALID,
              "spec_band_mask: spectra must be 8-byte aligned");
  B2A_REQUIRE(out != spec && out != g, B2A_E_INVALID, "spec_band_mask: the output must not alias an input");
  B2A_REQUIRE(rows * F < (int64_t)2147483647, B2A_E_UNSUPPORTED, "spec_band_mask: too many lines");
  const dim3 grid((unsigned)(rows * F)), block(N >= 256 ? 256 : 64);
  const float2* gp = reinterpret_cast<const float2*>(g);
  const float2* sp = reinterpret_cast<const float2*>(spec);
  float2* op = reinterpret_cast<float2*>(out);
  if (bwd)
    B2A_LAUNCH(band_mask_out_kernel<true>, grid, block, 0, stream, gp, sp, op, F, N, axis_vals, lo, hi, rows_per_item,
               axis, make_float2(0.f, 0.f));
  else
    B2A_LAUNCH(band_mask_out_kernel<false>, grid, block, 0, stream, gp, sp, op, F, N, axis_vals, lo, hi, rows_per_item,
               axis, fill);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" int b2a_spec_band_mask_out_f32(const float* spec, float* out, int64_t rows, int F, int N,
                                          const float* axis_vals, const float* lo, const float* hi, int rows_per_item,
                                          int axis, float fill_re, float fill_im, void* stream) {
  return band_mask_out(false, nullptr, spec, out, rows, F, N, axis_vals, lo, hi, rows_per_item, axis,
                       make_float2(fill_re, fill_im), stream);
}

extern "C" int b2a_spec_band_mask_backward_f32(const float* grad_out, const float* spec, int64_t rows, int F, int N,
                                               const float* axis_vals, const float* lo, const float* hi,
                                               int rows_per_item, int axis, float* grad_spec, void* stream) {
  return band_mask_out(true, grad_out, spec, grad_spec, rows, F, N, axis_vals, lo, hi, rows_per_item, axis,
                       make_float2(0.f, 0.f), stream);
}

extern "C" int b2a_spec_rotate_f32(float* spec, int64_t items, int64_t cells_per_item, const float* shift,
                                   int per_cell, void* stream) {
  B2A_REQUIRE(spec && shift, B2A_E_INVALID, "spec_rotate: null pointer");
  B2A_REQUIRE(items >= 1 && cells_per_item >= 1, B2A_E_INVALID, "spec_rotate: bad argument");
  B2A_REQUIRE(((uintptr_t)spec & 7) == 0, B2A_E_INVALID, "spec_rotate: spectra must be 8-byte aligned");
  const long long total = (long long)items * cells_per_item;
  B2A_LAUNCH(rotate_kernel, dim3(grid_for(total)), dim3(256), 0, stream, reinterpret_cast<float2*>(spec), total,
             (long long)cells_per_item, shift, per_cell ? 1 : 0);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" int b2a_spec_mask_low_f32(float* spec, int64_t items, int64_t cells_per_item, const float* db_cutoff,
                                     float amin_sq, float top_db, float val, void* ws /* >= 4 bytes */, void* stream) {
  B2A_REQUIRE(spec && db_cutoff && ws, B2A_E_INVALID, "spec_mask_low: null pointer");
  B2A_REQUIRE(items >= 1 && cells_per_item >= 1, B2A_E_INVALID, "spec_mask_low: bad argument");
  B2A_REQUIRE(((uintptr_t)spec & 7) == 0 && ((uintptr_t)ws & 3) == 0, B2A_E_INVALID, "spec_mask_low: alignment");
  const long long total = (long long)items * cells_per_item;
#ifdef B2A_SIM
  memset(ws, 0, 4);
#else
  B2A_CUDA_OK(cudaMemsetAsync(ws, 0, 4, (cudaStream_t)stream));
#endif
  B2A_LAUNCH(maxpow_kernel, dim3(grid_for(total)), dim3(256), 0, stream, reinterpret_cast<const float2*>(spec), total,
             (unsigned*)ws);
  B2A_LAUNCH(mask_low_kernel, dim3(grid_for(total)), dim3(256), 0, stream, reinterpret_cast<float2*>(spec), total,
             (long long)cells_per_item, db_cutoff, (const unsigned*)ws, amin_sq, top_db, val);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" int b2a_spec_mask_low_out_f32(const float* spec, float* out, int64_t items, int64_t cells_per_item,
                                         const float* db_cutoff, float amin_sq, float top_db, float val,
                                         void* ws /* >= 4 bytes, kept for the backward */, void* stream) {
  B2A_REQUIRE(spec && out && db_cutoff && ws, B2A_E_INVALID, "spec_mask_low_out: null pointer");
  B2A_REQUIRE(items >= 1 && cells_per_item >= 1, B2A_E_INVALID, "spec_mask_low_out: bad argument");
  B2A_REQUIRE((((uintptr_t)spec | (uintptr_t)out) & 7) == 0 && ((uintptr_t)ws & 3) == 0, B2A_E_INVALID,
              "spec_mask_low_out: alignment");
  B2A_REQUIRE(out != spec, B2A_E_INVALID, "spec_mask_low_out: out must not alias spec");
  const long long total = (long long)items * cells_per_item;
#ifdef B2A_SIM
  memset(ws, 0, 4);
#else
  B2A_CUDA_OK(cudaMemsetAsync(ws, 0, 4, (cudaStream_t)stream));
#endif
  B2A_LAUNCH(maxpow_kernel, dim3(grid_for(total)), dim3(256), 0, stream, reinterpret_cast<const float2*>(spec), total,
             (unsigned*)ws);
  B2A_LAUNCH(mask_low_out_kernel, dim3(grid_for(total)), dim3(256), 0, stream, reinterpret_cast<const float2*>(spec),
             reinterpret_cast<float2*>(out), total, (long long)cells_per_item, db_cutoff, (const unsigned*)ws, amin_sq,
             top_db, val);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" int b2a_spec_mask_low_backward_f32(const float* grad_out, const float* spec, int64_t items,
                                              int64_t cells_per_item, const float* db_cutoff, float amin_sq,
                                              float top_db, float val, const void* ws, float* grad_spec, void* stream) {
  B2A_REQUIRE(grad_out && spec && db_cutoff && ws && grad_spec, B2A_E_INVALID, "spec_mask_low_backward: null pointer");
  B2A_REQUIRE(items >= 1 && cells_per_item >= 1, B2A_E_INVALID, "spec_mask_low_backward: bad argument");
  B2A_REQUIRE((((uintptr_t)grad_out | (uintptr_t)spec | (uintptr_t)grad_spec) & 7) == 0 && ((uintptr_t)ws & 3) == 0,
              B2A_E_INVALID, "spec_mask_low_backward: alignment");
  const long long total = (long long)items * cells_per_item;
  B2A_LAUNCH(mask_low_bwd_kernel, dim3(grid_for(total)), dim3(256), 0, stream,
             reinterpret_cast<const float2*>(grad_out), reinterpret_cast<const float2*>(spec),
             reinterpret_cast<float2*>(grad_spec), total, (long long)cells_per_item, db_cutoff,
             (const unsigned*)ws, amin_sq, top_db, val);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

// gate_apply_kernel over (spec, mul) -> out with thresholds `thresh` [nz_rows, F]
static int gate_apply(const float2* spec, const float2* mul, float2* out, int64_t rows, int F, int64_t N,
                      const float* thresh, int64_t nz_rows, const float* amount, int rows_per_item,
                      const float* smooth_f_h, int n_f, const float* smooth_t_h, int n_t, void* stream) {
  GateParams p;
  memset(&p, 0, sizeof(p));
  p.spec = spec; p.mul = mul; p.out = out; p.thresh = thresh;
  p.amount = amount; p.F = F; p.N = (int)N; p.rows_per_item = rows_per_item; p.nz_rows = (int)nz_rows;
  p.hf = n_f / 2; p.ht = n_t / 2;
  double sum_f = 0, sum_t = 0;
  for (int i = 0; i < n_f; ++i) sum_f += smooth_f_h[i];
  for (int i = 0; i < n_t; ++i) sum_t += smooth_t_h[i];
  B2A_REQUIRE(sum_f * sum_t != 0.0, B2A_E_INVALID, "spec_gate: smoothing kernel sums to zero");
  for (int i = 0; i < n_f; ++i) p.rf[i] = (float)(smooth_f_h[i] / (sum_f * sum_t));
  for (int i = 0; i < n_t; ++i) p.rt[i] = smooth_t_h[i];
  B2A_LAUNCH(gate_apply_kernel, dim3((unsigned)((N + GT_T - 1) / GT_T), (unsigned)((F + GT_F - 1) / GT_F), (unsigned)rows),
             dim3(256), 0, stream, p);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

// the shape checks both gate entry points share
#define GATE_REQUIRE_SHAPE(what)                                                                                       \
  B2A_REQUIRE(rows >= 1 && rows <= 65535 && F >= 1 && N >= 1 && rows_per_item >= 1, B2A_E_INVALID,                     \
              what ": bad shape");                                                                                     \
  B2A_REQUIRE(nz_rows == 1 || nz_rows == rows, B2A_E_INVALID, what ": noise rows (%lld) must be 1 or %lld",            \
              (long long)nz_rows, (long long)rows);                                                                    \
  B2A_REQUIRE((n_f & 1) && (n_t & 1) && n_f <= 2 * G_MAXH + 1 && n_t <= 2 * G_MAXH + 1, B2A_E_UNSUPPORTED,            \
              what ": smoothing vectors must have odd lengths <= %d (got %d, %d)", 2 * G_MAXH + 1, n_f, n_t);          \
  B2A_REQUIRE(nz_rows * F < (int64_t)2147483647 && (F + GT_F - 1) / GT_F <= 65535, B2A_E_UNSUPPORTED, what ": too large")

extern "C" int b2a_spec_gate_f32(const float* spec, int64_t rows, int F, int64_t N, const float* nz_spec, int64_t nz_rows,
                                 int64_t nz_N, float n_std, const float* amount, int rows_per_item,
                                 const float* smooth_f_h, int n_f, const float* smooth_t_h, int n_t, float* out,
                                 void* ws, void* stream) {
  B2A_REQUIRE(spec && nz_spec && amount && smooth_f_h && smooth_t_h && out && ws, B2A_E_INVALID, "spec_gate: null pointer");
  B2A_REQUIRE(nz_N >= 1, B2A_E_INVALID, "spec_gate: bad shape");
  GATE_REQUIRE_SHAPE("spec_gate");
  B2A_REQUIRE(out != spec, B2A_E_INVALID, "spec_gate: out must not alias spec");
  B2A_REQUIRE((((uintptr_t)spec | (uintptr_t)nz_spec | (uintptr_t)out) & 7) == 0, B2A_E_INVALID, "spec_gate: alignment");
  float* thresh = reinterpret_cast<float*>(ws);  // [nz_rows, F]
  B2A_LAUNCH(gate_stats_kernel, dim3((unsigned)((nz_rows * F + 7) / 8)), dim3(256), 0, stream,
             reinterpret_cast<const float2*>(nz_spec), (int)(nz_rows * F), (int)nz_N, n_std, thresh);
  return gate_apply(reinterpret_cast<const float2*>(spec), reinterpret_cast<const float2*>(spec),
                    reinterpret_cast<float2*>(out), rows, F, N, thresh, nz_rows, amount, rows_per_item, smooth_f_h, n_f,
                    smooth_t_h, n_t, stream);
}

extern "C" int b2a_spec_gate_backward_f32(const float* grad_out, const float* spec, int64_t rows, int F, int64_t N,
                                          const float* thresh, int64_t nz_rows, const float* amount, int rows_per_item,
                                          const float* smooth_f_h, int n_f, const float* smooth_t_h, int n_t,
                                          float* grad_spec, void* stream) {
  B2A_REQUIRE(grad_out && spec && thresh && amount && smooth_f_h && smooth_t_h && grad_spec, B2A_E_INVALID,
              "spec_gate_backward: null pointer");
  GATE_REQUIRE_SHAPE("spec_gate_backward");
  B2A_REQUIRE(grad_spec != spec, B2A_E_INVALID, "spec_gate_backward: grad_spec must not alias spec");
  B2A_REQUIRE((((uintptr_t)grad_out | (uintptr_t)spec | (uintptr_t)grad_spec) & 7) == 0, B2A_E_INVALID,
              "spec_gate_backward: alignment");
  return gate_apply(reinterpret_cast<const float2*>(spec), reinterpret_cast<const float2*>(grad_out),
                    reinterpret_cast<float2*>(grad_spec), rows, F, N, thresh, nz_rows, amount, rows_per_item,
                    smooth_f_h, n_f, smooth_t_h, n_t, stream);
}
