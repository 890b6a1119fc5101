// effects.cu -- the element-wise / per-row-peak effects of EffectMixin on sm_90a (SURVEY.md 8f.2): each is ONE pass
// over the waveform (HBM-bound: read x once, write y once) instead of the reference's chain of tensor temporaries.
//
//   b2a_row_absmax_f32   peak[row] = max |x|                      ref:audiotools/core/effects.py:194 (ensure_max_of_audio),
//                                                                  :155,:176 (apply_ir peak restore), :639 (alter_drr)
//   b2a_limit_peak_f32   y = x * (peak > max ? max / peak : 1)    ref :181-198
//   b2a_mix_f32          y = x + g[item] * other                  ref :27-64 (the normalize() multiply of `other` and the add)
//   b2a_quantize_f32     linear / mu-law quantisation             ref :463-523 (same float32 operation order, incl. the
//                                                                  `x - (x - q)` straight-through residual)
//   b2a_order_stats_f32  k-th smallest values of one row           ref :452-453 (torch.quantile's sorted gather), by
//                        (exact: 4-pass radix select)               radix selection instead of a full sort
//   b2a_clamp_items_f32  y = min(max(x, lo[item]), hi[item])       ref :459
//   b2a_gain_f32         y = g[item] * x                          ref :219, :237 (normalize / volume_change)
#include "b2a_common.h"

namespace b2a {
namespace effects {

constexpr int TPB = 256;

// The walk of every element-wise kernel over its row (grid.y) of n floats, grid-stride: vec4(i) for the float4 at each
// i = 0, 4, 8, ... when vec_ok (n % 4 == 0 and the row's pointers 16-byte aligned), else one(i) for every element.
template <class V4, class V1>
__device__ __forceinline__ void walk(int64_t n, int vec_ok, V4 vec4, V1 one) {
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nt = (int64_t)gridDim.x * blockDim.x;
  if (vec_ok) {
    for (int64_t i = gid; i < n >> 2; i += nt) vec4(4 * i);
  } else {
    for (int64_t i = gid; i < n; i += nt) one(i);
  }
}

// y = f(x) over one row, streamed
template <class F>
__device__ __forceinline__ void map_row(const float* __restrict__ x, float* __restrict__ y, int64_t n, int vec_ok, F f) {
  walk(n, vec_ok,
       [&](int64_t i) {
         float4 v = ld_stream4(x + i);
         v.x = f(v.x); v.y = f(v.y); v.z = f(v.z); v.w = f(v.w);
         st_stream4(y + i, v);
       },
       [&](int64_t i) { y[i] = f(x[i]); });
}

// peak must be zeroed by the caller (memset inside the entry point).  |x| >= 0, so its float bits order like unsigned
// ints, and every NaN pattern of |x| ranks above +inf's 0x7f800000: a NaN anywhere in the row is its peak, as in the
// reference's x.abs().max(dim=-1) (fmaxf would drop it)
__device__ __forceinline__ unsigned abs_bits(float v) { return __float_as_uint(v) & 0x7fffffffu; }
__global__ void __launch_bounds__(TPB) absmax_kernel(const float* __restrict__ x, int64_t T, int vec_ok,
                                                     float* __restrict__ peak) {
  const int row = blockIdx.y;
  const float* xr = x + (size_t)row * (size_t)T;
  unsigned m = 0u;
  walk(T, vec_ok,
       [&](int64_t i) {
         const float4 v = ld_stream4(xr + i);
         m = max(max(m, max(abs_bits(v.x), abs_bits(v.y))), max(abs_bits(v.z), abs_bits(v.w)));
       },
       [&](int64_t i) { m = max(m, abs_bits(xr[i])); });
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ unsigned s[TPB / 32];
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < TPB / 32; ++w) m = max(m, s[w]);
    atomicMax(reinterpret_cast<unsigned*>(peak + row), m);
  }
}

// x.clamp(lo, hi) as torch computes it with tensor bounds: a NaN sample or a NaN bound gives NaN (fminf / fmaxf alone
// would return the other operand)
__device__ __forceinline__ float clamp_nan(float v, float lo, float hi) {
  const float r = fminf(fmaxf(v, lo), hi);
  return (v != v || lo != lo || hi != hi) ? v + lo + hi : r;
}

// MODE 0: limit peak (scale = peak > lim ? lim / peak : 1)   MODE 1: clamp to [lo, hi] of the item
template <int MODE>
__global__ void __launch_bounds__(TPB) rows_kernel(const float* __restrict__ x, float* __restrict__ out, int64_t T,
                                                   int vec_ok, const float* __restrict__ a, const float* __restrict__ b,
                                                   float lim) {
  const int row = blockIdx.y;
  const float* xr = x + (size_t)row * (size_t)T;
  float* yr = out + (size_t)row * (size_t)T;
  float p0, p1 = 0.f;
  if (MODE == 0) {
    const float pk = __ldg(a + row);
    p0 = pk > lim ? lim / pk : 1.0f;
  } else {
    p0 = __ldg(a + row); p1 = __ldg(b + row);
  }
  map_row(xr, yr, T, vec_ok, [&](float v) { return MODE == 0 ? v * p0 : clamp_nan(v, p0, p1); });
}

__global__ void __launch_bounds__(TPB) gain_kernel(const float* __restrict__ x, float* __restrict__ out,
                                                   int64_t per_item, int vec_ok, const float* __restrict__ gain) {
  const int b = blockIdx.y;
  const float g = __ldg(gain + b);
  map_row(x + (size_t)b * per_item, out + (size_t)b * per_item, per_item, vec_ok, [&](float v) { return v * g; });
}

__global__ void __launch_bounds__(TPB) mix_kernel(const float* __restrict__ x, const float* __restrict__ other,
                                                  const float* __restrict__ gain, float* __restrict__ out,
                                                  int64_t per_item, int vec_ok) {
  const int b = blockIdx.y;
  const float g = gain ? __ldg(gain + b) : 1.0f;
  const float* xr = x + (size_t)b * per_item;
  const float* orow = other + (size_t)b * per_item;
  float* yr = out + (size_t)b * per_item;
  // the reference multiplies first (normalize) and adds afterwards: two roundings, not one fused multiply-add
  auto f = [&](float a, float o) { return __fadd_rn(a, __fmul_rn(o, g)); };
  walk(per_item, vec_ok,
       [&](int64_t i) {
         const float4 a = ld_stream4(xr + i), o = ld_stream4(orow + i);
         st_stream4(yr + i, make_float4(f(a.x, o.x), f(a.y, o.y), f(a.z, o.z), f(a.w, o.w)));
       },
       [&](int64_t i) { yr[i] = f(xr[i], orow[i]); });
}

// ref:audiotools/core/effects.py:481-491 (linear) and :509-523 (mu-law), operation by operation in float32
__device__ __forceinline__ float quant_linear(float a, float q) {
  float x = __fdiv_rn(__fadd_rn(a, 1.0f), 2.0f);
  x = floorf(__fmul_rn(x, q));
  x = __fdiv_rn(x, q);
  x = __fadd_rn(__fmul_rn(2.0f, x), -1.0f);
  const float residual = __fadd_rn(a, -x);
  return __fadd_rn(a, -residual);
}
__device__ __forceinline__ float quant_mulaw(float a, float mu, float l1p) {
  const float sg = (a > 0.f) ? 1.f : ((a < 0.f) ? -1.f : 0.f);
  float x = __fdiv_rn(__fmul_rn(sg, log1pf(__fmul_rn(mu, fabsf(a)))), l1p);
  x = __fadd_rn(__fmul_rn(__fdiv_rn(__fadd_rn(x, 1.0f), 2.0f), mu), 0.5f);
  const float xi = (float)(long long)x;  // .to(torch.int64): truncation toward zero, then int / float
  x = __fadd_rn(__fmul_rn(__fdiv_rn(xi, mu), 2.0f), -1.0f);
  const float sx = (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f);
  x = __fdiv_rn(__fmul_rn(sx, __fadd_rn(expf(__fmul_rn(fabsf(x), l1p)), -1.0f)), mu);
  const float residual = __fadd_rn(a, -x);
  return __fadd_rn(a, -residual);
}

__global__ void __launch_bounds__(TPB) quantize_kernel(const float* __restrict__ x, float* __restrict__ out,
                                                       int64_t per_item, int vec_ok,
                                                       const float* __restrict__ channels, int mulaw) {
  const int b = blockIdx.y;
  const float q = __ldg(channels + b);
  const float mu = __fadd_rn(q, -1.0f), l1p = log1pf(mu);
  const float* xr = x + (size_t)b * per_item;
  float* yr = out + (size_t)b * per_item;
  map_row(xr, yr, per_item, vec_ok, [&](float v) { return mulaw ? quant_mulaw(v, mu, l1p) : quant_linear(v, q); });
}

// ---- exact k-th smallest by 4-pass (8 bits each) radix selection: one CTA per requested order statistic.  Every NaN,
// of either sign, gets the largest key, so NaNs rank above +inf as in torch.sort, and a NaN statistic comes back as the
// positive quiet NaN 0x7fffffff (ord_key alone would rank a NaN with the sign bit set below -inf).  -0 ranks before +0.
constexpr int ST = 1024;
__device__ __forceinline__ unsigned stat_key(float v) { return v != v ? 0xffffffffu : ord_key(v); }
__global__ void __launch_bounds__(ST) order_stat_kernel(const float* __restrict__ row, int64_t T,
                                                        const int64_t* __restrict__ ks, float* __restrict__ out) {
  __shared__ unsigned hist[256];
  __shared__ unsigned s_prefix;
  __shared__ long long s_k;
  const int tid = threadIdx.x;
  long long k = ks[blockIdx.x];
  if (k < 0) k = 0;
  if (k > T - 1) k = T - 1;
  unsigned prefix = 0, mask = 0;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    for (int i = tid; i < 256; i += ST) hist[i] = 0;
    __syncthreads();
    for (int64_t i = tid; i < T; i += ST) {
      const unsigned key = stat_key(__ldg(row + i));
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 0xff], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      long long c = 0;
      int bsel = 255;
      for (int bkt = 0; bkt < 256; ++bkt) {
        if (c + (long long)hist[bkt] > k) { bsel = bkt; break; }
        c += hist[bkt];
      }
      s_prefix = prefix | ((unsigned)bsel << shift);
      s_k = k - c;
    }
    __syncthreads();
    prefix = s_prefix;
    k = s_k;
    mask |= 0xffu << shift;
  }
  if (tid == 0) out[blockIdx.x] = ord_val(prefix);
}

// The checks and the launch of an element-wise kernel over `rows` rows of n floats: grid.y = row (so at most 65535
// rows), grid.x ~8 resident CTAs per SM across the rows, grid-stride inside.  vec_ok: n % 4 == 0 and `ptrs`, the OR of
// the row pointers, 16-byte aligned.
struct RowsLaunch {
  dim3 grid;
  int vec_ok;
};
static int rows_launch(const char* op, bool non_null, int64_t rows, int64_t n, uintptr_t ptrs, RowsLaunch* l) {
  B2A_REQUIRE(non_null, B2A_E_INVALID, "%s: null pointer", op);
  B2A_REQUIRE(rows >= 1 && rows <= 65535 && n >= 1, B2A_E_INVALID, "%s: bad shape", op);
  l->vec_ok = ptrs % 16 == 0 && n % 4 == 0;
  const int64_t want = ((l->vec_ok ? n / 4 : n) + TPB - 1) / TPB, cap = (int64_t)B2A_NUM_SMS * 8 / rows + 1;
  l->grid = dim3((unsigned)(want < cap ? want : cap), (unsigned)rows);
  return B2A_OK;
}

}  // namespace effects

namespace effects {
// ---------------------------------------------------------------------------------------------
// ImpulseResponseMixin.alter_drr (ref:audiotools/core/effects.py:540-647), one CTA per impulse-response row, one launch:
//   td = argmax(x), early = [td - t0, td + t0], window = the early region of the item's CHANNEL 0 (hann(1) == 1, so the
//   reference's window is that indicator), alpha from the quadratic of solve_alpha (:594-617, float32 like the
//   reference; with an indicator window b == 0), floored at max|late| / max|early|, out = alpha on (early AND window),
//   x elsewhere, then ensure_max_of_audio (:181-198).  The reference runs ~25 tensor passes for this.
// ---------------------------------------------------------------------------------------------
constexpr int DRR_T = 512;

// torch.argmax's order: NaN above every number, then the larger value, then the smaller index
struct ArgMax { float v; int i; };
__device__ __forceinline__ ArgMax better(ArgMax a, ArgMax b) {
  const bool an = a.v != a.v, bn = b.v != b.v;
  if (an || bn) return (bn && (!an || b.i < a.i)) ? b : a;
  return (b.v > a.v || (b.v == a.v && b.i < a.i)) ? b : a;
}
// T <= INT_MAX - DRR_T (checked by the entry point), so i += DRR_T cannot overflow
__device__ ArgMax block_argmax(const float* __restrict__ x, int T, ArgMax* sm) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  ArgMax m{-INFINITY, 0x7fffffff};
  for (int i = tid; i < T; i += DRR_T) {
    const float v = x[i];
    if (v > m.v || (v != v && m.v == m.v)) { m.v = v; m.i = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ArgMax t{__shfl_xor_sync(0xffffffffu, m.v, o), __shfl_xor_sync(0xffffffffu, m.i, o)};
    m = better(m, t);
  }
  __syncthreads();
  if (lane == 0) sm[warp] = m;
  __syncthreads();
  ArgMax r = sm[0];
  for (int w = 1; w < DRR_T / 32; ++w) r = better(r, sm[w]);
  if (r.i == 0x7fffffff) r.i = 0;
  return r;
}
__device__ float block_sum_f(float v, float* sm) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) sm[warp] = v;
  __syncthreads();
  float r = 0.f;
  for (int w = 0; w < DRR_T / 32; ++w) r += sm[w];
  return r;
}
__device__ float block_max_f(float v, float* sm) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) sm[warp] = v;
  __syncthreads();
  float r = sm[0];
  for (int w = 1; w < DRR_T / 32; ++w) r = fmaxf(r, sm[w]);
  return r;
}

__global__ void __launch_bounds__(DRR_T)
alter_drr_kernel(const float* __restrict__ x, float* __restrict__ out, int T, int C, int t0, const float* __restrict__ drr,
                 float max_abs) {
  __shared__ ArgMax s_am[DRR_T / 32];
  __shared__ float s_f[DRR_T / 32];
  const int row = blockIdx.x, item = row / C, tid = threadIdx.x;
  const float* xr = x + (size_t)row * T;
  const float* x0 = x + (size_t)item * C * T;  // channel 0 of the item: its early region is the window
  const int td = block_argmax(xr, T, s_am).i;
  const int tw = (C == 1 || row == item * C) ? td : block_argmax(x0, T, s_am).i;
  float a = 0.f, ce = 0.f, lsq = 0.f, ml = 0.f, me = 0.f, mew = 0.f, meo = 0.f;
  for (int i = tid; i < T; i += DRR_T) {
    const float v = xr[i], av = fabsf(v);
    const bool e = (i >= td - t0) && (i <= td + t0), w = (i >= tw - t0) && (i <= tw + t0);
    if (e) {
      me = fmaxf(me, av);
      if (w) { a = fmaf(v, v, a); mew = fmaxf(mew, av); }
      else { ce = fmaf(v, v, ce); meo = fmaxf(meo, av); }
    } else {
      lsq = fmaf(v, v, lsq);
      ml = fmaxf(ml, av);
    }
  }
  a = block_sum_f(a, s_f); ce = block_sum_f(ce, s_f); lsq = block_sum_f(lsq, s_f);
  ml = block_max_f(ml, s_f); me = block_max_f(me, s_f); mew = block_max_f(mew, s_f); meo = block_max_f(meo, s_f);
  // solve_alpha with an indicator window: b = 0, c = sum_{early, outside the window} x^2 - 10^(drr/10) sum_late x^2
  const float c = ce - powf(10.0f, __ldg(drr + item) / 10.0f) * lsq;
  const float b = 0.f;
  const float expr = sqrtf(b * b - 4.0f * a * c);
  const float r1 = (-b - expr) / (2.0f * a), r2 = (-b + expr) / (2.0f * a);
  float alpha = (r1 != r1 || r2 != r2) ? NAN : fmaxf(r1, r2);  // torch.maximum propagates nan
  const float min_alpha = ml / me;
  alpha = (alpha != alpha || min_alpha != min_alpha) ? NAN : fmaxf(alpha, min_alpha);
  // ensure_max_of_audio on the altered response.  A non-finite alpha (a = 0: the row's early region does not meet
  // the window, e.g. a second channel whose direct path lies > 2.5 ms from channel 0's) makes the reference's
  // `alpha * window * early` NaN on the WHOLE row (NaN * 0), its peak NaN and its peak gain 1: same here.
  const bool finite = (alpha - alpha) == 0.0f;
  const float peak = fmaxf(fmaxf(fabsf(alpha) * mew, meo), ml);
  const float pg = (finite && peak > max_abs) ? max_abs / peak : 1.0f;
  float* o = out + (size_t)row * T;
  for (int i = tid; i < T; i += DRR_T) {
    const float v = xr[i];
    const bool e = (i >= td - t0) && (i <= td + t0), w = (i >= tw - t0) && (i <= tw + t0);
    const float wf = w ? 1.0f : 0.0f, ev = e ? v : 0.0f, lv = e ? 0.0f : v;
    o[i] = (alpha * wf * ev + (1.0f - wf) * ev + lv) * pg;  // the reference's expression, term by term (:642)
  }
}

}  // namespace effects
}  // namespace b2a

using namespace b2a::effects;

extern "C" int b2a_row_absmax_f32(const float* x, int64_t rows, int64_t T, float* peak, void* stream) {
  RowsLaunch l;
  const int rc = rows_launch("row_absmax", x && peak, rows, T, (uintptr_t)x, &l);
  if (rc != B2A_OK) return rc;
  B2A_CUDA_OK(cudaMemsetAsync(peak, 0, (size_t)rows * sizeof(float), (cudaStream_t)stream));
  B2A_LAUNCH(absmax_kernel, l.grid, dim3(TPB), 0, stream, x, T, l.vec_ok, peak);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" int b2a_limit_peak_f32(const float* x, float* out, int64_t rows, int64_t T, const float* peak, float max_abs,
                                  void* stream) {
  RowsLaunch l;
  const int rc = rows_launch("limit_peak", x && out && peak, rows, T, (uintptr_t)x | (uintptr_t)out, &l);
  if (rc != B2A_OK) return rc;
  B2A_LAUNCH(rows_kernel<0>, l.grid, dim3(TPB), 0, stream, x, out, T, l.vec_ok, peak, (const float*)nullptr, max_abs);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" int b2a_clamp_items_f32(const float* x, float* out, int64_t B, int64_t per_item, const float* lo,
                                   const float* hi, void* stream) {
  RowsLaunch l;
  const int rc = rows_launch("clamp_items", x && out && lo && hi, B, per_item, (uintptr_t)x | (uintptr_t)out, &l);
  if (rc != B2A_OK) return rc;
  B2A_LAUNCH(rows_kernel<1>, l.grid, dim3(TPB), 0, stream, x, out, per_item, l.vec_ok, lo, hi, 0.f);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" int b2a_gain_f32(const float* x, float* out, int64_t B, int64_t per_item, const float* gain, void* stream) {
  RowsLaunch l;
  const int rc = rows_launch("gain", x && out && gain, B, per_item, (uintptr_t)x | (uintptr_t)out, &l);
  if (rc != B2A_OK) return rc;
  B2A_LAUNCH(gain_kernel, l.grid, dim3(TPB), 0, stream, x, out, per_item, l.vec_ok, gain);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" int b2a_mix_f32(const float* x, const float* other, const float* other_gain, float* out, int64_t B,
                           int64_t per_item, void* stream) {
  RowsLaunch l;
  const int rc = rows_launch("mix", x && other && out, B, per_item, (uintptr_t)x | (uintptr_t)other | (uintptr_t)out, &l);
  if (rc != B2A_OK) return rc;
  B2A_LAUNCH(mix_kernel, l.grid, dim3(TPB), 0, stream, x, other, other_gain, out, per_item, l.vec_ok);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" int b2a_quantize_f32(const float* x, float* out, int64_t B, int64_t per_item, const float* channels, int mulaw,
                                void* stream) {
  RowsLaunch l;
  const int rc = rows_launch("quantize", x && out && channels, B, per_item, (uintptr_t)x | (uintptr_t)out, &l);
  if (rc != B2A_OK) return rc;
  B2A_LAUNCH(quantize_kernel, l.grid, dim3(TPB), 0, stream, x, out, per_item, l.vec_ok, channels, mulaw ? 1 : 0);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" int b2a_order_stats_f32(const float* row, int64_t T, const int64_t* k, int nk, float* out, void* stream) {
  B2A_REQUIRE(row && k && out, B2A_E_INVALID, "order_stats: null pointer");
  B2A_REQUIRE(T >= 1 && nk >= 1 && nk <= 65535, B2A_E_INVALID, "order_stats: bad shape");
  B2A_LAUNCH(order_stat_kernel, dim3((unsigned)nk), dim3(ST), 0, stream, row, T, k, out);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" int b2a_alter_drr_f32(const float* ir, float* out, int64_t rows, int64_t T, int C, int t0, const float* drr,
                                 float max_abs, void* stream) {
  B2A_REQUIRE(ir && out && drr, B2A_E_INVALID, "alter_drr: null pointer");
  // the kernel's int sample index steps by DRR_T and reaches td + t0: both must stay below INT_MAX
  B2A_REQUIRE(rows >= 1 && T >= 1 && T <= INT_MAX - DRR_T && C >= 1 && rows % C == 0 && t0 >= 0 &&
                  (int64_t)t0 <= INT_MAX - T,
              B2A_E_INVALID, "alter_drr: bad shape");
  B2A_REQUIRE(out != ir, B2A_E_INVALID, "alter_drr: out must not alias ir");
  B2A_LAUNCH(alter_drr_kernel, dim3((unsigned)rows), dim3(DRR_T), 0, stream, ir, out, (int)T, C, t0, drr, max_abs);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

/* Backward of the per-row peak rescales (ensure_max_of_audio; apply_ir's peak restore), one CTA per row.
 * Pass 1 finds the first arg-max of |y| (and of |x_ref|) and dot(g, y) with a fixed-order reduction; pass 2 writes
 * the scaled gradient, then one thread adds the single-sample corrections (torch's max(dim) backward: the gradient
 * of the peak goes to the index max returns; the first one here, as for ties torch documents).
 *   limit   (x_ref == NULL):  y' = y p,  p = max/peak if peak > max else 1
 *           gy = p g - [peak > max] (max / peak^2) dot(g, y) sign(y_b) e_b
 *   restore (x_ref != NULL):  y' = y S,  S = clamp(Mx, 1e-8) / clamp(My, 1e-8),  Mx = max|x_ref|, My = max|y|
 *           gy = S g - [My >= 1e-8] S dot(g, y) / My sign(y_b) e_b
 *           gx_ref = [Mx >= 1e-8] dot(g, y) / clamp(My, 1e-8) sign(x_a) e_a   (zero elsewhere)
 *   bypass[row] != 0 (restore only): S = 1, gy = g, gx_ref = 0. */
namespace b2a {
namespace effects {

// The arg-max of |v| ranks the bits of |v| as unsigned ints, as absmax_kernel does: a NaN ranks above every number, as
// in torch.max(dim).  Ties (equal bits) go to the smaller index.
__device__ __forceinline__ void arg_better(unsigned& v, int& i, unsigned ov, int oi) {
  if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
}
__device__ __forceinline__ float sgn(float v) { return v > 0.f ? 1.f : (v < 0.f ? -1.f : 0.f); }
// clamp(v, 1e-8) as torch computes it: NaN stays NaN (fmaxf alone would return 1e-8)
__device__ __forceinline__ float clamp_peak(float v) { return v != v ? v : fmaxf(v, 1e-8f); }

__global__ void __launch_bounds__(TPB) peak_scale_bwd_kernel(const float* __restrict__ g, const float* __restrict__ y,
                                                             const float* __restrict__ xr_, int64_t T, float lim,
                                                             const int32_t* __restrict__ bypass, float* __restrict__ gy,
                                                             float* __restrict__ gxr) {
  __shared__ unsigned sv[TPB], sx[TPB];
  __shared__ float sd[TPB];
  __shared__ int si[TPB], sxi[TPB];
  const int row = blockIdx.x, tid = threadIdx.x;
  const float* gr = g + (size_t)row * T;
  const float* yr = y + (size_t)row * T;
  const float* xr = xr_ ? xr_ + (size_t)row * T : nullptr;
  unsigned bv = 0u, bx = 0u;
  float d = 0.f;
  int bi = 0x7fffffff, bxi = 0x7fffffff;
  for (int64_t i = tid; i < T; i += TPB) {
    const float v = yr[i];
    const unsigned av = abs_bits(v);
    if (av > bv || bi == 0x7fffffff) { bv = av; bi = (int)i; }
    d = fmaf(gr[i], v, d);
    if (xr) {
      const unsigned a = abs_bits(xr[i]);
      if (a > bx || bxi == 0x7fffffff) { bx = a; bxi = (int)i; }
    }
  }
  sv[tid] = bv; si[tid] = bi; sx[tid] = bx; sxi[tid] = bxi; sd[tid] = d;
  __syncthreads();
  for (int h = TPB / 2; h > 0; h >>= 1) {
    if (tid < h) {
      arg_better(sv[tid], si[tid], sv[tid + h], si[tid + h]);
      arg_better(sx[tid], sxi[tid], sx[tid + h], sxi[tid + h]);
      sd[tid] += sd[tid + h];
    }
    __syncthreads();
  }
  // A NaN peak: limit mode keeps the gain 1 (NaN > lim is false), as the reference's ensure_max_of_audio does; the
  // restore's clamp keeps it, so S and the whole row's gradient are NaN, as in the reference
  const float My = __uint_as_float(sv[0]), Mx = __uint_as_float(sx[0]), dot = sd[0];
  const int b = si[0];
  const bool byp = bypass && bypass[row];
  float S, cb = 0.f;
  if (!xr) {
    S = My > lim ? lim / My : 1.0f;
    if (My > lim) cb = -(lim / (My * My)) * dot * sgn(yr[b]);
  } else if (byp) {
    S = 1.0f;
  } else {
    S = clamp_peak(Mx) / clamp_peak(My);
    if (My >= 1e-8f) cb = -S * dot / My * sgn(yr[b]);
  }
  float* gyr = gy + (size_t)row * T;
  float* gxo = xr ? gxr + (size_t)row * T : nullptr;
  for (int64_t i = tid; i < T; i += TPB) {
    gyr[i] = S * gr[i];
    if (gxo) gxo[i] = 0.f;
  }
  __syncthreads();
  if (tid == 0) {
    gyr[b] = S * gr[b] + cb;
    if (gxo && !byp && Mx >= 1e-8f) gxo[sxi[0]] = dot / clamp_peak(My) * sgn(xr[sxi[0]]);
  }
}

}  // namespace effects
}  // namespace b2a

extern "C" int b2a_peak_scale_backward_f32(const float* grad_out, const float* y, const float* x_ref, int64_t rows,
                                           int64_t T, float max_abs, const int32_t* bypass, float* grad_y,
                                           float* grad_x_ref, void* stream) {
  B2A_REQUIRE(grad_out && y && grad_y, B2A_E_INVALID, "peak_scale_backward: null pointer");
  B2A_REQUIRE(!x_ref || grad_x_ref, B2A_E_INVALID, "peak_scale_backward: x_ref needs grad_x_ref");
  B2A_REQUIRE(rows >= 1 && rows < ((int64_t)1 << 31) && T >= 1 && T < ((int64_t)1 << 31), B2A_E_INVALID,
              "peak_scale_backward: bad shape");
  B2A_REQUIRE(grad_y != grad_out && grad_y != y, B2A_E_INVALID, "peak_scale_backward: grad_y must not alias its inputs");
  B2A_LAUNCH(peak_scale_bwd_kernel, dim3((unsigned)rows), dim3(TPB), 0, stream, grad_out, y, x_ref, T, max_abs, bypass,
             grad_y, grad_x_ref);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}
