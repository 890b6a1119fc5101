// loss.cu -- the reference's spectral L1 losses and their gradient in one pass over the two waveforms, on sm_90a.
//
// MultiScaleSTFTLoss and MelSpectrogramLoss with loss_fn = nn.L1Loss() (ref:audiotools/metrics/spectral.py:70-95,
// 159-192), one scale per launch:
//   STFT:  L = lw mean_{k,n} |lg(|X|) - lg(|Y|)| + mw mean_{k,n} ||X| - |Y||
//   mel:   L = lw mean_{m,n} |lg(mel_x) - lg(mel_y)| + mw mean_{m,n} |mel_x - mel_y|,   mel = fb |.|
//   with lg(v) = log10(max(v, eps)^pow).
// Every term is local to one frame, so the tile that computes a frame's terms also knows their derivative: dL/dX of the
// estimate's bins is written by the forward, and the backward is only the STFT adjoint (b2a_stft_backward_f32).  The
// derivatives are torch's: sign(a - b) with sign(0) = 0 (abs), the gradient passes clamp_min where v >= eps,
// pow(p).log10() gives p / (v ln10), |X| gives X / |X| (0 at X = 0), the mean's 1 / numel is folded in.
//
// Layout: the warp-per-frame FFT of spectral.cu (WPlan, warp_fft, the fused untangle), persistent CTAs of 256 threads
// over tiles of FR consecutive frames of one row, both waveforms' sample spans staged per tile (TMA for interior
// tiles).  A frame is owned by LPF lanes of one warp and never leaves it: after the tile's span barrier only
// __syncwarp orders the frame's shared-memory slot.  Per frame:
//   1. target y: frame, window, FFT, untangle; |Y| stays in registers (STFT) or goes to the slot -> mel_y (mel);
//   2. estimate x: the SAME instruction sequence (identical inputs give identical |X|, mel and terms: loss(x, x) = 0
//      with a zero gradient), then the terms and dL/d|X| per bin (STFT) or per (mel, frame) cell, projected back to the
//      bins through the transposed band table (mel), times X / |X| from registers -> grad_x;
//   3. only when y requires a gradient: y's FFT again, dL/d|Y| times Y / |Y| -> grad_y.
// The loss: per-thread sums (float within a frame, double across frames), one partial pair per CTA, and a one-warp
// kernel that adds the partials in a fixed order (float64).  No atomics: reruns are bit-identical.
#include "b2a_common.h"
#include "fft_warp.cuh"
#include "spectral_internal.h"

namespace b2a {
namespace loss {

using spectral::WPlan;

constexpr float LN10 = 2.302585092994046f;

struct LossParams {
  spectral::Params px, py;  // framing of the estimate / the target: identical but for the base pointer
  const float* mel_fb;      // mel: [n_mels, F] filterbank, its band table and the transposed one; null: STFT loss
  const int32_t* mel_lo;
  const int32_t* mel_hi;
  const int32_t* bin_lo;
  const int32_t* bin_hi;
  int n_mels;
  float eps, power;
  float cl, cm;  // log_weight / numel, mag_weight / numel
  int use_log, use_mag;
  float2* gx;  // [rows, F, n_frames] or null
  float2* gy;
  double* partial;  // [gridDim.x][2]: sums of |log terms|, |magnitude terms|
  int off_spy, off_win, off_tw, off_ut, off_slot, slot;
};

// floats of the exchange plane of warp_fft (writes l*33 + t, reads e + e/32): N + N/32, >= the N + 1 magnitudes
template <int LOG2N>
struct LPlan {
  static constexpr int N = 1 << LOG2N;
  static constexpr int EX = ((N + N / 32 + 3) / 4) * 4;
};

__device__ __forceinline__ float sgn(float v) { return v > 0.f ? 1.f : (v < 0.f ? -1.f : 0.f); }
__device__ __forceinline__ float cabs(float2 v) { return sqrtf(fmaf(v.x, v.x, v.y * v.y)); }

__device__ __forceinline__ float lg(float v, float eps, float power) {
  const float c = fmaxf(v, eps);
  return log10f(power == 2.0f ? c * c : powf(c, power));
}

// One cell (a bin of a frame, or a (mel, frame) cell): adds its two L1 terms to sl / sm, returns (dL/dx, dL/dy).
__device__ __forceinline__ float2 cell(const LossParams& q, float vx, float vy, float& sl, float& sm) {
  float dx = 0.f, dy = 0.f;
  if (q.use_log) {
    const float d = lg(vx, q.eps, q.power) - lg(vy, q.eps, q.power);
    sl += fabsf(d);
    const float s = sgn(d) * q.cl * q.power;
    if (vx >= q.eps) dx = s / (LN10 * vx);
    if (vy >= q.eps) dy = -s / (LN10 * vy);
  }
  if (q.use_mag) {
    const float d = vx - vy;
    sm += fabsf(d);
    const float s = sgn(d) * q.cm;
    dx += s;
    dy -= s;
  }
  return make_float2(dx, dy);
}

// dL/dX = dL/d|X| X / |X|, 0 at X = 0 (torch's abs)
__device__ __forceinline__ float2 along(float d, float2 v) {
  const float m = cabs(v);
  if (!(m > 0.f)) return make_float2(0.f, 0.f);
  const float r = d / m;
  return make_float2(v.x * r, v.y * r);
}

// mel of filter m from the frame's magnitudes (the banded FP32 sum of spectral.cu)
__device__ __forceinline__ float project(const LossParams& q, int F, int m, const float* mag) {
  return spectral::mel_band(q.mel_fb, q.mel_lo, q.mel_hi, F, m, mag);
}

// sum over the filters whose band holds bin k of fb[m][k] g[m] (mel_backward_kernel's transposed projection)
__device__ __forceinline__ float back_project(const LossParams& q, int F, int k, const float* g) {
  float d = 0.f;
  for (int m = __ldg(q.bin_lo + k); m < __ldg(q.bin_hi + k); ++m)
    if (__ldg(q.mel_lo + m) <= k && k < __ldg(q.mel_hi + m)) d = fmaf(__ldg(q.mel_fb + (size_t)m * F + k), g[m], d);
  return d;
}

// windowed frame (window halved, first radix-32 butterfly fused) -> N-point FFT, z[m] = Z[l + LPF m]
template <int LOG2N>
__device__ __forceinline__ void frame_fft(const float* fs, const float* win, int hop, float2 (&z)[32], float* xb,
                                          const float2* tw, int l) {
  spectral::load_frame<LOG2N>(fs, win, hop, z, l);
  spectral::warp_fft<LOG2N, true>(z, xb, tw, l);
}

using spectral::untangle;

template <int LOG2N, bool MEL>
__global__ void __launch_bounds__(256, 2) spectral_loss_kernel(LossParams q) {
  using PL = WPlan<LOG2N>;
  constexpr int N = PL::N, LPF = PL::LPF, FPW = PL::FPW, FR = PL::FR;
  static_assert(FR == PL::G, "one frame per warp slot: the slot of a frame is its index in the tile");
  const spectral::Params& p = q.px;
  B2A_DYN_SMEM(smem);
  float* spx = reinterpret_cast<float*>(smem);
  float* spy = reinterpret_cast<float*>(smem + q.off_spy);
  float* win = reinterpret_cast<float*>(smem + q.off_win);
  float2* tw = reinterpret_cast<float2*>(smem + q.off_tw);
  float2* ut = reinterpret_cast<float2*>(smem + q.off_ut);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int hop = p.hop, F = N + 1, nf = p.n_frames;
  const int l = lane & (LPF - 1), fw = lane / LPF;
  const int src_lane = spectral::partner_lane<LPF>(lane);           // holder of Z[N - k]
  const int f = warp * FPW + fw;                                         // frame within the tile = its slot
  float* xb = reinterpret_cast<float*>(smem + q.off_slot) + f * q.slot;  // exchange plane, then |.| of the frame
  float* mel_y = xb + LPlan<LOG2N>::EX;                                   // mel: mel_y, then dL/dmel_y
  float* gm_x = mel_y + q.n_mels;                                         // mel: dL/dmel_x
  const int total = p.rows * p.n_tiles;

  __shared__ __align__(8) unsigned long long s_bar[2];
  __shared__ double s_red[8][2];
  if (tid == 0) { mbar_init(&s_bar[0], 1); mbar_init(&s_bar[1], 1); }
  for (int i = tid; i < 2 * N; i += 256) win[i] = 0.5f * __ldg(p.window + i);  // halved: see spectral_warp_kernel
  spectral::warp_fft_tables<LOG2N, PL::NUT>(tw, ut);

  unsigned par_x = 0, par_y = 0;
  double acc_l = 0.0, acc_m = 0.0;
#pragma unroll 1
  for (int t = blockIdx.x; t < total; t += gridDim.x) {
    const int row = t / p.n_tiles, tile = t - row * p.n_tiles;
    const int n0 = tile * FR;
    const int ws = (n0 + p.drop_edge) * hop + p.origin;
    __syncthreads();  // the previous tile is done with both spans (first tile: barriers and tables are set up)
    const bool tx = spectral::stage_span_async(q.px, spx, row, ws, &s_bar[0]);
    const bool ty = spectral::stage_span_async(q.py, spy, row, ws, &s_bar[1]);
    if (tx) { mbar_wait(&s_bar[0], par_x); par_x ^= 1u; }
    if (ty) { mbar_wait(&s_bar[1], par_y); par_y ^= 1u; }
    __syncthreads();

    const int n = n0 + f;
    const bool live = n < nf;
    const size_t o = (size_t)row * F * nf + n;
    float2* gx = (q.gx && live) ? q.gx + o : nullptr;
    float2* gy = (q.gy && live) ? q.gy + o : nullptr;
    float sl = 0.f, sm = 0.f;
    float2 z[32], a[16], b[16], h;

    frame_fft<LOG2N>(spy + f * hop, win, hop, z, xb, tw, l);
    untangle<LOG2N>(z, ut, l, src_lane, a, b, h);
    if constexpr (!MEL) {
      float ya[16], yb[16], yh;  // |Y| of the lane's bins
#pragma unroll
      for (int m = 0; m < 16; ++m) { ya[m] = cabs(a[m]); yb[m] = cabs(b[m]); }
      yh = cabs(h);
      frame_fft<LOG2N>(spx + f * hop, win, hop, z, xb, tw, l);
      untangle<LOG2N>(z, ut, l, src_lane, a, b, h);
      float da[16], db[16], dh = 0.f;  // dL/d|Y|
#pragma unroll
      for (int m = 0; m < 16; ++m) {
        const int k = l + LPF * m;
        const float2 ga = cell(q, cabs(a[m]), ya[m], sl, sm);
        const float2 gb = cell(q, cabs(b[m]), yb[m], sl, sm);
        if (gx) {
          gx[(size_t)k * nf] = along(ga.x, a[m]);
          gx[(size_t)(N - k) * nf] = along(gb.x, b[m]);
        }
        da[m] = ga.y;
        db[m] = gb.y;
      }
      if (l == 0) {
        const float2 gh = cell(q, cabs(h), yh, sl, sm);
        if (gx) gx[(size_t)(N / 2) * nf] = along(gh.x, h);
        dh = gh.y;
      }
      if (q.gy) {
        __syncwarp();
        frame_fft<LOG2N>(spy + f * hop, win, hop, z, xb, tw, l);
        untangle<LOG2N>(z, ut, l, src_lane, a, b, h);
        if (gy) {
#pragma unroll
          for (int m = 0; m < 16; ++m) {
            const int k = l + LPF * m;
            gy[(size_t)k * nf] = along(da[m], a[m]);
            gy[(size_t)(N - k) * nf] = along(db[m], b[m]);
          }
          if (l == 0) gy[(size_t)(N / 2) * nf] = along(dh, h);
        }
      }
    } else {
      const int n_mels = q.n_mels;
      // |Y| -> slot -> mel_y
#pragma unroll
      for (int m = 0; m < 16; ++m) {
        const int k = l + LPF * m;
        xb[k] = cabs(a[m]);
        xb[N - k] = cabs(b[m]);
      }
      if (l == 0) xb[N / 2] = cabs(h);
      __syncwarp();
      for (int mm = l; mm < n_mels; mm += LPF) mel_y[mm] = project(q, F, mm, xb);
      __syncwarp();
      // |X| -> slot -> mel_x, the terms, dL/dmel of both
      frame_fft<LOG2N>(spx + f * hop, win, hop, z, xb, tw, l);
      untangle<LOG2N>(z, ut, l, src_lane, a, b, h);
#pragma unroll
      for (int m = 0; m < 16; ++m) {
        const int k = l + LPF * m;
        xb[k] = cabs(a[m]);
        xb[N - k] = cabs(b[m]);
      }
      if (l == 0) xb[N / 2] = cabs(h);
      __syncwarp();
      for (int mm = l; mm < n_mels; mm += LPF) {
        const float2 g = cell(q, project(q, F, mm, xb), mel_y[mm], sl, sm);
        gm_x[mm] = g.x;
        mel_y[mm] = g.y;
      }
      __syncwarp();
      if (gx) {
#pragma unroll
        for (int m = 0; m < 16; ++m) {
          const int k = l + LPF * m;
          gx[(size_t)k * nf] = along(back_project(q, F, k, gm_x), a[m]);
          gx[(size_t)(N - k) * nf] = along(back_project(q, F, N - k, gm_x), b[m]);
        }
        if (l == 0) gx[(size_t)(N / 2) * nf] = along(back_project(q, F, N / 2, gm_x), h);
      }
      if (q.gy) {
        frame_fft<LOG2N>(spy + f * hop, win, hop, z, xb, tw, l);
        untangle<LOG2N>(z, ut, l, src_lane, a, b, h);
        if (gy) {
#pragma unroll
          for (int m = 0; m < 16; ++m) {
            const int k = l + LPF * m;
            gy[(size_t)k * nf] = along(back_project(q, F, k, mel_y), a[m]);
            gy[(size_t)(N - k) * nf] = along(back_project(q, F, N - k, mel_y), b[m]);
          }
          if (l == 0) gy[(size_t)(N / 2) * nf] = along(back_project(q, F, N / 2, mel_y), h);
        }
      }
    }
    if (live) {
      acc_l += (double)sl;
      acc_m += (double)sm;
    }
  }

  // the CTA's partial sums: fixed shuffle tree, then the 8 warps in order
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    acc_l += __shfl_xor_sync(0xffffffffu, acc_l, s);
    acc_m += __shfl_xor_sync(0xffffffffu, acc_m, s);
  }
  if (lane == 0) { s_red[warp][0] = acc_l; s_red[warp][1] = acc_m; }
  __syncthreads();
  if (tid == 0) {
    double sl = 0.0, sm = 0.0;
    for (int w = 0; w < 8; ++w) { sl += s_red[w][0]; sm += s_red[w][1]; }
    q.partial[2 * blockIdx.x] = sl;
    q.partial[2 * blockIdx.x + 1] = sm;
  }
}

// loss = wl * sum(partial log terms) + wm * sum(partial magnitude terms), the partials added in a fixed order
__global__ void __launch_bounds__(32) loss_finalize_kernel(const double* __restrict__ partial, int n, double wl, double wm,
                                                           float* __restrict__ out) {
  const int lane = threadIdx.x;
  double sl = 0.0, sm = 0.0;
  for (int i = lane; i < n; i += 32) { sl += partial[2 * i]; sm += partial[2 * i + 1]; }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    sl += __shfl_xor_sync(0xffffffffu, sl, s);
    sm += __shfl_xor_sync(0xffffffffu, sm, s);
  }
  if (lane == 0) out[0] = (float)(wl * sl + wm * sm);
}

constexpr int MAX_CTAS_PER_SM = 8;  // 256-thread CTAs: the partials buffer holds this many per SM

// shared-memory layout of one launch; returns the bytes
template <int LOG2N>
static int layout(LossParams& q, int hop, int n_mels) {
  using PL = WPlan<LOG2N>;
  const int span = (PL::FR - 1) * hop + 2 * PL::N;
  int o = align16(span * 4);
  q.off_spy = o; o = align16(o + span * 4);
  q.off_win = o; o = align16(o + 2 * PL::N * 4);
  q.off_tw = o; o = align16(o + PL::NTW * PL::LPF * 8 + 16);
  q.off_ut = o; o = align16(o + PL::NUT * PL::LPF * 8);
  q.slot = LPlan<LOG2N>::EX + ((2 * n_mels + 3) & ~3);
  q.off_slot = o; o = align16(o + PL::FR * q.slot * 4);
  return o;
}

static int smem_bytes(int n_fft, int hop, int n_mels) {
  LossParams q;
  switch (n_fft) {
    case 64: return layout<5>(q, hop, n_mels);
    case 128: return layout<6>(q, hop, n_mels);
    case 256: return layout<7>(q, hop, n_mels);
    case 512: return layout<8>(q, hop, n_mels);
    case 1024: return layout<9>(q, hop, n_mels);
    case 2048: return layout<10>(q, hop, n_mels);
  }
  return -1;
}

template <int LOG2N>
static int launch(LossParams& q, int64_t numel, double log_weight, double mag_weight, float* loss_out, void* stream) {
  using PL = WPlan<LOG2N>;
  spectral::Params& p = q.px;
  p.span = (PL::FR - 1) * p.hop + p.n_fft;
  p.n_tiles = (p.n_frames + PL::FR - 1) / PL::FR;
  q.py.span = p.span;
  q.py.n_tiles = p.n_tiles;
  const int o = layout<LOG2N>(q, p.hop, q.mel_fb ? q.n_mels : 0);
  B2A_REQUIRE(o <= 227 * 1024, B2A_E_UNSUPPORTED,
              "spectral_loss: n_fft=%d hop=%d n_mels=%d needs %d bytes of shared memory (> 227 KB)", p.n_fft, p.hop,
              q.n_mels, o);
  const int64_t total = (int64_t)p.rows * p.n_tiles;
  B2A_REQUIRE(total < (int64_t)2147483647, B2A_E_UNSUPPORTED, "spectral_loss: too many tiles");
  auto kern = q.mel_fb ? spectral_loss_kernel<LOG2N, true> : spectral_loss_kernel<LOG2N, false>;
  B2A_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, o));
  int64_t grid;
  const int rc = persistent_grid(kern, o, total, &grid, MAX_CTAS_PER_SM);
  if (rc != B2A_OK) return rc;
  B2A_LAUNCH(kern, dim3((unsigned)grid), dim3(256), (size_t)o, stream, q);
  B2A_CUDA_OK(cudaGetLastError());
  B2A_LAUNCH(loss_finalize_kernel, dim3(1), dim3(32), 0, stream, q.partial, (int)grid, log_weight / (double)numel,
             mag_weight / (double)numel, loss_out);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

static bool pow2_window(int n_fft) { return n_fft >= 64 && n_fft <= 2048 && (n_fft & (n_fft - 1)) == 0; }

}  // namespace loss
}  // namespace b2a

using namespace b2a::loss;

extern "C" int b2a_spectral_loss_supported(int n_fft, int hop, int n_mels) {
  if (!pow2_window(n_fft) || hop < 1 || hop > n_fft || n_mels < 0) return 0;
  return smem_bytes(n_fft, hop, n_mels) <= 227 * 1024;
}

extern "C" size_t b2a_spectral_loss_workspace_bytes(int n_fft, int hop, int n_mels) {
  if (!b2a_spectral_loss_supported(n_fft, hop, n_mels)) return 0;
  return (size_t)b2a::num_sms() * MAX_CTAS_PER_SM * 2 * sizeof(double);
}

extern "C" int b2a_spectral_loss_f32(const float* x, const float* y, int64_t rows, int64_t T, int n_fft, int hop,
                                     const float* window, int pad, int right_pad, int pad_mode, int drop_edge,
                                     const float* mel_fb, const int32_t* mel_lo, const int32_t* mel_hi,
                                     const int32_t* bin_lo, const int32_t* bin_hi, int n_mels, float clamp_eps,
                                     float power, float log_weight, float mag_weight, float* loss_out, float* grad_x,
                                     float* grad_y, void* workspace, size_t workspace_bytes, void* stream) {
  B2A_REQUIRE(x && y && window && loss_out && workspace, B2A_E_INVALID, "spectral_loss: null pointer");
  B2A_REQUIRE(rows >= 1 && rows <= 65535 && T >= 1 && T < ((int64_t)1 << 30), B2A_E_INVALID,
              "spectral_loss: bad shape");
  B2A_REQUIRE(hop >= 1 && hop <= n_fft, B2A_E_INVALID, "spectral_loss: hop_length must be in [1, window_length]");
  B2A_REQUIRE(pow2_window(n_fft), B2A_E_UNSUPPORTED,
              "spectral_loss: window_length must be a power of two in [64, 2048] (got %d)", n_fft);
  const bool mel = mel_fb != nullptr;
  B2A_REQUIRE(!mel || (mel_lo && mel_hi && bin_lo && bin_hi && n_mels >= 1), B2A_E_INVALID,
              "spectral_loss: mel arguments");
  B2A_REQUIRE(clamp_eps > 0.f && power > 0.f, B2A_E_INVALID, "spectral_loss: clamp_eps and pow must be > 0");
  int64_t nfr;
  const int rc = b2a::spectral::check_framing("spectral_loss", T, n_fft, hop, pad, right_pad, pad_mode, drop_edge, &nfr);
  if (rc != B2A_OK) return rc;
  B2A_REQUIRE(workspace_bytes >= b2a_spectral_loss_workspace_bytes(n_fft, hop, mel ? n_mels : 0) &&
                  ((uintptr_t)workspace & 7) == 0,
              B2A_E_INVALID, "spectral_loss: workspace too small or not 8-byte aligned");
  B2A_REQUIRE(((uintptr_t)grad_x & 7) == 0 && ((uintptr_t)grad_y & 7) == 0, B2A_E_INVALID,
              "spectral_loss: gradients must be 8-byte aligned");
  LossParams q;
  memset(&q, 0, sizeof(q));
  b2a::spectral::Params& p = q.px;
  p.x = x; p.window = window;
  p.rows = (int)rows; p.T = (int)T; p.n_fft = n_fft; p.hop = hop; p.pad = pad; p.right_pad = right_pad;
  p.pad_mode = pad_mode; p.drop_edge = drop_edge; p.n_frames = (int)nfr; p.rows_per_gain = 1;
  p.center = 1; p.origin = -(n_fft / 2) - pad; p.row_origin = nullptr;
  q.py = p;
  q.py.x = y;
  q.mel_fb = mel_fb; q.mel_lo = mel_lo; q.mel_hi = mel_hi; q.bin_lo = bin_lo; q.bin_hi = bin_hi;
  q.n_mels = mel ? n_mels : 0;
  q.eps = clamp_eps; q.power = power;
  const int F = n_fft / 2 + 1;
  const int64_t numel = rows * (mel ? (int64_t)n_mels : (int64_t)F) * nfr;
  q.cl = (float)((double)log_weight / (double)numel);
  q.cm = (float)((double)mag_weight / (double)numel);
  q.use_log = log_weight != 0.f;
  q.use_mag = mag_weight != 0.f;
  q.gx = reinterpret_cast<float2*>(grad_x);
  q.gy = reinterpret_cast<float2*>(grad_y);
  q.partial = reinterpret_cast<double*>(workspace);
  switch (n_fft) {
    case 64: return launch<5>(q, numel, log_weight, mag_weight, loss_out, stream);
    case 128: return launch<6>(q, numel, log_weight, mag_weight, loss_out, stream);
    case 256: return launch<7>(q, numel, log_weight, mag_weight, loss_out, stream);
    case 512: return launch<8>(q, numel, log_weight, mag_weight, loss_out, stream);
    case 1024: return launch<9>(q, numel, log_weight, mag_weight, loss_out, stream);
    default: return launch<10>(q, numel, log_weight, mag_weight, loss_out, stream);
  }
}
