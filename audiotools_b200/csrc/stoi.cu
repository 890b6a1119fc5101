// stoi.cu -- short-time objective intelligibility (STOI) and extended STOI of a batch, on sm_90a.
//
// Replaces the per-item pystoi loop of ref:audiotools/metrics/quality.py:11-57: to_mono, then pystoi.stoi(ref, est, sr,
// extended) with the CLEAN signal as pystoi's x.  Four launches, no atomics (reruns are bit-identical):
//   1. resample_kernel  mono (float32 mean over channels) and scipy.signal.resample_poly(x, up, down, window=taps) to
//                       10 kHz, both signals in one launch: zero-padded polyphase FIR,
//                         out[m] = sum_n taps[m*down + half - n*up] x[n],  half = (n_taps - 1) / 2,
//                       m < ceil(T up / down); taps in float64, accumulation in float64, output float32.
//   2. mask_kernel      one CTA per item: energies (float64) of the 256-sample Hann frames of the clean signal at hop
//                       128, starts 0, 128, ... < n10 - 256; keep a frame when max - 40 - e < 0; a block scan writes
//                       the kept frame indices in order and their count K.
//   3. band_kernel      the STFT of the silence-removed signals (M = K - 1 frames) without materialising them: sample
//                       j*128 + n of a silence-removed signal is w[n] x[s_j + n] + w[n + 128] x[s_(j-1) + n + 128]
//                       (s_j = start of kept frame j).  Each frame is windowed again, zero-padded to 512 and
//                       transformed by the warp FFT of fft_warp.cuh (256 complex points, 8 lanes per frame);
//                       |X|^2 is summed over the 15 contiguous third-octave bands -> tob[signal][item][band][frame].
//   4. score_kernel     one CTA per item, float64: the segments of 30 frames, standard (scale, clip at -15 dB SDR,
//                       correlation) or extended (row then column normalisation); 1e-5 and a flag when M < 30.
// The backward (metrics.quality.STOILoss: dL/dscore -> dL/d estimate, the references are constants) reads the forward's
// workspace and is four more launches, no atomics, each the adjoint of one forward stage in reverse order:
// score_bwd_kernel (float64 cells, then a per-frame gather), band_bwd_kernel (the estimate's frame spectra recomputed
// by the same frame_spectrum as band_kernel, weighted, inverse real FFT), unframe_kernel (the adjoint of the silence
// removal, a gather) and resample_bwd_kernel (the transposed polyphase FIR, a gather, then the 1/C of the mono mix).
#include "b2a_common.h"
#include "fft_warp.cuh"

namespace b2a {
namespace stoi {

constexpr int THREADS = 256;
constexpr int OPT = 4;                       // outputs per thread of the resampler
constexpr int OUT_PER_CTA = THREADS * OPT;
constexpr int FRAME = 256, HOP = 128;        // pystoi's N_FRAME and its hop (overlap 2)
constexpr int LOG2N = 8;                     // 512-point real FFT = 256-point complex FFT
constexpr int NBAND = 15, SEG = 30;          // third-octave bands, frames per segment
constexpr int FRAMES_PER_CTA = 32;           // band_kernel: 8 warps x 4 frames
constexpr double EPS = 2.220446049250313e-16;  // np.finfo(float).eps
constexpr double DYN_RANGE = 40.0;

// bin edges of the third-octave bands (pystoi's thirdoct(10000, 512, 15, 150), band k = bins [edge(k), edge(k + 1)))
__device__ __forceinline__ int band_edge(int k) {
  switch (k) {
    case 0: return 7;    case 1: return 9;    case 2: return 11;   case 3: return 14;
    case 4: return 17;   case 5: return 22;   case 6: return 27;   case 7: return 34;
    case 8: return 43;   case 9: return 55;   case 10: return 69;  case 11: return 87;
    case 12: return 109; case 13: return 138; case 14: return 174; default: return 219;
  }
}

// np.hanning(258)[1:-1][n] = 0.5 + 0.5 cos(pi (2n + 2 - 257) / 257)
__device__ __forceinline__ double hann(int n) {
  double s, c;
  sincospi((double)(2 * n + 2 - 257) / 257.0, &s, &c);
  return 0.5 + 0.5 * c;
}

// np.minimum / np.max: a NaN operand gives NaN (fmin and fmax return the other operand)
__device__ __forceinline__ double min_nan(double a, double b) { return isnan(a) || isnan(b) ? a + b : fmin(a, b); }
__device__ __forceinline__ double max_nan(double a, double b) { return isnan(a) || isnan(b) ? a + b : fmax(a, b); }
// d min(a, b) / d a: 1, 1/2 at a tie (as torch.minimum), 0; NaN when either operand is NaN
__device__ __forceinline__ double tie_mask(double a, double b) {
  return isnan(a) || isnan(b) ? a + b : (a < b ? 1.0 : (a == b ? 0.5 : 0.0));
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// fixed-order block sum of one double per thread (the result is valid on thread 0)
__device__ __forceinline__ double block_sum_d(double v, double* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int h = THREADS / 2; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  return red[0];
}

// rows [0, B) of `out` are the estimates, [B, 2B) the references
__global__ void __launch_bounds__(THREADS)
resample_kernel(const float* __restrict__ est, const float* __restrict__ ref, int B, int C, int64_t T,
                const double* __restrict__ taps, int n_taps, int up, int down, int KP, int64_t n10, int tiles,
                float* __restrict__ out) {
  B2A_DYN_SMEM(smem);
  float* xs = reinterpret_cast<float*>(smem);
  const int row = blockIdx.x / tiles, tile = blockIdx.x - row * tiles;
  const float* x = row < B ? est + (size_t)row * C * T : ref + (size_t)(row - B) * C * T;
  const int64_t half = (n_taps - 1) / 2;
  const int64_t o0 = (int64_t)tile * OUT_PER_CTA;
  const int64_t o_end = min(o0 + OUT_PER_CTA, n10);
  const int64_t nlo = (o0 * down + half) / up - (KP - 1);  // first input sample the tile reads (may be < 0)
  const int64_t nhi = ((o_end - 1) * down + half) / up;
  const int span = (int)(nhi - nlo + 1);
  for (int i = threadIdx.x; i < span; i += THREADS) {
    const int64_t u = nlo + i;
    float v = 0.f;  // zero padding outside the signal
    if (u >= 0 && u < T) {
      float s = __ldg(x + u);
      for (int c = 1; c < C; ++c) s += __ldg(x + (size_t)c * T + u);
      v = s / (float)C;
    }
    xs[i] = v;
  }
  __syncthreads();
  float* orow = out + (size_t)row * n10;
#pragma unroll
  for (int j = 0; j < OPT; ++j) {
    const int64_t m = o0 + threadIdx.x + (int64_t)THREADS * j;
    if (m >= o_end) break;
    const int64_t a = m * down + half;
    const int64_t nh = a / up;               // newest input sample of output m; it meets tap r
    const int r = (int)(a - nh * up);
    const float* xr = xs + (nh - nlo);       // xr[-k] = x[nh - k] meets tap r + k up
    double acc = 0.0;
    for (int k = 0, t = r; k < KP && t < n_taps; ++k, t += up) acc = fma((double)xr[-k], __ldg(taps + t), acc);
    orow[m] = (float)acc;
  }
}

__global__ void __launch_bounds__(THREADS)
mask_kernel(const float* __restrict__ ref10, int64_t n10, int n_fr, double* __restrict__ energy,
            int32_t* __restrict__ kept, int32_t* __restrict__ count) {
  __shared__ double red[THREADS / 32];
  __shared__ int wtot[THREADS / 32];
  const int item = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* x = ref10 + (size_t)item * n10;
  double* e = energy + (size_t)item * n_fr;
  int32_t* list = kept + (size_t)item * n_fr;
  double w[FRAME / 32];
#pragma unroll
  for (int i = 0; i < FRAME / 32; ++i) w[i] = hann(lane + 32 * i);
  // 1. frame energies in dB, one warp per frame; running maximum
  double emax = -INFINITY;
  for (int f = warp; f < n_fr; f += THREADS / 32) {
    const float* xf = x + (int64_t)f * HOP;
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < FRAME / 32; ++i) {
      const double v = w[i] * (double)__ldg(xf + lane + 32 * i);
      s = fma(v, v, s);
    }
    const double ef = 20.0 * log10(sqrt(warp_sum_d(s)) + EPS);
    if (lane == 0) e[f] = ef;
    emax = max_nan(emax, ef);
  }
  if (lane == 0) red[warp] = emax;
  __syncthreads();  // also orders the energies written above before the reads below
  emax = red[0];
  for (int i = 1; i < THREADS / 32; ++i) emax = max_nan(emax, red[i]);
  // 2. keep flags -> exclusive scan -> indices of the kept frames, in order (a NaN energy makes emax NaN and keeps
  //    no frame, as pystoi's np.max: the item is short)
  int carry = 0;
  for (int f0 = 0; f0 < n_fr; f0 += THREADS) {
    const int f = f0 + tid;
    const int keep = (f < n_fr && (emax - DYN_RANGE - e[f]) < 0.0) ? 1 : 0;
    int incl = keep;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += t;
    }
    if (lane == 31) wtot[warp] = incl;
    __syncthreads();
    int off = carry + incl - keep, total = 0;
    for (int i = 0; i < THREADS / 32; ++i) {
      if (i < warp) off += wtot[i];
      total += wtot[i];
    }
    if (keep) list[off] = f;
    carry += total;
    __syncthreads();  // wtot is rewritten by the next chunk
  }
  if (tid == 0) count[item] = carry;
}

// sample n (0 <= n < 256) of frame i of the silence-removed signal (kept frames s_prev, s_i, s_next; s_prev < 0: none)
__device__ __forceinline__ float removed_sample(const float* x, const float* win, int64_t s_prev, int64_t s_i,
                                                int64_t s_next, int n) {
  const float head = win[n] * __ldg(x + s_i + n);
  if (n < HOP) return s_prev >= 0 ? fmaf(win[n + HOP], __ldg(x + s_prev + n + HOP), head) : head;
  return fmaf(win[n - HOP], __ldg(x + s_next + n - HOP), head);
}

// The 512-point rFFT of one STOI frame of the silence-removed signal x (kept frame starts s_prev, s_i, s_next), held by
// the LPF lanes of its frame: a[m] = X[k], b[m] = X[256 - k] for k = l + LPF m (m < 16), h = X[128] (valid on l == 0).
// band_kernel and band_bwd_kernel both call it, so the backward transforms exactly the frames the forward did.
// pb is the frame's exchange plane; warp_fft ends on a __syncwarp after its last read of it.
__device__ __forceinline__ void frame_spectrum(const float* x, const float* win, int64_t s_prev, int64_t s_i,
                                               int64_t s_next, float* pb, const float2* tw, const float2* ut, int l,
                                               int src_lane, float2 (&a)[16], float2 (&b)[16], float2& h) {
  constexpr int LPF = spectral::WPlan<LOG2N>::LPF;
  float2 z[32];
  // complex element e = l + LPF m holds samples 2e, 2e + 1 (times the halved window); elements 128..255 are the zero
  // padding, so the first butterfly stage (e, e + 128) gives the same value twice
#pragma unroll
  for (int m = 0; m < 16; ++m) {
    const int n = 2 * (l + LPF * m);
    const float v0 = 0.5f * win[n] * removed_sample(x, win, s_prev, s_i, s_next, n);
    const float v1 = 0.5f * win[n + 1] * removed_sample(x, win, s_prev, s_i, s_next, n + 1);
    z[m] = z[m + 16] = make_float2(v0, v1);
  }
  spectral::warp_fft<LOG2N, true>(z, pb, tw, l);
  spectral::untangle<LOG2N>(z, ut, l, src_lane, a, b, h);
}

__global__ void __launch_bounds__(THREADS)
band_kernel(const float* __restrict__ sig10, int B, int64_t n10, int n_fr, const int32_t* __restrict__ kept,
            const int32_t* __restrict__ count, float* __restrict__ tob) {
  using PL = spectral::WPlan<LOG2N>;
  constexpr int LPF = PL::LPF, FPW = PL::FPW;
  static_assert(FRAMES_PER_CTA == (THREADS / 32) * FPW, "one frame per LPF lanes");
  constexpr int XB = 33 * LPF;  // exchange plane of warp_fft (writes l*33 + t, reads e + e/32), then |X|^2 (257)
  static_assert(XB >= FRAME + 1, "");
  __shared__ float2 tw[PL::NTW * LPF];
  __shared__ float2 ut[16 * LPF];
  __shared__ float win[FRAME];
  __shared__ float xb[FRAMES_PER_CTA][XB];
  const int item = blockIdx.y;
  const int M = __ldg(count + item) - 1;
  const int i0 = blockIdx.x * FRAMES_PER_CTA;
  if (i0 >= M) return;  // the grid covers the longest possible item
  spectral::warp_fft_tables<LOG2N, 16>(tw, ut);
  for (int n = threadIdx.x; n < FRAME; n += THREADS) win[n] = (float)hann(n);
  __syncthreads();
  const int lane = threadIdx.x & 31, l = lane & (LPF - 1);
  const int slot = (threadIdx.x >> 5) * FPW + lane / LPF;
  const bool live = i0 + slot < M;
  const int i = live ? i0 + slot : M - 1;  // lanes of a frame past M repeat the last one and write nothing
  const int32_t* list = kept + (size_t)item * n_fr;
  const int64_t s_i = (int64_t)__ldg(list + i) * HOP, s_next = (int64_t)__ldg(list + i + 1) * HOP;
  const int64_t s_prev = i >= 1 ? (int64_t)__ldg(list + i - 1) * HOP : -1;
  const int src_lane = spectral::partner_lane<LPF>(lane);
  float* pb = xb[slot];
  for (int sig = 0; sig < 2; ++sig) {
    const float* x = sig10 + ((size_t)sig * B + item) * n10;
    float2 a[16], b[16], h;
    frame_spectrum(x, win, s_prev, s_i, s_next, pb, tw, ut, l, src_lane, a, b, h);
#pragma unroll
    for (int m = 0; m < 16; ++m) {  // warp_fft ends on a __syncwarp after its last read of pb
      const int k = l + LPF * m;
      pb[k] = fmaf(a[m].x, a[m].x, a[m].y * a[m].y);
      pb[PL::N - k] = fmaf(b[m].x, b[m].x, b[m].y * b[m].y);  // X[256 - k]; k = 0 gives the Nyquist bin
    }
    if (l == 0) pb[PL::N / 2] = fmaf(h.x, h.x, h.y * h.y);
    __syncwarp();
    if (live) {
      for (int band = l; band < NBAND; band += LPF) {
        float s = 0.f;
        for (int k = band_edge(band); k < band_edge(band + 1); ++k) s += pb[k];
        tob[(((size_t)sig * B + item) * NBAND + band) * n_fr + i] = sqrtf(s);
      }
    }
    __syncwarp();  // pb is the exchange plane of the next signal's FFT
  }
}

__global__ void __launch_bounds__(THREADS)
score_kernel(const float* __restrict__ tob, int B, int n_fr, const int32_t* __restrict__ count, int extended,
             double* __restrict__ out, int32_t* __restrict__ kept_out, int32_t* __restrict__ short_out) {
  __shared__ double red[THREADS];
  const int item = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int K = __ldg(count + item), M = K - 1;
  if (tid == 0) {
    kept_out[item] = K;
    short_out[item] = M < SEG;
  }
  if (M < SEG) {
    if (tid == 0) out[item] = 1e-5;
    return;
  }
  const int J = M - SEG + 1;
  const float* tx = tob + ((size_t)B + item) * NBAND * n_fr;  // clean (the reference): pystoi's x
  const float* ty = tob + (size_t)item * NBAND * n_fr;        // processed (the estimate): pystoi's y
  double acc = 0.0;
  if (!extended) {
    const double clip = 1.0 + pow(10.0, 15.0 / 20.0);  // 1 + 10^(-BETA/20)
    for (int p = tid; p < J * NBAND; p += THREADS) {
      const int j = p / NBAND, band = p - j * NBAND;
      const float* xr = tx + (size_t)band * n_fr + j;
      const float* yr = ty + (size_t)band * n_fr + j;
      double sxx = 0.0, syy = 0.0;
      for (int t = 0; t < SEG; ++t) {
        const double xv = xr[t], yv = yr[t];
        sxx = fma(xv, xv, sxx);
        syy = fma(yv, yv, syy);
      }
      const double c = sqrt(sxx) / (sqrt(syy) + EPS);
      double mx = 0.0, my = 0.0;
      for (int t = 0; t < SEG; ++t) {
        const double xv = xr[t];
        mx += xv;
        my += min_nan((double)yr[t] * c, xv * clip);
      }
      mx /= SEG;
      my /= SEG;
      double sxy = 0.0, sx2 = 0.0, sy2 = 0.0;
      for (int t = 0; t < SEG; ++t) {
        const double xv = xr[t];
        const double dx = xv - mx, dy = min_nan((double)yr[t] * c, xv * clip) - my;
        sxy = fma(dx, dy, sxy);
        sx2 = fma(dx, dx, sx2);
        sy2 = fma(dy, dy, sy2);
      }
      acc += sxy / ((sqrt(sx2) + EPS) * (sqrt(sy2) + EPS));
    }
    acc = block_sum_d(acc, red) / ((double)J * NBAND);
  } else {
    // one warp per segment: lanes 0..14 normalise the band rows, lanes 0..29 then the frame columns
    const int t = lane < SEG ? lane : SEG - 1;
    double wacc = 0.0;
    for (int j = warp; j < J; j += THREADS / 32) {
      double mux = 0.0, isx = 0.0, muy = 0.0, isy = 0.0;  // row mean and 1 / norm of the centred row
      if (lane < NBAND) {
        const float* xr = tx + (size_t)lane * n_fr + j;
        const float* yr = ty + (size_t)lane * n_fr + j;
        for (int s = 0; s < SEG; ++s) { mux += xr[s]; muy += yr[s]; }
        mux /= SEG;
        muy /= SEG;
        double vx = 0.0, vy = 0.0;
        for (int s = 0; s < SEG; ++s) {
          const double dx = xr[s] - mux, dy = yr[s] - muy;
          vx = fma(dx, dx, vx);
          vy = fma(dy, dy, vy);
        }
        isx = 1.0 / sqrt(vx);
        isy = 1.0 / sqrt(vy);
      }
      double u[NBAND], v[NBAND], nu = 0.0, nv = 0.0;
#pragma unroll
      for (int band = 0; band < NBAND; ++band) {
        const double mx = __shfl_sync(0xffffffffu, mux, band), ix = __shfl_sync(0xffffffffu, isx, band);
        const double my = __shfl_sync(0xffffffffu, muy, band), iy = __shfl_sync(0xffffffffu, isy, band);
        u[band] = ((double)tx[(size_t)band * n_fr + j + t] - mx) * ix;
        v[band] = ((double)ty[(size_t)band * n_fr + j + t] - my) * iy;
        nu += u[band];
        nv += v[band];
      }
      nu /= NBAND;
      nv /= NBAND;
      double suv = 0.0, suu = 0.0, svv = 0.0;
#pragma unroll
      for (int band = 0; band < NBAND; ++band) {
        const double du = u[band] - nu, dv = v[band] - nv;
        suv = fma(du, dv, suv);
        suu = fma(du, du, suu);
        svv = fma(dv, dv, svv);
      }
      const double col = lane < SEG ? suv / (sqrt(suu) * sqrt(svv)) : 0.0;
      wacc += warp_sum_d(col) / SEG;
    }
    acc = block_sum_d(lane == 0 ? wacc : 0.0, red) / J;
  }
  if (tid == 0) {
    out[item] = acc;
  }
}

// ---- backward (dL/dscore -> dL/d estimate); notation of b2a.h: y the estimate's 10 kHz signal, s_j the kept frame
//      starts, M = K - 1 STOI frames, tob[b][i] the band envelopes of the estimate

// 1. dL/dtob_y.  Phase 1 writes the derivative of each cell's term by the estimate's envelope into cell[j][b][t]
//    (standard: d rho_{j,b} / d y_t of one (segment, band) cell; extended: d (sum of segment j's column correlations
//    / 30) / d y[b][t]).  Phase 2 gathers the <= 30 cells of every (band, frame) in segment order, times
//    dL/dscore / (number of terms of the mean).  The frame -> kept-position map of the un-framing is built here too.
__global__ void __launch_bounds__(THREADS)
score_bwd_kernel(const double* __restrict__ grad_score, const float* __restrict__ tob, int B, int n_fr,
                 const int32_t* __restrict__ kept, const int32_t* __restrict__ count, int extended,
                 float* __restrict__ cell, double* __restrict__ gbar, int32_t* __restrict__ pos) {
  const int item = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int K = __ldg(count + item), M = K - 1;
  int32_t* pm = pos + (size_t)item * n_fr;
  for (int f = tid; f < n_fr; f += THREADS) pm[f] = -1;
  __syncthreads();
  for (int j = tid; j < K; j += THREADS) pm[__ldg(kept + (size_t)item * n_fr + j)] = j;
  if (M < SEG) return;  // scored 1e-5: a constant, zero gradient (the later kernels write zeros for it)
  const int J = M - SEG + 1;
  const float* tx = tob + ((size_t)B + item) * NBAND * n_fr;
  const float* ty = tob + (size_t)item * NBAND * n_fr;
  float* cl = cell + (size_t)item * n_fr * NBAND * SEG;  // [J][NBAND][SEG]
  if (!extended) {
    const double clip = 1.0 + pow(10.0, 15.0 / 20.0);
    for (int p = tid; p < J * NBAND; p += THREADS) {
      const int j = p / NBAND, band = p - j * NBAND;
      const float* xr = tx + (size_t)band * n_fr + j;
      const float* yr = ty + (size_t)band * n_fr + j;
      // the forward's statistics, in its order
      double sxx = 0.0, syy = 0.0;
      for (int t = 0; t < SEG; ++t) {
        const double xv = xr[t], yv = yr[t];
        sxx = fma(xv, xv, sxx);
        syy = fma(yv, yv, syy);
      }
      const double nx = sqrt(sxx), ny = sqrt(syy);
      const double c = nx / (ny + EPS);
      double mx = 0.0, my = 0.0;
      for (int t = 0; t < SEG; ++t) {
        const double xv = xr[t];
        mx += xv;
        my += min_nan((double)yr[t] * c, xv * clip);
      }
      mx /= SEG;
      my /= SEG;
      double sxy = 0.0, sx2 = 0.0, sy2 = 0.0;
      for (int t = 0; t < SEG; ++t) {
        const double xv = xr[t];
        const double dx = xv - mx, dy = min_nan((double)yr[t] * c, xv * clip) - my;
        sxy = fma(dx, dy, sxy);
        sx2 = fma(dx, dx, sx2);
        sy2 = fma(dy, dy, sy2);
      }
      const double nu = sqrt(sx2), nv = sqrt(sy2);
      const double iuv = 1.0 / ((nu + EPS) * (nv + EPS));
      const double rho = sxy * iuv;
      const double rv = nv > 0.0 ? rho / (nv * (nv + EPS)) : 0.0;  // a zero norm backpropagates 0
      // A_t = d rho / d a_t, m_t = d a_t / d (c y_t) (1/2 at a tie, as torch.minimum); S = sum_t m_t y_t A_t
      double S = 0.0;
      for (int t = 0; t < SEG; ++t) {
        const double xv = xr[t], yv = yr[t];
        const double cy = yv * c, kx = xv * clip;
        const double A = (xv - mx) * iuv - rv * (min_nan(cy, kx) - my);
        const double mt = tie_mask(cy, kx);
        S = fma(mt * yv, A, S);
      }
      const double q = ny > 0.0 ? nx * S / (ny * (ny + EPS) * (ny + EPS)) : 0.0;  // -d c / d y_s = q' y_s
      float* o = cl + ((size_t)j * NBAND + band) * SEG;
      for (int t = 0; t < SEG; ++t) {
        const double xv = xr[t], yv = yr[t];
        const double cy = yv * c, kx = xv * clip;
        const double A = (xv - mx) * iuv - rv * (min_nan(cy, kx) - my);
        const double mt = tie_mask(cy, kx);
        o[t] = (float)(c * mt * A - q * yv);
      }
    }
  } else {
    // one warp per segment as in score_kernel: lane t < 30 owns column t.  The vector-Jacobian product of a unit
    // normalisation z = (w - mean w) / |w - mean w| is (g - mean g - z (z . g)) / |w - mean w|: columns, then rows.
    const int t = lane < SEG ? lane : SEG - 1;
    for (int j = warp; j < J; j += THREADS / 32) {
      double mux = 0.0, isx = 0.0, muy = 0.0, isy = 0.0;
      if (lane < NBAND) {
        const float* xr = tx + (size_t)lane * n_fr + j;
        const float* yr = ty + (size_t)lane * n_fr + j;
        for (int s = 0; s < SEG; ++s) { mux += xr[s]; muy += yr[s]; }
        mux /= SEG;
        muy /= SEG;
        double vx = 0.0, vy = 0.0;
        for (int s = 0; s < SEG; ++s) {
          const double dx = xr[s] - mux, dy = yr[s] - muy;
          vx = fma(dx, dx, vx);
          vy = fma(dy, dy, vy);
        }
        isx = 1.0 / sqrt(vx);
        isy = 1.0 / sqrt(vy);
      }
      double u[NBAND], v[NBAND], nu = 0.0, nv = 0.0;
#pragma unroll
      for (int band = 0; band < NBAND; ++band) {
        const double mx = __shfl_sync(0xffffffffu, mux, band), ix = __shfl_sync(0xffffffffu, isx, band);
        const double my = __shfl_sync(0xffffffffu, muy, band), iy = __shfl_sync(0xffffffffu, isy, band);
        u[band] = ((double)tx[(size_t)band * n_fr + j + t] - mx) * ix;
        v[band] = ((double)ty[(size_t)band * n_fr + j + t] - my) * iy;
        nu += u[band];
        nv += v[band];
      }
      nu /= NBAND;
      nv /= NBAND;
      double suv = 0.0, suu = 0.0, svv = 0.0;
#pragma unroll
      for (int band = 0; band < NBAND; ++band) {
        const double du = u[band] - nu, dv = v[band] - nv;
        suv = fma(du, dv, suv);
        suu = fma(du, du, suu);
        svv = fma(dv, dv, svv);
      }
      const double su = sqrt(suu), sv = sqrt(svv);
      const double col = suv / (su * sv);
      // column VJP: g = the normalised column of x, z = the normalised column of y, z . g = col; the 1/30 of the
      // segment's mean folded in.  u[] becomes the gradient by the row-normalised y.
      double gm = 0.0;
#pragma unroll
      for (int band = 0; band < NBAND; ++band) gm += (u[band] - nu) / su;
      gm /= NBAND;
#pragma unroll
      for (int band = 0; band < NBAND; ++band)
        u[band] = lane < SEG ? ((u[band] - nu) / su - gm - (v[band] - nv) / sv * col) / sv / SEG : 0.0;
      // row VJP: row b of y is normalised over the 30 columns (z = v[b] across the lanes)
      float* o = cl + (size_t)j * NBAND * SEG;
#pragma unroll
      for (int band = 0; band < NBAND; ++band) {
        const double iy = __shfl_sync(0xffffffffu, isy, band);
        const double hm = warp_sum_d(u[band]) / SEG;
        const double zh = warp_sum_d(lane < SEG ? v[band] * u[band] : 0.0);
        if (lane < SEG) o[band * SEG + lane] = (float)((u[band] - hm - v[band] * zh) * iy);
      }
    }
  }
  __syncthreads();  // the cells of other threads are read below
  const double scale = __ldg(grad_score + item) / (extended ? (double)J : (double)J * NBAND);
  for (int p = tid; p < NBAND * M; p += THREADS) {
    const int band = p / M, i = p - band * M;
    double acc = 0.0;
    for (int j = max(0, i - SEG + 1); j <= min(i, J - 1); ++j) acc += cl[((size_t)j * NBAND + band) * SEG + i - j];
    gbar[((size_t)item * NBAND + band) * n_fr + i] = acc * scale;
  }
}

// 2. dL/d(STOI frame i of the estimate): W_k = Gbar[b][i] Y_k / tob[b][i] on the bins of band b (0 where tob = 0 and
//    outside bins 7..218), then ghat_i[n] = w[n] sum_k Re(W_k e^{+2 pi i k n / 512}), n < 256.  The inverse real FFT is
//    conj(FFT(conj Z)) of the 256-point complex Z[k] = (P + i E) / 2, P = W_k + conj W_{256-k},
//    E = e^{i pi k / 256} (W_k - conj W_{256-k}), whose output z[e] = h[2e] + i h[2e + 1] (istft_kernel's packing).
//    A lane holds W_k and W_{256-k} of its k = l + LPF m, so Z[k] and Z[256 - k] are both formed in registers and the
//    latter is handed to the partner lane that owns element 256 - k.
__global__ void __launch_bounds__(THREADS)
band_bwd_kernel(const float* __restrict__ sig10, int64_t n10, int n_fr, const int32_t* __restrict__ kept,
                const int32_t* __restrict__ count, const float* __restrict__ tob, const double* __restrict__ gbar,
                float* __restrict__ ghat) {
  using PL = spectral::WPlan<LOG2N>;
  constexpr int LPF = PL::LPF, FPW = PL::FPW, N = PL::N;
  constexpr int XB = 33 * LPF;  // exchange plane of warp_fft, then the per-bin weights Gbar / tob (257)
  static_assert(XB >= N + 1, "");
  __shared__ float2 tw[PL::NTW * LPF];
  __shared__ float2 ut[16 * LPF];
  __shared__ float win[FRAME];
  __shared__ float xb[FRAMES_PER_CTA][XB];
  const int item = blockIdx.y;
  const int M = __ldg(count + item) - 1;
  const int i0 = blockIdx.x * FRAMES_PER_CTA;
  if (M < SEG || i0 >= M) return;  // a short item's frames carry no gradient
  spectral::warp_fft_tables<LOG2N, 16>(tw, ut);
  for (int n = threadIdx.x; n < FRAME; n += THREADS) win[n] = (float)hann(n);
  __syncthreads();
  const int lane = threadIdx.x & 31, l = lane & (LPF - 1);
  const int slot = (threadIdx.x >> 5) * FPW + lane / LPF;
  const bool live = i0 + slot < M;
  const int i = live ? i0 + slot : M - 1;
  const int32_t* list = kept + (size_t)item * n_fr;
  const int64_t s_i = (int64_t)__ldg(list + i) * HOP, s_next = (int64_t)__ldg(list + i + 1) * HOP;
  const int64_t s_prev = i >= 1 ? (int64_t)__ldg(list + i - 1) * HOP : -1;
  const int src_lane = spectral::partner_lane<LPF>(lane);
  float* pb = xb[slot];
  float2 a[16], b[16], h;
  frame_spectrum(sig10 + (size_t)item * n10, win, s_prev, s_i, s_next, pb, tw, ut, l, src_lane, a, b, h);
  for (int k = l; k <= N; k += LPF) pb[k] = 0.f;
  __syncwarp();
  const float* ty = tob + (size_t)item * NBAND * n_fr + i;
  const double* gb = gbar + (size_t)item * NBAND * n_fr + i;
  for (int band = l; band < NBAND; band += LPF) {
    const float tv = ty[(size_t)band * n_fr];
    const float cf = tv > 0.f ? (float)(gb[(size_t)band * n_fr] / (double)tv) : 0.f;
    for (int k = band_edge(band); k < band_edge(band + 1); ++k) pb[k] = cf;
  }
  __syncwarp();
  float2 z[32], pz[16];  // z: 2 conj Z[e] of the lane's elements e = l + LPF m; pz[m]: 2 conj Z[256 - k] of pair m
#pragma unroll
  for (int m = 0; m < 16; ++m) {
    const int k = l + LPF * m;
    const float ck = pb[k], cn = pb[N - k];
    const float2 wk = make_float2(a[m].x * ck, a[m].y * ck), wn = make_float2(b[m].x * cn, b[m].y * cn);
    const float2 P = make_float2(wk.x + wn.x, wk.y - wn.y), Q = make_float2(wk.x - wn.x, wk.y + wn.y);
    const float2 w = ut[m * LPF + l];  // exp(-i pi k / N)
    const float2 E = make_float2(fmaf(w.x, Q.x, w.y * Q.y), fmaf(w.x, Q.y, -w.y * Q.x));  // conj(w) Q
    z[m] = make_float2(P.x - E.y, -(P.y + E.x));  // conj(P + i E)
    pz[m] = make_float2(P.x + E.y, P.y - E.x);    // P - i E = 2 conj Z[N - k]
  }
  const float ch = pb[N / 2];
  const float2 zh = make_float2(2.f * h.x * ch, 2.f * h.y * ch);  // element N/2 (lane 0): 2 conj Z[N/2] = 2 W_{N/2}
#pragma unroll
  for (int m = 0; m < 16; ++m) {
    float2 rv;
    rv.x = __shfl_sync(0xffffffffu, pz[m].x, src_lane);
    rv.y = __shfl_sync(0xffffffffu, pz[m].y, src_lane);
    if (l == 0) rv = (m < 15) ? pz[m + 1] : zh;
    z[31 - m] = rv;
  }
  __syncwarp();  // every lane has read its weights: pb becomes the exchange plane
  spectral::warp_fft<LOG2N>(z, pb, tw, l);
  if (live) {
    float* o = ghat + ((size_t)item * n_fr + i) * FRAME;
#pragma unroll
    for (int m = 0; m < 16; ++m) {  // elements e < 128: samples 2e, 2e + 1 < 256; h = conj(out) / 2
      const int n = 2 * (l + LPF * m);
      *reinterpret_cast<float2*>(o + n) = make_float2(0.5f * z[m].x * win[n], -0.5f * z[m].y * win[n + 1]);
    }
  }
}

// 3. dL/dy: the adjoint of the silence removal, a gather.  Sample q lies in frames f = q / 128 and f - 1; for each of
//    them that was kept (position j) it reads the removed signal's r[p], p = 128 j + q - s_j, whose gradient is the sum
//    of the <= 2 STOI frames i < M covering p.  Samples of dropped frames only get exactly 0, as do short items.
__global__ void __launch_bounds__(THREADS)
unframe_kernel(const float* __restrict__ ghat, int64_t n10, int n_fr, const int32_t* __restrict__ count,
               const int32_t* __restrict__ pos, float* __restrict__ gy) {
  __shared__ float win[FRAME];
  for (int n = threadIdx.x; n < FRAME; n += THREADS) win[n] = (float)hann(n);
  __syncthreads();
  const int item = blockIdx.y;
  const int64_t q = (int64_t)blockIdx.x * THREADS + threadIdx.x;
  if (q >= n10) return;
  const int M = __ldg(count + item) - 1;
  const float* gi = ghat + (size_t)item * n_fr * FRAME;
  float acc = 0.f;
  if (M >= SEG) {
    const int f = (int)(q / HOP);
    for (int ff = f - 1; ff <= f; ++ff) {
      if (ff < 0 || ff >= n_fr) continue;
      const int j = __ldg(pos + (size_t)item * n_fr + ff);
      if (j < 0) continue;
      const int o = (int)(q - (int64_t)ff * HOP);
      const int p = j * HOP + o, i1 = p / HOP;
      float gr = 0.f;
      if (i1 >= 1 && i1 - 1 < M) gr += __ldg(gi + (size_t)(i1 - 1) * FRAME + p - (i1 - 1) * HOP);
      if (i1 < M) gr += __ldg(gi + (size_t)i1 * FRAME + p - i1 * HOP);
      acc = fmaf(win[o], gr, acc);
    }
  }
  gy[(size_t)item * n10 + q] = acc;
}

__host__ __device__ __forceinline__ int64_t floor_div(int64_t a, int64_t b) {  // b > 0
  return a >= 0 ? a / b : -((-a + b - 1) / b);
}

// 4. the transpose of resample_kernel's zero-padded polyphase FIR, a gather over the outputs that read input n:
//    gmono[n] = sum_m taps[m down + half - n up] gy[m] (float64 taps and accumulation), then grad[b][c][n] = gmono / C
__global__ void __launch_bounds__(THREADS)
resample_bwd_kernel(const float* __restrict__ gy, int C, int64_t T, const double* __restrict__ taps, int n_taps, int up,
                    int down, int64_t n10, int tiles, float* __restrict__ grad) {
  B2A_DYN_SMEM(smem);
  float* gs = reinterpret_cast<float*>(smem);
  const int item = blockIdx.x / tiles, tile = blockIdx.x - item * tiles;
  const int64_t half = (n_taps - 1) / 2;
  const int64_t n0 = (int64_t)tile * OUT_PER_CTA;
  const int64_t n_end = min(n0 + OUT_PER_CTA, T);
  const int64_t mlo = max(floor_div(n0 * up - half + down - 1, down), (int64_t)0);  // first output the tile reads
  const int64_t mhi = min(floor_div((n_end - 1) * up - half + n_taps - 1, down), n10 - 1);
  const float* g = gy + (size_t)item * n10;
  for (int64_t m = mlo + threadIdx.x; m <= mhi; m += THREADS) gs[m - mlo] = __ldg(g + m);
  __syncthreads();
#pragma unroll
  for (int j = 0; j < OPT; ++j) {
    const int64_t n = n0 + threadIdx.x + (int64_t)THREADS * j;
    if (n >= n_end) break;
    const int64_t a = n * up - half;
    const int64_t m0 = max(floor_div(a + down - 1, down), mlo);
    double acc = 0.0;
    int64_t t = m0 * down - a;
    for (int64_t m = m0; m <= mhi && t < n_taps; ++m, t += down) acc = fma((double)gs[m - mlo], __ldg(taps + t), acc);
    const float v = (float)(acc / C);
    for (int c = 0; c < C; ++c) grad[((size_t)item * C + c) * T + n] = v;
  }
}

struct Layout {
  int64_t n10, n_fr;
  size_t off_energy, off_kept, off_count, off_tob, bytes;
};

inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

inline int64_t out_len(int64_t T, int up, int down) {
  return (int64_t)(((__int128)T * up + down - 1) / down);  // ceil(T up / down), resample_poly's length
}

inline Layout layout(int64_t B, int64_t T, int up, int down) {
  Layout L;
  L.n10 = out_len(T, up, down);
  L.n_fr = L.n10 > FRAME ? (L.n10 - FRAME + HOP - 1) / HOP : 0;  // len(range(0, n10 - 256, 128))
  size_t o = align256((size_t)2 * B * L.n10 * sizeof(float));
  L.off_energy = o;
  o = align256(o + (size_t)B * L.n_fr * sizeof(double));
  L.off_kept = o;
  o = align256(o + (size_t)B * L.n_fr * sizeof(int32_t));
  L.off_count = o;
  o = align256(o + (size_t)B * sizeof(int32_t));
  L.off_tob = o;
  L.bytes = o + (size_t)2 * B * NBAND * L.n_fr * sizeof(float);
  return L;
}

// backward scratch: cells [B][n_fr][15][30] float, Gbar [B][15][n_fr] float64, frame -> kept position [B][n_fr] int32,
// ghat [B][n_fr][256] float, dL/dy [B][n10] float
struct BwdLayout {
  size_t off_gbar, off_pos, off_ghat, off_gy, bytes;
};

inline BwdLayout bwd_layout(int64_t B, const Layout& L) {
  BwdLayout W;
  size_t o = align256((size_t)B * L.n_fr * NBAND * SEG * sizeof(float));
  W.off_gbar = o;
  o = align256(o + (size_t)B * NBAND * L.n_fr * sizeof(double));
  W.off_pos = o;
  o = align256(o + (size_t)B * L.n_fr * sizeof(int32_t));
  W.off_ghat = o;
  o = align256(o + (size_t)B * L.n_fr * FRAME * sizeof(float));
  W.off_gy = o;
  W.bytes = o + (size_t)B * L.n10 * sizeof(float);
  return W;
}

// shared memory of resample_bwd_kernel: the outputs m that one tile of OUT_PER_CTA inputs reads
inline size_t resample_bwd_smem(int n_taps, int up, int down) {
  return (size_t)((((int64_t)(OUT_PER_CTA - 1) * up + n_taps - 1) / down) + 2) * sizeof(float);
}

}  // namespace stoi
}  // namespace b2a

extern "C" size_t b2a_stoi_workspace_bytes(int64_t batch, int64_t T, int up, int down) {
  if (batch < 1 || T < 1 || up < 1 || down < 1) return 0;
  return b2a::stoi::layout(batch, T, up, down).bytes;
}

extern "C" int b2a_stoi_f32(const float* est, const float* ref, int64_t batch, int channels, int64_t T, int extended,
                            const double* taps, int n_taps, int up, int down, double* out, int32_t* kept_out,
                            int32_t* short_out, void* ws, size_t ws_bytes, void* stream) {
  using namespace b2a::stoi;
  B2A_REQUIRE(est && ref && taps && out && kept_out && short_out && ws, B2A_E_INVALID, "stoi: null pointer");
  B2A_REQUIRE(batch >= 1 && channels >= 1 && T >= 1 && up >= 1 && down >= 1 && n_taps >= 1, B2A_E_INVALID,
              "stoi: bad argument");
  B2A_REQUIRE(n_taps % 2 == 1, B2A_E_INVALID, "stoi: the resampling filter needs an odd number of taps (got %d)",
              n_taps);
  B2A_REQUIRE(T < ((int64_t)1 << 31) / channels, B2A_E_UNSUPPORTED, "stoi: items longer than 2^31 samples");
  const Layout L = layout(batch, T, up, down);
  B2A_REQUIRE(L.n_fr >= 1, B2A_E_INVALID, "stoi: the signal has no full 256-sample frame at 10 kHz (%lld samples)",
              (long long)L.n10);
  B2A_REQUIRE(L.n10 < ((int64_t)1 << 31), B2A_E_UNSUPPORTED, "stoi: items longer than 2^31 samples at 10 kHz");
  B2A_REQUIRE(ws_bytes >= L.bytes, B2A_E_INVALID, "stoi: workspace of %zu bytes, %zu needed", ws_bytes, L.bytes);
  const int KP = (n_taps + up - 1) / up;
  const size_t span_max = (size_t)(((int64_t)(OUT_PER_CTA - 1) * down) / up) + 2 + KP;
  const size_t smem = span_max * sizeof(float);
  B2A_REQUIRE(smem <= 200 * 1024, B2A_E_UNSUPPORTED, "stoi: resampling %d/%d needs %zu bytes of shared memory", up,
              down, smem);
  const int64_t tiles = (L.n10 + OUT_PER_CTA - 1) / OUT_PER_CTA;
  B2A_REQUIRE(2 * batch * tiles < (int64_t)2147483647 && batch < 65536, B2A_E_UNSUPPORTED, "stoi: grid too large");
  unsigned char* w = static_cast<unsigned char*>(ws);
  float* sig10 = reinterpret_cast<float*>(w);
  double* energy = reinterpret_cast<double*>(w + L.off_energy);
  int32_t* kept = reinterpret_cast<int32_t*>(w + L.off_kept);
  int32_t* count = reinterpret_cast<int32_t*>(w + L.off_count);
  float* tob = reinterpret_cast<float*>(w + L.off_tob);

  B2A_CUDA_OK(cudaFuncSetAttribute(resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  B2A_LAUNCH(resample_kernel, dim3((unsigned)(2 * batch * tiles)), dim3(THREADS), smem, stream, est, ref, (int)batch,
             channels, T, taps, n_taps, up, down, KP, L.n10, (int)tiles, sig10);
  B2A_LAUNCH(mask_kernel, dim3((unsigned)batch), dim3(THREADS), 0, stream, sig10 + (size_t)batch * L.n10, L.n10,
             (int)L.n_fr, energy, kept, count);
  if (L.n_fr >= 2) {  // at most n_fr - 1 STFT frames per item
    const unsigned ftiles = (unsigned)((L.n_fr - 1 + FRAMES_PER_CTA - 1) / FRAMES_PER_CTA);
    B2A_LAUNCH(band_kernel, dim3(ftiles, (unsigned)batch), dim3(THREADS), 0, stream, sig10, (int)batch, L.n10,
               (int)L.n_fr, kept, count, tob);
  }
  B2A_LAUNCH(score_kernel, dim3((unsigned)batch), dim3(THREADS), 0, stream, tob, (int)batch, (int)L.n_fr, count,
             extended, out, kept_out, short_out);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" size_t b2a_stoi_backward_workspace_bytes(int64_t batch, int64_t T, int up, int down) {
  if (batch < 1 || T < 1 || up < 1 || down < 1) return 0;
  return b2a::stoi::bwd_layout(batch, b2a::stoi::layout(batch, T, up, down)).bytes;
}

extern "C" int b2a_stoi_backward_f32(const double* grad_score, const void* fwd_ws, size_t fwd_ws_bytes, int64_t batch,
                                     int channels, int64_t T, int extended, const double* taps, int n_taps, int up,
                                     int down, float* grad_est, void* ws, size_t ws_bytes, void* stream) {
  using namespace b2a::stoi;
  B2A_REQUIRE(grad_score && fwd_ws && taps && grad_est && ws, B2A_E_INVALID, "stoi_backward: null pointer");
  B2A_REQUIRE(batch >= 1 && channels >= 1 && T >= 1 && up >= 1 && down >= 1 && n_taps >= 1, B2A_E_INVALID,
              "stoi_backward: bad argument");
  B2A_REQUIRE(n_taps % 2 == 1, B2A_E_INVALID,
              "stoi_backward: the resampling filter needs an odd number of taps (got %d)", n_taps);
  B2A_REQUIRE(T < ((int64_t)1 << 31) / channels, B2A_E_UNSUPPORTED, "stoi_backward: items longer than 2^31 samples");
  const Layout L = layout(batch, T, up, down);
  B2A_REQUIRE(L.n_fr >= 1, B2A_E_INVALID,
              "stoi_backward: the signal has no full 256-sample frame at 10 kHz (%lld samples)", (long long)L.n10);
  B2A_REQUIRE(L.n10 < ((int64_t)1 << 31), B2A_E_UNSUPPORTED,
              "stoi_backward: items longer than 2^31 samples at 10 kHz");
  B2A_REQUIRE(fwd_ws_bytes >= L.bytes, B2A_E_INVALID, "stoi_backward: forward workspace of %zu bytes, %zu needed",
              fwd_ws_bytes, L.bytes);
  const BwdLayout W = bwd_layout(batch, L);
  B2A_REQUIRE(ws_bytes >= W.bytes, B2A_E_INVALID, "stoi_backward: workspace of %zu bytes, %zu needed", ws_bytes,
              W.bytes);
  const size_t smem = resample_bwd_smem(n_taps, up, down);
  B2A_REQUIRE(smem <= 200 * 1024, B2A_E_UNSUPPORTED, "stoi_backward: resampling %d/%d needs %zu bytes of shared memory",
              up, down, smem);
  const int64_t tiles = (T + OUT_PER_CTA - 1) / OUT_PER_CTA;
  B2A_REQUIRE(batch * tiles < (int64_t)2147483647 && batch < 65536, B2A_E_UNSUPPORTED, "stoi_backward: grid too large");
  const unsigned char* f = static_cast<const unsigned char*>(fwd_ws);
  const float* sig10 = reinterpret_cast<const float*>(f);
  const int32_t* kept = reinterpret_cast<const int32_t*>(f + L.off_kept);
  const int32_t* count = reinterpret_cast<const int32_t*>(f + L.off_count);
  const float* tob = reinterpret_cast<const float*>(f + L.off_tob);
  unsigned char* w = static_cast<unsigned char*>(ws);
  float* cell = reinterpret_cast<float*>(w);
  double* gbar = reinterpret_cast<double*>(w + W.off_gbar);
  int32_t* pos = reinterpret_cast<int32_t*>(w + W.off_pos);
  float* ghat = reinterpret_cast<float*>(w + W.off_ghat);
  float* gy = reinterpret_cast<float*>(w + W.off_gy);

  B2A_LAUNCH(score_bwd_kernel, dim3((unsigned)batch), dim3(THREADS), 0, stream, grad_score, tob, (int)batch,
             (int)L.n_fr, kept, count, extended, cell, gbar, pos);
  if (L.n_fr >= 2) {  // as in the forward: with one frame at 10 kHz no item has an STFT frame
    const unsigned ftiles = (unsigned)((L.n_fr - 1 + FRAMES_PER_CTA - 1) / FRAMES_PER_CTA);
    B2A_LAUNCH(band_bwd_kernel, dim3(ftiles, (unsigned)batch), dim3(THREADS), 0, stream, sig10, L.n10, (int)L.n_fr,
               kept, count, tob, gbar, ghat);
  }
  B2A_LAUNCH(unframe_kernel, dim3((unsigned)((L.n10 + THREADS - 1) / THREADS), (unsigned)batch), dim3(THREADS), 0,
             stream, ghat, L.n10, (int)L.n_fr, count, pos, gy);
  B2A_CUDA_OK(cudaFuncSetAttribute(resample_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  B2A_LAUNCH(resample_bwd_kernel, dim3((unsigned)(batch * tiles)), dim3(THREADS), smem, stream, gy, channels, T, taps,
             n_taps, up, down, L.n10, (int)tiles, grad_est);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}
