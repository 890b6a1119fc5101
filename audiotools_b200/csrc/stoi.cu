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
    emax = fmax(emax, ef);
  }
  if (lane == 0) red[warp] = emax;
  __syncthreads();  // also orders the energies written above before the reads below
  emax = red[0];
  for (int i = 1; i < THREADS / 32; ++i) emax = fmax(emax, red[i]);
  // 2. keep flags -> exclusive scan -> indices of the kept frames, in order
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
    float2 a[16], b[16], h;
    spectral::untangle<LOG2N>(z, ut, l, src_lane, a, b, h);
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
        my += fmin((double)yr[t] * c, xv * clip);
      }
      mx /= SEG;
      my /= SEG;
      double sxy = 0.0, sx2 = 0.0, sy2 = 0.0;
      for (int t = 0; t < SEG; ++t) {
        const double xv = xr[t];
        const double dx = xv - mx, dy = fmin((double)yr[t] * c, xv * clip) - my;
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
