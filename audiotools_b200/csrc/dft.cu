// dft.cu -- STFT / inverse STFT for window lengths the FFT kernels do not cover, as dense DFTs on sm_90a.
//
// AudioSignal.stft accepts ANY window_length (ref:audiotools/core/audio_signal.py:1123-1212 -> torch.stft), e.g. the
// 400 / 480 / 1200-sample (25 ms) windows of speech front-ends; spectral.cu covers the powers of two in [32, 4096].
// Everything else runs here: the windowed real DFT of all frames of a batch is ONE real x complex matrix product
//     X[f][k] = sum_n x[(f + drop_edge) hop + origin + n] . M[n][k],     M[n][k] = w[n] exp(-2 pi i nk / n_fft)
// -- genuinely GEMM-shaped (64 k frames x 400 x 201 at 64 x 10 s @ 16 kHz / hop 160), computed in FP32 so that the
// 1e-4 parity bar holds without operand splitting: a register-tiled product of complex multiply-accumulates on
// (re, im) pairs (fma2: the sample broadcast to both halves, the (re, im) of M as the pair).  The framing is
// implicit (A is read straight from the waveform with torch's two nested paddings resolved per sample, bit-exact in
// the frame / sample indexing like spectral.cu), M is built once per (n_fft, window) by dft_matrix_kernel with the
// angle reduced in integers (nk mod n_fft) and evaluated in float64.
//
// The inverse (AudioSignal.istft, ref:audiotools/core/audio_signal.py:1214-1296 -> torch.istft) is the transposed
// product  y[f][n] = sum_k Re(X[f][k] . conj-weighted M)  followed by the overlap-add / envelope fold; it also serves
// the two power-of-two sizes istft.cu does not (32, 4096), which removes the last torch.istft delegation.
//
// Tile: 64 frames x 64 outputs per CTA (256 threads, 4 x 4 micro-tile), reduction in chunks of 16 through
// double-buffered shared memory; 3 (forward) / 4 (inverse) 128-bit shared loads per 16 complex fma2.
#include "b2a_common.h"
#include "dft_internal.h"
#include "grad_internal.h"
#include "spectral_internal.h"

namespace b2a {
namespace dft {

constexpr int BM = 64;   // frames per CTA tile
constexpr int BN = 64;   // outputs (bins / samples) per CTA tile
constexpr int BK = 16;   // reduction chunk
constexpr int ASTR = BM + 4;  // padded row of the real A tile (floats): 16 B aligned, conflict-free

__host__ __device__ inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

// ---------------------------------------------------------------------------------------------
// matrices.  forward: Mt[n][k] (k fastest, [Np][Fp]) = w[n] (cos, -sin)(2 pi nk / N), zero padded.
//            inverse: Mi[k][n] (n fastest, [Fq][Np]) = c_k / N . w[n] (cos, -sin)(2 pi nk / N), c = 1 for k = 0 and
//            k = N/2 (N even), else 2 (the Hermitian half folded in); y[n] = sum_k Xr Mi.x + Xi Mi.y.
//            adjoint (kind 2): the inverse layout with weight 1 on every bin -- the STFT's adjoint (gradient wrt x).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void unit(int n, int k, int N, double* cs, double* sn) {
  const long long r = ((long long)n * (long long)k) % (long long)N;
#ifdef B2A_SIM
  const double a = 2.0 * 3.14159265358979323846 * (double)r / (double)N;
  *cs = cos(a); *sn = sin(a);
#else
  sincospi(2.0 * (double)r / (double)N, sn, cs);
#endif
}

__global__ void __launch_bounds__(256) dft_matrix_kernel(const float* __restrict__ window, int N, int F, int Np, int Fp,
                                                         int Fq, int inverse, float2* __restrict__ M) {
  const long long total = inverse ? (long long)Fq * Np : (long long)Np * Fp;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int n, k;
    if (inverse) { k = (int)(i / Np); n = (int)(i - (long long)k * Np); }
    else { n = (int)(i / Fp); k = (int)(i - (long long)n * Fp); }
    float2 v = make_float2(0.f, 0.f);
    if (n < N && k < F) {
      double cs, sn;
      unit(n, k, N, &cs, &sn);
      double s = (double)window[n];
      if (inverse == 1) s *= ((k == 0 || 2 * k == N) ? 1.0 : 2.0) / (double)N;
      v = make_float2((float)(s * cs), (float)(-s * sn));
    }
    M[i] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// forward: stft_out[row][k][f] = sum_n x(row, f, n) Mt[n][k]
// ---------------------------------------------------------------------------------------------
struct FwdParams {
  const float* x;
  const float2* Mt;
  float2* out;
  int rows, T, n_fft, hop, pad, right_pad, pad_mode, drop_edge, n_frames, F, Np, Fp, tiles_f;
  int origin, center;  // frame f starts at x-coordinate (f + drop_edge) hop + origin; center: src_index's framing flag
};

__global__ void __launch_bounds__(256) dft_forward_kernel(FwdParams p) {
  __shared__ __align__(16) float As[2][BK][ASTR];
  __shared__ __align__(16) float2 Bs[2][BK][BN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int row = blockIdx.x / p.tiles_f, f0 = (blockIdx.x - row * p.tiles_f) * BM;
  const int k0 = blockIdx.y * BN;
  const float* xr = p.x + (size_t)row * (size_t)p.T;
  const int origin = p.origin;
  // interior tile: every sample the tile touches is inside [0, T) -> no index resolution
  const long long lo = (long long)(f0 + p.drop_edge) * p.hop + origin;
  const long long hi = (long long)(min(f0 + BM, p.n_frames) - 1 + p.drop_edge) * p.hop + origin + p.n_fft;
  const bool interior = lo >= 0 && hi <= (long long)p.T && f0 + BM <= p.n_frames;

  // loader roles
  const int a_nn = tid & 15, a_ff = tid >> 4;   // A: 16 consecutive samples of frames a_ff + 16 j
  const int b_kk = tid & 63, b_nn = tid >> 6;   // B: 64 consecutive bins of samples b_nn + 4 j
  float ra[4];
  float2 rb[4];
  auto load = [&](int n0) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int ff = a_ff + 16 * j, n = n0 + a_nn;
      float v = 0.f;
      if (interior) {
        if (n < p.n_fft) v = __ldg(xr + (size_t)((long long)(f0 + ff + p.drop_edge) * p.hop + origin + n));
      } else if (n < p.n_fft && f0 + ff < p.n_frames) {
        const long long w = (long long)(f0 + ff + p.drop_edge) * p.hop + origin + n;
        const int u = spectral::src_index((int)w, p.T, p.pad, p.right_pad, p.pad_mode, p.center);
        if (u >= 0) v = __ldg(xr + u);
      }
      ra[j] = v;
      rb[j] = __ldg(p.Mt + (size_t)(n0 + b_nn + 4 * j) * p.Fp + k0 + b_kk);
    }
  };
  auto store = [&](int buf) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      As[buf][a_nn][a_ff + 16 * j] = ra[j];
      Bs[buf][b_nn + 4 * j][b_kk] = rb[j];
    }
  };

  float2 acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = make_float2(0.f, 0.f);

  load(0);
  store(0);
  __syncthreads();
  const int nchunk = p.Np / BK;
  for (int c = 0; c < nchunk; ++c) {
    const int buf = c & 1;
    if (c + 1 < nchunk) load((c + 1) * BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&As[buf][kk][4 * tx]);
      const float4 b01 = *reinterpret_cast<const float4*>(&Bs[buf][kk][4 * ty]);
      const float4 b23 = *reinterpret_cast<const float4*>(&Bs[buf][kk][4 * ty + 2]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float2 bv[4] = {make_float2(b01.x, b01.y), make_float2(b01.z, b01.w), make_float2(b23.x, b23.y),
                            make_float2(b23.z, b23.w)};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fma2(bcast2(av[i]), bv[j], acc[i][j]);
    }
    if (c + 1 < nchunk) store(buf ^ 1);
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int k = k0 + 4 * ty + j;
    if (k >= p.F) continue;
    float2* o = p.out + ((size_t)row * p.F + k) * (size_t)p.n_frames;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int f = f0 + 4 * tx + i;
      if (f < p.n_frames) o[f] = acc[i][j];
    }
  }
}

// ---------------------------------------------------------------------------------------------
// |X| -> banded mel -> post-op from a materialised STFT (the fused kernel of spectral.cu does this in-flight for the
// power-of-two windows): lane = frame (coalesced along the frame axis), warp = filter.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) mel_from_stft_kernel(const float2* __restrict__ spec, int F, int n_frames,
                                                            const float* __restrict__ fb,
                                                            const int32_t* __restrict__ lo, const int32_t* __restrict__ hi,
                                                            int n_mels, int post, float eps, float power,
                                                            float* __restrict__ out) {
  const int f = blockIdx.x * 32 + (threadIdx.x & 31);
  const int m = blockIdx.y * 8 + (threadIdx.x >> 5);
  const int row = blockIdx.z;
  if (f >= n_frames || m >= n_mels) return;
  const float2* s = spec + (size_t)row * F * (size_t)n_frames + f;
  const float* w = fb + (size_t)m * F;
  float acc = 0.f;
  for (int k = __ldg(lo + m); k < __ldg(hi + m); ++k) {
    const float2 v = s[(size_t)k * n_frames];
    acc = fmaf(__ldg(w + k), sqrtf(fmaf(v.x, v.x, v.y * v.y)), acc);
  }
  if (post == B2A_POST_LOG10) {
    float c = fmaxf(acc, eps);
    c = (power == 2.0f) ? c * c : powf(c, power);
    acc = log10f(c);
  } else if (post == B2A_POST_LN) {
    acc = logf(acc + eps);
  }
  out[((size_t)row * n_mels + m) * (size_t)n_frames + f] = acc;
}

// ---------------------------------------------------------------------------------------------
// mfcc: out[row][j][n] = sum_m dct[m][j] * logmel[row][m][n]   (ref:audiotools/core/audio_signal.py:1420-1426:
// `mel_spectrogram.transpose(-1, -2) @ create_dct(n_mfcc, n_mels, "ortho")` transposed back: a cuBLAS batched GEMM there).
// lane = frame (coalesced along n), each thread keeps up to 32 coefficients in registers, the DCT basis in shared memory.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) mel_dct_kernel(const float* __restrict__ logmel, const float* __restrict__ dct,
                                                      int n_mels, int n_mfcc, int n_frames, float* __restrict__ out) {
  B2A_DYN_SMEM(smem);
  float* sd = reinterpret_cast<float*>(smem);  // [n_mels][n_mfcc]
  for (int i = threadIdx.x; i < n_mels * n_mfcc; i += blockDim.x) sd[i] = __ldg(dct + i);
  __syncthreads();
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int row = blockIdx.y;
  if (n >= n_frames) return;
  const float* in = logmel + (size_t)row * n_mels * (size_t)n_frames + n;
  float* o = out + (size_t)row * n_mfcc * (size_t)n_frames + n;
  for (int j0 = 0; j0 < n_mfcc; j0 += 32) {
    float acc[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] = 0.f;
    const int nj = min(32, n_mfcc - j0);
    for (int m = 0; m < n_mels; ++m) {
      const float v = in[(size_t)m * n_frames];
      const float* d = sd + m * n_mfcc + j0;
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j < nj) acc[j] = fmaf(v, d[j], acc[j]);
    }
#pragma unroll
    for (int j = 0; j < 32; ++j)
      if (j < nj) o[(size_t)(j0 + j) * n_frames] = acc[j];
  }
}

// ---------------------------------------------------------------------------------------------
// inverse: frames[row][f][n] = sum_k spec[row][k][f].re Mi[k][n].x + spec[row][k][f].im Mi[k][n].y  (window applied)
// ---------------------------------------------------------------------------------------------
struct InvParams {
  const float2* spec;
  const float2* Mi;
  float* frames;
  int rows, n_frames, n_fft, F, Fq, Np, tiles_f;
};

__global__ void __launch_bounds__(256) dft_inverse_kernel(InvParams p) {
  __shared__ __align__(16) float2 As[2][BK][BM + 2];
  __shared__ __align__(16) float2 Bs[2][BK][BN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;  // tx: samples 4 tx .. +3, ty: frames 4 ty .. +3
  const int row = blockIdx.x / p.tiles_f, f0 = (blockIdx.x - row * p.tiles_f) * BM;
  const int n0 = blockIdx.y * BN;
  const float2* sr = p.spec + (size_t)row * p.F * (size_t)p.n_frames;
  const int l_i = tid & 63, l_k = tid >> 6;  // loaders: 64 consecutive frames / samples of bins l_k + 4 j
  float2 ra[4], rb[4];
  auto load = [&](int k0) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + l_k + 4 * j;
      ra[j] = (k < p.F && f0 + l_i < p.n_frames) ? sr[(size_t)k * p.n_frames + f0 + l_i] : make_float2(0.f, 0.f);
      rb[j] = __ldg(p.Mi + (size_t)k * p.Np + n0 + l_i);
    }
  };
  auto store = [&](int buf) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      As[buf][l_k + 4 * j][l_i] = ra[j];
      Bs[buf][l_k + 4 * j][l_i] = rb[j];
    }
  };
  float2 acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = make_float2(0.f, 0.f);
  load(0);
  store(0);
  __syncthreads();
  const int nchunk = p.Fq / BK;
  for (int c = 0; c < nchunk; ++c) {
    const int buf = c & 1;
    if (c + 1 < nchunk) load((c + 1) * BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      const float4 a01 = *reinterpret_cast<const float4*>(&As[buf][kk][4 * ty]);
      const float4 a23 = *reinterpret_cast<const float4*>(&As[buf][kk][4 * ty + 2]);
      const float4 b01 = *reinterpret_cast<const float4*>(&Bs[buf][kk][4 * tx]);
      const float4 b23 = *reinterpret_cast<const float4*>(&Bs[buf][kk][4 * tx + 2]);
      const float2 av[4] = {make_float2(a01.x, a01.y), make_float2(a01.z, a01.w), make_float2(a23.x, a23.y),
                            make_float2(a23.z, a23.w)};
      const float2 bv[4] = {make_float2(b01.x, b01.y), make_float2(b01.z, b01.w), make_float2(b23.x, b23.y),
                            make_float2(b23.z, b23.w)};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fma2(av[i], bv[j], acc[i][j]);
    }
    if (c + 1 < nchunk) store(buf ^ 1);
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int f = f0 + 4 * ty + i;
    if (f >= p.n_frames) continue;
    float* o = p.frames + ((size_t)row * p.n_frames + f) * (size_t)p.n_fft;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + 4 * tx + j;
      if (n < p.n_fft) o[n] = acc[i][j].x + acc[i][j].y;
    }
  }
}

// overlap-add (gather) + window envelope: out[row][i] = y[start + i] / env[start + i] for start + i < expected, else 0
__global__ void __launch_bounds__(256) fold_kernel(const float* __restrict__ frames, const float* __restrict__ window,
                                                   int n_frames, int n_fft, int hop, int pad_frames, long long start,
                                                   long long out_len, long long expected, int divide,
                                                   float* __restrict__ out) {
  const int row = blockIdx.y;
  const float* fr = frames + (size_t)row * n_frames * (size_t)n_fft;
  float* o = out + (size_t)row * (size_t)out_len;
  const int NP = n_frames + 2 * pad_frames;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < out_len; i += (long long)gridDim.x * blockDim.x) {
    const long long t = start + i;
    float v = 0.f;
    if (t < expected) {
      long long g_hi = t / hop;                       // last frame starting at or before t
      long long g_lo = (t - n_fft + hop) / hop;       // first frame that still covers t: ceil((t - n_fft + 1) / hop)
      if (t - n_fft + 1 <= 0) g_lo = 0;
      if (g_hi > NP - 1) g_hi = NP - 1;
      float acc = 0.f, env = 0.f;
      for (long long g = g_lo; g <= g_hi; ++g) {
        const int n = (int)(t - g * hop);
        if (n < 0 || n >= n_fft) continue;
        const float wv = __ldg(window + n);
        env = fmaf(wv, wv, env);
        const long long f = g - pad_frames;
        if (f >= 0 && f < n_frames) acc += fr[(size_t)f * n_fft + n];
      }
      v = divide ? acc / env : acc;
    }
    o[i] = v;
  }
}

}  // namespace dft
}  // namespace b2a

using namespace b2a::dft;

static inline int np_of(int n_fft) { return round_up(n_fft, BN); }          // samples, padded (multiple of BN >= BK)
static inline int fp_of(int n_fft) { return round_up(n_fft / 2 + 1, BN); }  // bins, padded for the forward tile
static inline int fq_of(int n_fft) { return round_up(n_fft / 2 + 1, BK); }  // bins, padded for the inverse reduction

// the window lengths of the dense DFT: any n_fft in [2, 8192], powers of two included (the inverse: 1 <= hop <= n_fft)
static bool supported(int n_fft, int hop) { return n_fft >= 2 && n_fft <= 8192 && hop >= 1; }

extern "C" size_t b2a_dft_matrix_floats(int n_fft, int inverse) {
  if (n_fft < 2 || n_fft > 8192 || inverse < 0 || inverse > 2) return 0;
  return 2 * (inverse ? (size_t)fq_of(n_fft) * np_of(n_fft) : (size_t)np_of(n_fft) * fp_of(n_fft));
}

extern "C" int b2a_dft_matrix_f32(const float* window, int n_fft, int inverse, float* matrix, void* stream) {
  B2A_REQUIRE(window && matrix, B2A_E_INVALID, "dft_matrix: null pointer");
  B2A_REQUIRE(n_fft >= 2 && n_fft <= 8192, B2A_E_UNSUPPORTED, "dft_matrix: window_length %d (2..8192)", n_fft);
  B2A_REQUIRE(inverse >= 0 && inverse <= 2, B2A_E_INVALID, "dft_matrix: kind %d (0 forward, 1 inverse, 2 adjoint)", inverse);
  const int F = n_fft / 2 + 1;
  const size_t total = b2a_dft_matrix_floats(n_fft, inverse) / 2;
  const unsigned grid = (unsigned)((total + 255) / 256 < 4096 ? (total + 255) / 256 : 4096);
  B2A_LAUNCH(dft_matrix_kernel, dim3(grid), dim3(256), 0, stream, window, n_fft, F, np_of(n_fft), fp_of(n_fft),
             fq_of(n_fft), inverse, reinterpret_cast<float2*>(matrix));
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

static int launch_forward(FwdParams& p, int64_t rows, void* stream);

int b2a::dft::stft(const float* x, int64_t rows, int64_t T, int n_fft, int hop, const float* matrix, int pad,
                   int right_pad, int pad_mode, int drop_edge, float* stft_out, void* stream) {
  B2A_REQUIRE(x && matrix && stft_out, B2A_E_INVALID, "stft_dense: null pointer");
  B2A_REQUIRE(rows >= 1 && T >= 1, B2A_E_INVALID, "stft_dense: empty input");
  B2A_REQUIRE(T < (int64_t)1 << 30, B2A_E_UNSUPPORTED, "stft_dense: rows longer than 2^30 samples");
  B2A_REQUIRE(supported(n_fft, hop), B2A_E_UNSUPPORTED, "stft_dense: window_length %d hop %d", n_fft, hop);
  int64_t nfr;
  const int rc = b2a::spectral::check_framing("stft_dense", T, n_fft, hop, pad, right_pad, pad_mode, drop_edge, &nfr);
  if (rc != B2A_OK) return rc;
  FwdParams p;
  p.x = x; p.Mt = reinterpret_cast<const float2*>(matrix); p.out = reinterpret_cast<float2*>(stft_out);
  p.rows = (int)rows; p.T = (int)T; p.n_fft = n_fft; p.hop = hop; p.pad = pad; p.right_pad = right_pad;
  p.pad_mode = pad_mode; p.drop_edge = drop_edge; p.n_frames = (int)nfr; p.F = n_fft / 2 + 1;
  p.origin = -(n_fft / 2) - pad; p.center = 1;
  return launch_forward(p, rows, stream);
}

static int launch_forward(FwdParams& p, int64_t rows, void* stream) {
  p.Np = np_of(p.n_fft); p.Fp = fp_of(p.n_fft); p.tiles_f = (p.n_frames + BM - 1) / BM;
  const int64_t gx = rows * p.tiles_f;
  B2A_REQUIRE(gx < (int64_t)2147483647, B2A_E_UNSUPPORTED, "stft_dense: too many tiles");
  B2A_LAUNCH(dft_forward_kernel, dim3((unsigned)gx, (unsigned)(p.Fp / BN)), dim3(256), 0, stream, p);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

int b2a::dft::forward_raw(const float* x, int64_t rows, int64_t T, int n_fft, int hop, const float* matrix,
                          int64_t origin, int64_t n_frames, float* out, void* stream) {
  B2A_REQUIRE(supported(n_fft, hop), B2A_E_UNSUPPORTED, "stft_dense: window_length %d hop %d", n_fft, hop);
  B2A_REQUIRE(T < (int64_t)1 << 30 && n_frames < (int64_t)1 << 30 && origin > -((int64_t)1 << 30) &&
                  origin < ((int64_t)1 << 30),
              B2A_E_UNSUPPORTED, "stft_dense: too large");
  FwdParams p;
  memset(&p, 0, sizeof(p));
  p.x = x; p.Mt = reinterpret_cast<const float2*>(matrix); p.out = reinterpret_cast<float2*>(out);
  p.rows = (int)rows; p.T = (int)T; p.n_fft = n_fft; p.hop = hop; p.pad_mode = B2A_PAD_CONSTANT;
  p.n_frames = (int)n_frames; p.F = n_fft / 2 + 1; p.origin = (int)origin; p.center = 0;
  return launch_forward(p, rows, stream);
}

int b2a::dft::mel_from_stft(const float* stft, int64_t rows, int F, int64_t n_frames, const float* mel_fb,
                            const int32_t* mel_lo, const int32_t* mel_hi, int n_mels, int post, float post_eps,
                            float post_power, float* mel_out, void* stream) {
  B2A_REQUIRE(stft && mel_fb && mel_lo && mel_hi && mel_out, B2A_E_INVALID, "mel_from_stft: null pointer");
  B2A_REQUIRE(rows >= 1 && rows <= 65535 && F >= 1 && n_frames >= 1 && n_mels >= 1, B2A_E_INVALID,
              "mel_from_stft: bad shape");
  B2A_REQUIRE(post >= 0 && post <= 2, B2A_E_INVALID, "mel_from_stft: post-op %d", post);
  B2A_LAUNCH(mel_from_stft_kernel, dim3((unsigned)((n_frames + 31) / 32), (unsigned)((n_mels + 7) / 8), (unsigned)rows),
             dim3(256), 0, stream, reinterpret_cast<const float2*>(stft), F, (int)n_frames, mel_fb, mel_lo, mel_hi, n_mels,
             post, post_eps, post_power, mel_out);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

int b2a::dft::istft(const float* spec, int64_t rows, int64_t n_frames, int n_fft, int hop, const float* window,
                    const float* imatrix, int pad_frames, int64_t start, int64_t out_len, float* out, void* ws,
                    size_t ws_bytes, void* stream) {
  B2A_REQUIRE(spec && window && imatrix && out && ws, B2A_E_INVALID, "istft_dense: null pointer");
  B2A_REQUIRE(rows >= 1 && rows <= 65535 && n_frames >= 1 && out_len >= 1 && pad_frames >= 0 && start >= 0, B2A_E_INVALID,
              "istft_dense: bad argument");
  B2A_REQUIRE(supported(n_fft, hop) && hop <= n_fft, B2A_E_UNSUPPORTED, "istft_dense: n_fft=%d hop=%d", n_fft, hop);
  B2A_REQUIRE(ws_bytes >= (size_t)rows * (size_t)n_frames * (size_t)n_fft * sizeof(float), B2A_E_INVALID,
              "istft_dense: workspace too small");
  B2A_REQUIRE(((uintptr_t)spec & 7) == 0, B2A_E_INVALID, "istft_dense: spectra must be 8-byte aligned");
  float* frames = reinterpret_cast<float*>(ws);
  const int rc = inverse_frames(spec, rows, n_frames, n_fft, imatrix, frames, stream);
  if (rc != B2A_OK) return rc;
  return launch_fold(frames, window, rows, (int)n_frames, n_fft, hop, pad_frames, start, out_len, 1, out, stream);
}

int b2a::dft::inverse_frames(const float* spec, int64_t rows, int64_t n_frames, int n_fft, const float* imatrix,
                             float* frames, void* stream) {
  InvParams p;
  p.spec = reinterpret_cast<const float2*>(spec); p.Mi = reinterpret_cast<const float2*>(imatrix);
  p.frames = frames;
  p.rows = (int)rows; p.n_frames = (int)n_frames; p.n_fft = n_fft; p.F = n_fft / 2 + 1; p.Fq = fq_of(n_fft);
  p.Np = np_of(n_fft); p.tiles_f = (int)((n_frames + BM - 1) / BM);
  const int64_t gx = rows * p.tiles_f;
  B2A_REQUIRE(gx < (int64_t)2147483647, B2A_E_UNSUPPORTED, "istft_dense: too many tiles");
  B2A_LAUNCH(dft_inverse_kernel, dim3((unsigned)gx, (unsigned)(p.Np / BN)), dim3(256), 0, stream, p);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

int b2a::dft::launch_fold(const float* frames, const float* window, int64_t rows, int n_frames, int n_fft, int hop,
                          int pad_frames, int64_t start, int64_t out_len, int divide, float* out, void* stream) {
  const long long expected = (long long)(n_frames + 2 * pad_frames - 1) * hop + n_fft;
  const long long want = (out_len + 255) / 256;
  B2A_LAUNCH(fold_kernel, dim3((unsigned)(want < 2048 ? want : 2048), (unsigned)rows), dim3(256), 0, stream, frames,
             window, n_frames, n_fft, hop, pad_frames, (long long)start, (long long)out_len, expected, divide, out);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" int b2a_mel_dct_f32(const float* logmel, int64_t rows, int n_mels, int64_t n_frames, const float* dct, int n_mfcc,
                               float* out, void* stream) {
  B2A_REQUIRE(logmel && dct && out, B2A_E_INVALID, "mel_dct: null pointer");
  // the kernel's frame index is an int that runs to the end of the last 128-frame tile
  B2A_REQUIRE(rows >= 1 && rows <= 65535 && n_mels >= 1 && n_mfcc >= 1 && n_frames >= 1 && n_frames <= INT_MAX - 127,
              B2A_E_INVALID, "mel_dct: bad shape");
  const size_t smem = (size_t)n_mels * n_mfcc * sizeof(float);
  B2A_REQUIRE(smem <= 200 * 1024, B2A_E_UNSUPPORTED, "mel_dct: %d x %d basis does not fit shared memory", n_mels, n_mfcc);
  B2A_CUDA_OK(cudaFuncSetAttribute(mel_dct_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  B2A_LAUNCH(mel_dct_kernel, dim3((unsigned)((n_frames + 127) / 128), (unsigned)rows), dim3(128), smem, stream, logmel, dct,
             n_mels, n_mfcc, (int)n_frames, out);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}
