// grad.cu -- backward passes of the spectral front end on sm_90a: the gradients of AudioSignal.stft, istft and
// mel_spectrogram / mfcc (ref:audiotools/core/audio_signal.py:1123-1296, 1333-1426; differentiable through torch
// there, ref:tests/core/test_grad.py).  Conventions follow torch: a complex output's incoming gradient is
// G = dL/dRe + i dL/dIm.  With theta = 2 pi k n / n_fft:
//
//   STFT adjoint   g_frame[n] = w[n] sum_k Re(G_k e^{i theta}) for every kept frame, overlap-added WITHOUT envelope
//                  division over the padded range, then folded back through torch's two nested paddings (pad adjoint
//                  below).  Relative to the inverse transform only the bin weights change (1 instead of c_k / n_fft),
//                  so each forward route's inverse machinery computes it in an adjoint mode:
//                  istft_kernel (64 .. 2048), istft_large_kernel + fold (4096 .. 32768), dense adjoint matrix + fold.
//   iSTFT adjoint  u = g / env placed on the overlap-add range, framed with the window, forward real FFT, bin k scaled
//                  by c_k / n_fft (c = 1 at DC / Nyquist, else 2), imaginary parts of DC / Nyquist zero (a C2R
//                  transform ignores them).  u is zero outside the output range, so the frames are raw (un-centred)
//                  windows of u with zeros outside: the forward kernels' raw framing (frames_fft, forward_raw).
//   mel            mel = fb |X|:  dX = (fb^T dmel') X / |X|  (0 where |X| = 0, as torch's abs), dmel' = dmel times the
//                  post-op's derivative: POST_LOG10 power / (ln10 mel) where mel >= eps (else 0), POST_LN 1 / (mel + eps).
//
// Everything is deterministic: no atomics; every sum runs in a fixed order.
#include "b2a_common.h"
#include "dft_internal.h"
#include "grad_internal.h"
#include "spectral_internal.h"

namespace b2a {
namespace grad {

// ---------------------------------------------------------------------------------------------
// pad adjoint: gx[u] = sum of gp over every padded position whose sample (spectral::src_index) is u.
// gp covers x-coordinates w in [-(half + pad), T + pad + right_pad + half): gp[j] <-> w = j - half - pad.
// The preimages of u are enumerated by inverting the two paddings (explicit F.pad mode, then the centre reflect) and
// each candidate is kept only if src_index maps it to u, so the forward framing and this fold cannot disagree.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float centre_preimages(const float* gp, int u, int u2, int T, int half, int pad,
                                                  int right_pad, int pad_mode) {
  const int Lp = T + 2 * pad + right_pad;
  const int v = u2 + pad;  // position in the F.pad-ed signal, [0, Lp)
  float acc = 0.f;
  int cand[3] = {v, -v, 2 * (Lp - 1) - v};
  const bool ok[3] = {true, v > 0 && v <= half, v < Lp - 1 && 2 * (Lp - 1) - v < Lp + half};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    if (!ok[c]) continue;
    const int w = cand[c] - pad;
    if (spectral::src_index(w, T, pad, right_pad, pad_mode, 1) == u) acc += gp[cand[c] + half];
  }
  return acc;
}

__global__ void __launch_bounds__(256) pad_adjoint_kernel(const float* __restrict__ gp, long long Lpp, int T, int half,
                                                          int pad, int right_pad, int pad_mode, float* __restrict__ gx) {
  const int row = blockIdx.y;
  const float* g = gp + (size_t)row * (size_t)Lpp;
  float* o = gx + (size_t)row * (size_t)T;
  const int lo_int = half + pad, hi_int = T - 2 - half - pad - right_pad;  // u strictly inside: its own sample only
  for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < T; u += gridDim.x * blockDim.x) {
    if (u > lo_int && u < hi_int) {
      o[u] = g[u + half + pad];
      continue;
    }
    // explicit-pad preimages u2 in [-pad, T + pad + right_pad), in a fixed order
    float acc = centre_preimages(g, u, u, T, half, pad, right_pad, pad_mode);
    if (pad_mode == B2A_PAD_REFLECT) {
      if (u > 0 && u <= pad) acc += centre_preimages(g, u, -u, T, half, pad, right_pad, pad_mode);
      if (u < T - 1 && 2 * (T - 1) - u < T + pad + right_pad)
        acc += centre_preimages(g, u, 2 * (T - 1) - u, T, half, pad, right_pad, pad_mode);
    } else if (pad_mode == B2A_PAD_REPLICATE) {
      if (u == 0)
        for (int u2 = -1; u2 >= -pad; --u2) acc += centre_preimages(g, u, u2, T, half, pad, right_pad, pad_mode);
      if (u == T - 1)
        for (int u2 = T; u2 < T + pad + right_pad; ++u2)
          acc += centre_preimages(g, u, u2, T, half, pad, right_pad, pad_mode);
    }
    o[u] = acc;
  }
}

// ---------------------------------------------------------------------------------------------
// iSTFT backward, step 1: u[row][i] = g[row][i] / env[start + i] for start + i < expected, else 0 (the envelope of
// fold_kernel: every one of the NP = n_frames + 2 pad_frames frames counts).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) envelope_divide_kernel(const float* __restrict__ g, const float* __restrict__ window,
                                                              int NP, int n_fft, int hop, long long start, long long out_len,
                                                              long long expected, float* __restrict__ u) {
  const int row = blockIdx.y;
  const float* gr = g + (size_t)row * (size_t)out_len;
  float* ur = u + (size_t)row * (size_t)out_len;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < out_len; i += (long long)gridDim.x * blockDim.x) {
    const long long t = start + i;
    float v = 0.f;
    if (t < expected) {
      long long f_hi = t / hop;
      long long f_lo = (t - n_fft + hop) / hop;
      if (t - n_fft + 1 <= 0) f_lo = 0;
      if (f_hi > NP - 1) f_hi = NP - 1;
      float env = 0.f;
      for (long long f = f_lo; f <= f_hi; ++f) {
        const int n = (int)(t - f * hop);
        if (n < 0 || n >= n_fft) continue;
        const float wv = __ldg(window + n);
        env = fmaf(wv, wv, env);
      }
      v = gr[i] / env;
    }
    ur[i] = v;
  }
}

// iSTFT backward, step 3: spec[row][k][f] *= c_k / n_fft; the imaginary parts of DC / Nyquist are zero
__global__ void __launch_bounds__(256) bin_scale_kernel(float2* __restrict__ spec, long long total, int F, int n_frames,
                                                        int n_fft) {
  const float inv = 1.0f / (float)n_fft;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)((i / n_frames) % F);
    float2 v = spec[i];
    if (k == 0 || 2 * k == n_fft) {
      v = make_float2(v.x * inv, 0.f);
    } else {
      v = make_float2(v.x * (2.f * inv), v.y * (2.f * inv));
    }
    spec[i] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// mel backward: one CTA per (row, 32-frame tile), lane = frame (coalesced along the frame axis).
//   1. warp w recomputes mel[m] for m = w, w + 8, ... from the banded filters, applies the post-op derivative to the
//      incoming gradient and parks it in shared memory [n_mels][32];
//   2. warp w takes bins k = w, w + 8, ...: d|X|_k = sum over the filters m in [bin_lo[k], bin_hi[k]) whose band holds
//      k of fb[m][k] dmel'[m] (the transposed banded projection, ascending m), dX_k = d|X|_k X_k / |X_k|.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) mel_backward_kernel(const float2* __restrict__ spec, int F, int n_frames,
                                                           const float* __restrict__ fb, const int32_t* __restrict__ lo,
                                                           const int32_t* __restrict__ hi, int n_mels,
                                                           const int32_t* __restrict__ bin_lo,
                                                           const int32_t* __restrict__ bin_hi, int post, float eps,
                                                           float power, const float* __restrict__ gmel,
                                                           float2* __restrict__ gspec) {
  B2A_DYN_SMEM(smem);
  float* ps = reinterpret_cast<float*>(smem);  // [n_mels][32]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int f = blockIdx.x * 32 + lane;
  const int row = blockIdx.y;
  const bool live = f < n_frames;
  const float2* s = spec + (size_t)row * F * (size_t)n_frames + f;
  const float* gm = gmel + (size_t)row * n_mels * (size_t)n_frames + f;
  for (int m = warp; m < n_mels; m += 8) {
    float pm = 0.f;
    if (live) {
      const float* w = fb + (size_t)m * F;
      float acc = 0.f;
      for (int k = __ldg(lo + m); k < __ldg(hi + m); ++k) {
        const float2 v = s[(size_t)k * n_frames];
        acc = fmaf(__ldg(w + k), sqrtf(fmaf(v.x, v.x, v.y * v.y)), acc);
      }
      const float g = gm[(size_t)m * n_frames];
      if (post == B2A_POST_LOG10) pm = acc >= eps ? g * power / (2.302585092994046f * acc) : 0.f;
      else if (post == B2A_POST_LN) pm = g / (acc + eps);
      else pm = g;
    }
    ps[m * 32 + lane] = pm;
  }
  __syncthreads();
  if (!live) return;
  float2* o = gspec + (size_t)row * F * (size_t)n_frames + f;
  for (int k = warp; k < F; k += 8) {
    float d = 0.f;
    for (int m = __ldg(bin_lo + k); m < __ldg(bin_hi + k); ++m)
      if (__ldg(lo + m) <= k && k < __ldg(hi + m)) d = fmaf(__ldg(fb + (size_t)m * F + k), ps[m * 32 + lane], d);
    const float2 v = s[(size_t)k * n_frames];
    const float mag = sqrtf(fmaf(v.x, v.x, v.y * v.y));
    float2 r = make_float2(0.f, 0.f);
    if (mag > 0.f) {
      const float q = d / mag;
      r = make_float2(v.x * q, v.y * q);
    }
    o[(size_t)k * n_frames] = r;
  }
}

static inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

static unsigned grid_for(long long n) {
  const long long b = (n + 255) / 256;
  return (unsigned)(b < 2048 ? (b > 0 ? b : 1) : 2048);
}

}  // namespace grad
}  // namespace b2a

using namespace b2a::grad;

extern "C" size_t b2a_stft_backward_workspace_bytes(int64_t rows, int64_t T, int n_fft, int hop, int pad, int right_pad,
                                                    int drop_edge) {
  const int r = b2a_stft_route(n_fft, hop, 1);
  const int64_t nfr = b2a_stft_num_frames(T, n_fft, hop, pad, right_pad, drop_edge);
  if (r == B2A_ROUTE_NONE || rows < 1 || nfr < 1) return 0;
  const int64_t Lpp = T + 2 * (int64_t)(n_fft / 2 + pad) + right_pad;
  size_t b = align256((size_t)rows * (size_t)Lpp * sizeof(float));
  if (r != B2A_ROUTE_FFT) b += (size_t)rows * (size_t)nfr * (size_t)n_fft * sizeof(float);
  return b;
}

extern "C" int b2a_stft_backward_f32(const float* grad_spec, int64_t rows, int64_t T, int n_fft, int hop,
                                     const float* window, const float* amatrix, int pad, int right_pad, int pad_mode,
                                     int drop_edge, float* grad_x, void* ws, size_t ws_bytes, void* stream) {
  B2A_REQUIRE(grad_spec && window && grad_x && ws, B2A_E_INVALID, "stft_backward: null pointer");
  B2A_REQUIRE(rows >= 1 && rows <= 65535 && T >= 1 && T < ((int64_t)1 << 30), B2A_E_INVALID, "stft_backward: bad shape");
  const int r = b2a_stft_route(n_fft, hop, 1);
  B2A_REQUIRE(r != B2A_ROUTE_NONE, B2A_E_UNSUPPORTED,
              "stft_backward: window_length %d hop %d (hop <= window_length; powers of two up to 32768, any other length "
              "up to 8192)", n_fft, hop);
  B2A_REQUIRE(r != B2A_ROUTE_DENSE || amatrix, B2A_E_INVALID,
              "stft_backward: window_length %d needs the adjoint DFT matrix", n_fft);
  int64_t nfr;
  int rc = b2a::spectral::check_framing("stft_backward", T, n_fft, hop, pad, right_pad, pad_mode, drop_edge, &nfr);
  if (rc != B2A_OK) return rc;
  B2A_REQUIRE(ws_bytes >= b2a_stft_backward_workspace_bytes(rows, T, n_fft, hop, pad, right_pad, drop_edge),
              B2A_E_INVALID, "stft_backward: workspace too small");
  B2A_REQUIRE(((uintptr_t)grad_spec & 7) == 0 && ((uintptr_t)ws & 7) == 0, B2A_E_INVALID,
              "stft_backward: spectra and workspace must be 8-byte aligned");
  const int half = n_fft / 2;
  const int64_t Lpp = T + 2 * ((int64_t)half + pad) + right_pad;  // the padded signal and the centre padding
  float* gp = reinterpret_cast<float*>(ws);
  // 1. adjoint transform + overlap-add (no envelope) over the whole padded range; the dropped frames are zero frames
  if (r == B2A_ROUTE_FFT) {
    rc = b2a::istft::run(grad_spec, rows, nfr, n_fft, hop, window, drop_edge, 0, Lpp, gp, 1, stream);
  } else {
    float* frames = reinterpret_cast<float*>(reinterpret_cast<char*>(ws) + align256((size_t)rows * Lpp * sizeof(float)));
    rc = (r == B2A_ROUTE_LARGE) ? b2a::large::inverse_frames(grad_spec, rows, nfr, n_fft, window, frames, 1, stream)
                                : b2a::dft::inverse_frames(grad_spec, rows, nfr, n_fft, amatrix, frames, stream);
    if (rc == B2A_OK)
      rc = b2a::dft::launch_fold(frames, window, rows, (int)nfr, n_fft, hop, drop_edge, 0, Lpp, 0, gp, stream);
  }
  if (rc != B2A_OK) return rc;
  // 2. fold the padded range back onto the signal
  B2A_LAUNCH(pad_adjoint_kernel, dim3(grid_for(T), (unsigned)rows), dim3(256), 0, stream, gp, (long long)Lpp, (int)T,
             half, pad, right_pad, pad_mode, grad_x);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" size_t b2a_istft_backward_workspace_bytes(int64_t rows, int64_t out_len) {
  if (rows < 1 || out_len < 1) return 0;
  return (size_t)rows * (size_t)out_len * sizeof(float);
}

extern "C" int b2a_istft_backward_f32(const float* grad_out, int64_t rows, int64_t n_frames, int n_fft, int hop,
                                      const float* window, const float* matrix, int pad_frames, int64_t start,
                                      int64_t out_len, float* grad_spec, void* ws, size_t ws_bytes, void* stream) {
  B2A_REQUIRE(grad_out && window && grad_spec && ws, B2A_E_INVALID, "istft_backward: null pointer");
  B2A_REQUIRE(rows >= 1 && rows <= 65535 && n_frames >= 1 && out_len >= 1 && out_len < ((int64_t)1 << 30) &&
                  pad_frames >= 0 && start >= 0,
              B2A_E_INVALID, "istft_backward: bad argument");
  const int r = b2a_stft_route(n_fft, hop, 1);
  B2A_REQUIRE(r != B2A_ROUTE_NONE, B2A_E_UNSUPPORTED,
              "istft_backward: window_length %d hop %d (hop <= window_length; powers of two up to 32768, any other "
              "length up to 8192)", n_fft, hop);
  B2A_REQUIRE(r != B2A_ROUTE_DENSE || matrix, B2A_E_INVALID,
              "istft_backward: window_length %d needs the forward DFT matrix", n_fft);
  B2A_REQUIRE(ws_bytes >= b2a_istft_backward_workspace_bytes(rows, out_len), B2A_E_INVALID,
              "istft_backward: workspace too small");
  B2A_REQUIRE(((uintptr_t)grad_spec & 7) == 0, B2A_E_INVALID, "istft_backward: spectra must be 8-byte aligned");
  const int NP = (int)(n_frames + 2 * pad_frames);
  const long long expected = (long long)(NP - 1) * hop + n_fft;
  float* u = reinterpret_cast<float*>(ws);
  B2A_LAUNCH(envelope_divide_kernel, dim3(grid_for(out_len), (unsigned)rows), dim3(256), 0, stream, grad_out, window, NP,
             n_fft, hop, (long long)start, (long long)out_len, expected, u);
  B2A_CUDA_OK(cudaGetLastError());
  // frame f (padded frame f + pad_frames) covers overlap-add coordinates [(f + pad_frames) hop, + n_fft), i.e. u from
  // (f + pad_frames) hop - start on: raw framing with that origin, zeros outside [0, out_len)
  const int64_t origin = (int64_t)pad_frames * hop - start;
  int rc;
  if (r == B2A_ROUTE_FFT) {
    B2A_REQUIRE(origin > -((int64_t)1 << 30) && origin < ((int64_t)1 << 30) && n_frames < ((int64_t)1 << 30),
                B2A_E_UNSUPPORTED, "istft_backward: too large");
    rc = b2a::spectral::frames_fft(u, (int)rows, (int)out_len, n_fft, hop, window, (int)origin, nullptr,
                                   B2A_PAD_CONSTANT, (int)n_frames, reinterpret_cast<float2*>(grad_spec), stream);
  } else if (r == B2A_ROUTE_LARGE) {
    rc = b2a::large::forward_raw(u, rows, out_len, n_fft, hop, window, origin, n_frames, grad_spec, stream);
  } else {
    rc = b2a::dft::forward_raw(u, rows, out_len, n_fft, hop, matrix, origin, n_frames, grad_spec, stream);
  }
  if (rc != B2A_OK) return rc;
  const int F = n_fft / 2 + 1;
  const long long total = (long long)rows * F * n_frames;
  B2A_LAUNCH(bin_scale_kernel, dim3(grid_for(total)), dim3(256), 0, stream, reinterpret_cast<float2*>(grad_spec), total, F,
             (int)n_frames, n_fft);
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}

extern "C" int b2a_mel_backward_f32(const float* stft, int64_t rows, int F, int64_t n_frames, const float* mel_fb,
                                    const int32_t* mel_lo, const int32_t* mel_hi, int n_mels, const int32_t* bin_lo,
                                    const int32_t* bin_hi, int post, float post_eps, float post_power,
                                    const float* grad_mel, float* grad_stft, void* stream) {
  B2A_REQUIRE(stft && mel_fb && mel_lo && mel_hi && bin_lo && bin_hi && grad_mel && grad_stft, B2A_E_INVALID,
              "mel_backward: null pointer");
  B2A_REQUIRE(rows >= 1 && rows <= 65535 && F >= 1 && n_frames >= 1 && n_frames < ((int64_t)1 << 30) && n_mels >= 1,
              B2A_E_INVALID, "mel_backward: bad shape");
  B2A_REQUIRE(post >= 0 && post <= 2, B2A_E_INVALID, "mel_backward: post-op %d", post);
  B2A_REQUIRE(((uintptr_t)stft & 7) == 0 && ((uintptr_t)grad_stft & 7) == 0, B2A_E_INVALID,
              "mel_backward: spectra must be 8-byte aligned");
  const size_t smem = (size_t)n_mels * 32 * sizeof(float);
  B2A_REQUIRE(smem <= 200 * 1024, B2A_E_UNSUPPORTED, "mel_backward: %d mel filters do not fit shared memory", n_mels);
  B2A_CUDA_OK(cudaFuncSetAttribute(mel_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  B2A_LAUNCH(mel_backward_kernel, dim3((unsigned)((n_frames + 31) / 32), (unsigned)rows), dim3(256), smem, stream,
             reinterpret_cast<const float2*>(stft), F, (int)n_frames, mel_fb, mel_lo, mel_hi, n_mels, bin_lo, bin_hi, post,
             post_eps, post_power, grad_mel, reinterpret_cast<float2*>(grad_stft));
  B2A_CUDA_OK(cudaGetLastError());
  return B2A_OK;
}
