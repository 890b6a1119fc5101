// grad_internal.h -- the pieces of the STFT / inverse STFT kernels that other translation units reuse: the forward
// routes of b2a_spectral_f32 (spectral.cu), the inverse routes of b2a_istft_f32 (istft.cu) and the backward passes
// (grad.cu).
#pragma once
#include "b2a_common.h"

namespace b2a {
namespace istft {
// The fused inverse of istft.cu (b2a_istft_f32's arguments).  adjoint = 1: the STFT's adjoint instead -- bin weights 1
// (not c_k / n_fft) and no envelope division, so out[i] = sum over frames of w[n] sum_k Re(X_k e^{2 pi i kn / n_fft}).
int run(const float* spec, int64_t rows, int64_t n_frames, int n_fft, int hop, const float* window, int pad_frames,
        int64_t start, int64_t out_len, float* out, int adjoint, void* stream);
}  // namespace istft

namespace large {
// The STFT of b2a_spectral_f32 on B2A_ROUTE_LARGE (its framing arguments) -> stft_out [rows, n_fft/2+1, n_frames].
int stft(const float* x, int64_t rows, int64_t T, int n_fft, int hop, const float* window, int pad, int right_pad,
         int pad_mode, int drop_edge, float* stft_out, void* stream);
// b2a_istft_f32 on B2A_ROUTE_LARGE: inverse_frames into ws (rows * n_frames * n_fft floats), then dft.cu's fold.
int istft(const float* spec, int64_t rows, int64_t n_frames, int n_fft, int hop, const float* window, int pad_frames,
          int64_t start, int64_t out_len, float* out, void* ws, size_t ws_bytes, void* stream);
// Windowed inverse frames of fft_large.cu -> frames [rows, n_frames, n_fft] (n_fft 4096 .. 32768); adjoint as above.
int inverse_frames(const float* spec, int64_t rows, int64_t n_frames, int n_fft, const float* window, float* frames,
                   int adjoint, void* stream);
// Forward FFT of raw (un-centred) frames: frame f covers x-coordinates [f hop + origin, + n_fft), zeros outside [0, T).
int forward_raw(const float* x, int64_t rows, int64_t T, int n_fft, int hop, const float* window, int64_t origin,
                int64_t n_frames, float* out, void* stream);
}  // namespace large

namespace dft {
// The STFT of b2a_spectral_f32 on B2A_ROUTE_DENSE, with the kind 0 matrix instead of the window.
int stft(const float* x, int64_t rows, int64_t T, int n_fft, int hop, const float* matrix, int pad, int right_pad,
         int pad_mode, int drop_edge, float* stft_out, void* stream);
// |X| -> banded mel -> post-op of a materialised STFT [rows, F, n_frames] (b2a_spectral_f32's mel arguments).
int mel_from_stft(const float* stft, int64_t rows, int F, int64_t n_frames, const float* mel_fb, const int32_t* mel_lo,
                  const int32_t* mel_hi, int n_mels, int post, float post_eps, float post_power, float* mel_out,
                  void* stream);
// b2a_istft_f32 on B2A_ROUTE_DENSE (also runs n_fft 32 and 4096): inverse_frames with the kind 1 matrix into ws, then
// the fold.
int istft(const float* spec, int64_t rows, int64_t n_frames, int n_fft, int hop, const float* window,
          const float* imatrix, int pad_frames, int64_t start, int64_t out_len, float* out, void* ws, size_t ws_bytes,
          void* stream);
// Dense inverse frames of dft.cu with a kind 1 (inverse) or kind 2 (adjoint) matrix -> frames [rows, n_frames, n_fft].
int inverse_frames(const float* spec, int64_t rows, int64_t n_frames, int n_fft, const float* imatrix, float* frames,
                   void* stream);
// Dense forward DFT (kind 0 matrix) of raw frames, framed as large::forward_raw.
int forward_raw(const float* x, int64_t rows, int64_t T, int n_fft, int hop, const float* matrix, int64_t origin,
                int64_t n_frames, float* out, void* stream);
}  // namespace dft
}  // namespace b2a
