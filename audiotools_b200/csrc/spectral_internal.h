// spectral_internal.h -- entry points of spectral.cu used by other translation units of libb2a.
#pragma once
#include "b2a_common.h"

namespace b2a {
namespace spectral {

struct Params {
  const float* x;
  const float* window;
  const float* gain;
  float* y_out;
  const float* mel_fb;
  const int32_t* mel_lo;
  const int32_t* mel_hi;
  float* mel_out;
  float2* stft_out;
  int rows, T, n_fft, hop, pad, right_pad, pad_mode, drop_edge;
  int n_frames, n_tiles, n_mels, rows_per_gain, post;
  int mel_packed_len;  // sum over filters of the 4-aligned band widths (0: read weights from global)
  int off_mpk, off_mseg;
  // framing: frame n of a row starts at x-coordinate (n + drop_edge)*hop + origin (+ row_origin[row]);
  // center = 1: torch.stft(center=True) semantics (reflect about the F.pad-ed signal), 0: raw
  int center, origin;
  const int32_t* row_origin;
  float post_eps, post_power;
  int span;  // (FR-1)*hop + n_fft
  // shared memory offsets (bytes)
  int off_win, off_tw, off_ut, off_buf, off_mag, off_mel, smem_bytes;
  int xb_stride;   // floats per frame slot of the exchange / |X| buffer (WPlan::XB, or 2N+4 when the STFT is staged)
  int stage_stft;  // STFT-only launch: complex frames are parked in their slots and written with frame-contiguous runs
};

// index of sample `w` (in un-padded x coordinates, may be outside [0,T)) after torch's two
// paddings; -1 => zero.   ref:audiotools/core/audio_signal.py:1192-1202
#define B2A_PAD_CIRCULAR 3  // internal (FFT convolution): index modulo T

__device__ __forceinline__ int src_index(int w, int T, int pad, int right_pad, int pad_mode, int center = 1) {
  int u = w;
  if (center) {
    const int Lp = T + 2 * pad + right_pad;
    int v = w + pad;  // position in the F.pad-ed signal
    if (v < 0) v = -v;                       // torch.stft(center=True): reflect, no edge repeat
    else if (v >= Lp) v = 2 * (Lp - 1) - v;
    if (v < 0 || v >= Lp) return -1;         // only reachable from frames past the end (never stored)
    u = v - pad;
  }
  if (u >= 0 && u < T) return u;
  if (pad_mode == B2A_PAD_REFLECT) u = u < 0 ? -u : 2 * (T - 1) - u;
  else if (pad_mode == B2A_PAD_REPLICATE) u = u < 0 ? 0 : T - 1;
  else if (pad_mode == B2A_PAD_CIRCULAR) { u %= T; if (u < 0) u += T; }
  else return -1;
  return (u >= 0 && u < T) ? u : -1;
}

// ---- asynchronous staging (warp kernels of spectral.cu and loss.cu): raw x -> shared memory by the TMA engine, so
// that the copy overlaps the per-CTA table set-up and, later, the previous tile's FFTs; the gain is applied after the
// (linear) mel projection and the scaled waveform x*g is written back from shared memory.
// Returns true when the span was handed to the TMA engine (completion on `bar`), false when it was staged with
// cp.async / plain stores (completion by cp_async_wait_all + the CTA barrier).  The choice is CTA-uniform.
__device__ __forceinline__ bool stage_span_async(const Params& p, float* sp, int row, int ws, unsigned long long* bar) {
  const int tid = threadIdx.x, T = p.T, span = p.span;
  const float* xr = p.x + (size_t)row * (size_t)T;
  const bool interior = (ws >= 0) && (ws + span <= T);
  if (interior && ((((uintptr_t)(xr + ws)) & 15) == 0) && ((span & 3) == 0)) {
    // interior tile: its (FR-1)*hop + n_fft samples are one contiguous, 16 B aligned run of the row -> ONE bulk copy
    if (tid == 0) tma_load_1d(sp, xr + ws, (unsigned)span * 4u, bar);
    return true;
  } else if (interior) {
    for (int i = tid; i < span; i += (int)blockDim.x) sp[i] = __ldg(xr + ws + i);
  } else {
    for (int i = tid; i < span; i += (int)blockDim.x) {
      const int u = src_index(ws + i, T, p.pad, p.right_pad, p.pad_mode, p.center);
      sp[i] = (u >= 0) ? __ldg(xr + u) : 0.f;
    }
  }
  return false;
}

// banded mel projection of filter m: sum over its band k in [mel_lo[m], mel_hi[m]) of fb[m][k] mag[k], ascending k, so
// that the fused loss projects exactly as the forward kernels do
__device__ __forceinline__ float mel_band(const float* fb, const int32_t* mel_lo, const int32_t* mel_hi, int F, int m,
                                          const float* mag) {
  const int lo = __ldg(mel_lo + m), hi = __ldg(mel_hi + m);
  const float* w = fb + (size_t)m * F;
  float acc = 0.f;
  for (int k = lo; k < hi; ++k) acc = fmaf(__ldg(w + k), mag[k], acc);
  return acc;
}

// torch's stft(center=True) framing of the explicitly padded signal (F.pad(pad, pad + right_pad, pad_mode), then the
// centre reflect), shared by every STFT entry point: B2A_OK and the frame count, or the error code with the message
// prefixed by `who`.  Which kernel family runs a window length is b2a_stft_route (include/b2a.h), defined beside it.
int check_framing(const char* who, int64_t T, int n_fft, int hop, int pad, int right_pad, int pad_mode, int drop_edge,
                  int64_t* n_frames);

// Forward real FFT of raw (un-centred) blocks: block n of row r covers x-coordinates
// [n*hop + origin + row_origin[r], +n_fft), out of range samples resolved by pad_mode
// (B2A_PAD_CONSTANT zero / B2A_PAD_REPLICATE / 3 = circular).  out: [rows, n_fft/2+1, n_frames] (re,im).
// n_fft: power of two in [64, 2048] (the warp kernel).
int frames_fft(const float* x, int rows, int T, int n_fft, int hop, const float* window, int origin,
               const int32_t* row_origin, int pad_mode, int n_frames, float2* out, void* stream);

}  // namespace spectral
}  // namespace b2a
