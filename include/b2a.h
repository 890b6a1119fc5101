/* b2a.h -- C ABI of libb2a.so, the H100-native (sm_90a) engine behind the
 * AudioSignal transform/augment hot path of descriptinc/audiotools.
 *
 * The reference is 100% Python and has NO plugin/FFI interface (SURVEY.md §8b): the
 * "API for this path" is the AudioSignal method surface.  Each entry point below
 * therefore names the reference *method* (file:line under /root/reference) whose
 * device-side work it replaces; audiotools_b200/ (Python, ctypes) keeps the
 * method-level names and semantics on top of it.  INTEGRATION.md shows the binding.
 *
 * Conventions
 *  - plain C types only; every pointer is a DEVICE pointer unless suffixed _h (host);
 *  - the caller owns every buffer (inputs, outputs, workspaces);
 *  - every call is asynchronous on `stream` (a cudaStream_t passed as void*);
 *  - returns 0 on success, <0 on error (B2A_E_*); b2a_last_error() gives the
 *    thread-local message.  Nothing throws, nothing falls back to the CPU.
 *  - waveforms are float32, contiguous [rows, T] with rows = B*C (row = b*C + c).
 */
#ifndef B2A_H_
#define B2A_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2A_VERSION 100 /* 0.1.0 */

#define B2A_OK 0
#define B2A_E_INVALID -1     /* bad argument (the message says which)               */
#define B2A_E_UNSUPPORTED -2 /* valid in the reference, not implemented on device   */
#define B2A_E_CUDA -3        /* a CUDA runtime call / launch failed                 */

/* pad modes of torch.nn.functional.pad used by AudioSignal.stft (padding_type) */
#define B2A_PAD_REFLECT 0
#define B2A_PAD_CONSTANT 1
#define B2A_PAD_REPLICATE 2

/* post-ops fused behind the mel projection */
#define B2A_POST_NONE 0   /* mel                                      audio_signal.py:1367-1368 */
#define B2A_POST_LOG10 1  /* log10(clamp(mel, eps)^power)             metrics/spectral.py:187-190 */
#define B2A_POST_LN 2     /* ln(mel + eps)                            audio_signal.py:1421 (mfcc) */

int b2a_version(void);
const char* b2a_last_error(void);

/* ---- STFT / mel ---------------------------------------------------------------------
 * Replaces the device work of AudioSignal.stft (audiotools/core/audio_signal.py:1123-1212:
 * F.pad(pad, pad+right_pad, padding_type) -> torch.stft(center=True, reflect) -> optional
 * drop of 2+2 edge frames) and AudioSignal.mel_spectrogram (:1333-1369: |X| @ mel_basis.T),
 * fused: framing -> window -> real FFT -> |.| -> banded mel -> post-op, one pass over x.
 *
 *   x        [rows, T]
 *   window   [n_fft]              (AudioSignal.get_window, :1009-1039)
 *   n_fft    power of two in [32, 4096] (b2a_stft_route's B2A_ROUTE_FFT); hop >= 1
 *   pad/right_pad/pad_mode        compute_stft_padding (:1089-1121); 0/0 when !match_stride
 *   drop_edge                     frames dropped at each end (2 when match_stride, else 0)
 *   gain     nullable [rows/rows_per_gain]: x is multiplied by gain[row / rows_per_gain] first
 *            (EffectMixin.normalize's x*gain, effects.py:219) and, if y_out != NULL, the scaled
 *            waveform is written there ([rows, T]) by the same pass.
 *   mel_fb   nullable [n_mels, F] row-major dense filterbank (get_mel_filters, :1298-1331);
 *   mel_lo/mel_hi  [n_mels] int32: mel_fb[m, k] == 0 outside mel_lo[m] <= k < mel_hi[m]
 *            (the caller derives them from the actual non-zeros, so the banded sum equals the
 *            dense matmul exactly for ANY matrix).
 *   mel_packed_len  floats of the kernel's shared-memory band table (0: read the weights from global):
 *            with n4[m] = (ceil4(mel_hi[m]) - floor4(mel_lo[m]))/4, 4 * sum over filters m of
 *            even(max(n4[m'] : m' in {4g .. 4g + 3})) where g = m / 4, even(v) = (v+1) & ~1
 *            (the 4 consecutive filters one warp projects in one step share a trip count; the loop is unrolled by two).
 *   mel_out  nullable [rows, n_mels, n_frames]    stft_out  nullable [rows, F, n_frames] (re,im)
 *   n_frames = 1 + (T + 2*pad + right_pad)/hop - 2*drop_edge,  F = n_fft/2 + 1
 */
int64_t b2a_stft_num_frames(int64_t T, int n_fft, int hop, int pad, int right_pad, int drop_edge);
int b2a_spectral_f32(const float* x, int64_t rows, int64_t T, int n_fft, int hop, const float* window,
                     int pad, int right_pad, int pad_mode, int drop_edge,
                     const float* gain, int rows_per_gain, float* y_out,
                     const float* mel_fb, const int32_t* mel_lo, const int32_t* mel_hi, int n_mels,
                     int mel_packed_len, int post, float post_eps, float post_power,
                     float* mel_out, float* stft_out, void* stream);

/* ---- the one route table: which kernel family runs an STFT of (n_fft, hop) -------------------------------------
 * inverse 0: the forward STFT (b2a_spectral_f32 / b2a_stft_large_f32 / b2a_stft_dense_f32).  inverse 1: b2a_istft_f32
 * and both backward passes, which route by it themselves.  Everything not in the table is B2A_ROUTE_NONE.
 *                      FFT                          LARGE                          DENSE
 *   inverse 0, hop>=1  power of two in [32, 4096]   power of two in [8192, 32768]  any other length in [2, 8192]
 *   inverse 1, hop in  power of two in [64, 2048]   power of two in [4096, 32768]  any other length in [2, 8192]
 *   [1, n_fft]                                                                     (incl. 32) */
#define B2A_ROUTE_NONE 0  /* not supported                                     */
#define B2A_ROUTE_FFT 1   /* spectral.cu (forward) / istft.cu (inverse)        */
#define B2A_ROUTE_LARGE 2 /* fft_large.cu                                      */
#define B2A_ROUTE_DENSE 3 /* dft.cu (needs the b2a_dft_matrix_f32 matrix)      */
int b2a_stft_route(int n_fft, int hop, int inverse);

/* ---- inverse STFT ---------------------------------------------------------------------------------
 * Replaces AudioSignal.istft (audiotools/core/audio_signal.py:1214-1296 -> torch.istft(center=True, onesided,
 * window of n_fft samples)): inverse real FFT of every frame, window, overlap-add, division by the window
 * envelope, on the route b2a_stft_route(n_fft, hop, 1): FFT -> one pass (rows < 2^24); LARGE / DENSE -> the windowed
 * frames of fft_large.cu / dft.cu into ws, then dft.cu's overlap-add fold (rows <= 65535).
 *   spec   [rows, n_fft/2+1, n_frames] complex64 (re,im), 8-byte aligned (the layout b2a_spectral_f32 writes)
 *   matrix nullable; on DENSE the kind 1 matrix of b2a_dft_matrix_f32
 *   pad_frames  zero frames put back on either side (match_stride: 2, :1276-1279); they count in the envelope
 *   start  overlap-add coordinate of out[0]: n_fft/2 (+ the match_stride trim `pad`, :1291-1292)
 *   out    [rows, out_len]; samples at or beyond (n_frames + 2*pad_frames - 1)*hop + n_fft are zero, as torch pads
 *   ws     b2a_istft_workspace_bytes(...) bytes, 8-byte aligned; 0 on FFT, where ws may be NULL
 * The caller checks the envelope (torch raises when its minimum over the kept range is < 1e-11). */
size_t b2a_istft_workspace_bytes(int64_t rows, int64_t n_frames, int n_fft, int hop);
int b2a_istft_f32(const float* spec, int64_t rows, int64_t n_frames, int n_fft, int hop, const float* window,
                  const float* matrix, int pad_frames, int64_t start, int64_t out_len, float* out, void* ws,
                  size_t ws_bytes, void* stream);

/* ---- STFT for ANY window length (dense DFT, csrc/dft.cu) -------------------------------------------------------
 * AudioSignal.stft / istft accept any window_length (audiotools/core/audio_signal.py:1123-1212, 1214-1296 -> torch.stft /
 * torch.istft), e.g. 400 / 480 / 1200-sample speech windows (B2A_ROUTE_DENSE).  Their STFT is ONE real x complex
 * matrix product over all frames of the batch (FP32 FMA):
 *   b2a_dft_matrix_f32     builds the matrix of (n_fft, window) once: inverse 0 -> M[n][k] = w[n] exp(-2 pi i nk/n_fft)
 *                          for b2a_stft_dense_f32, inverse 1 -> c_k/n_fft . w[n] exp(-2 pi i nk/n_fft) (c = 1 for DC and
 *                          Nyquist, else 2) for b2a_istft_f32, inverse 2 -> the layout of 1 with weight 1 on every
 *                          bin for b2a_stft_backward_f32; `matrix`: b2a_dft_matrix_floats(n_fft, inverse)
 *                          floats, 16-byte aligned; angles reduced in integers (nk mod n_fft), evaluated in float64
 *   b2a_stft_dense_f32     the arguments of b2a_spectral_f32 (same framing / padding semantics, bit-exact frame
 *                          indexing) -> stft_out [rows, n_fft/2+1, n_frames] (re,im)
 *   b2a_mel_from_stft_f32  |X| -> banded mel -> post-op from a materialised STFT (AudioSignal.mel_spectrogram :1333-1369
 *                          for the LARGE and DENSE routes; the FFT kernel fuses it) */
size_t b2a_dft_matrix_floats(int n_fft, int inverse);
int b2a_dft_matrix_f32(const float* window, int n_fft, int inverse, float* matrix, void* stream);
int b2a_stft_dense_f32(const float* x, int64_t rows, int64_t T, int n_fft, int hop, const float* matrix,
                       int pad, int right_pad, int pad_mode, int drop_edge, float* stft_out, void* stream);
int b2a_mel_from_stft_f32(const float* stft, int64_t rows, int F, int64_t n_frames, const float* mel_fb,
                          const int32_t* mel_lo, const int32_t* mel_hi, int n_mels, int post, float post_eps,
                          float post_power, float* mel_out, void* stream);
/* AudioSignal.mfcc's `log-mel^T @ create_dct(n_mfcc, n_mels, "ortho")` (audio_signal.py:1420-1426):
 * out[row][j][n] = sum_m dct[m][j] * logmel[row][m][n];  logmel [rows, n_mels, n_frames], dct [n_mels, n_mfcc] row-major. */
int b2a_mel_dct_f32(const float* logmel, int64_t rows, int n_mels, int64_t n_frames, const float* dct, int n_mfcc,
                    float* out, void* stream);

/* ---- STFT for LARGE power-of-two windows (FFT, one CTA per frame, csrc/fft_large.cu) ---------------------------
 * B2A_ROUTE_LARGE: the default window of AudioSignal.stft_params is 2^ceil(log2(0.032 sr)) = 4096 at 88.2 / 96 kHz and
 * 8192 at 176.4 / 192 kHz; 16384 / 32768 serve fine frequency resolution.  FP32; no matrix, no table to build.
 *   b2a_stft_large_f32         the arguments of b2a_stft_dense_f32 with the window instead of the matrix (same framing /
 *                              padding semantics, bit-exact frame indexing) -> stft_out [rows, n_fft/2+1, n_frames] */
int b2a_stft_large_f32(const float* x, int64_t rows, int64_t T, int n_fft, int hop, const float* window, int pad,
                       int right_pad, int pad_mode, int drop_edge, float* stft_out, void* stream);

/* ---- backward passes of the spectral front end (csrc/grad.cu) ---------------------------------------------------
 * Gradients of AudioSignal.stft / istft / mel_spectrogram / mfcc (audiotools/core/audio_signal.py:1123-1296, 1333-1426;
 * differentiable through torch there, tests/core/test_grad.py).  A complex gradient is G = dL/dRe + i dL/dIm (torch's
 * convention); every pass is deterministic (no atomics, fixed summation order).  Both backward passes exist where
 * b2a_stft_route(n_fft, hop, 1) is not B2A_ROUTE_NONE, and run on that route.
 *   b2a_stft_backward_f32        grad_spec [rows, n_fft/2+1, n_frames] (re,im) -> grad_x [rows, T], for the STFT that
 *                                b2a_spectral_f32 / b2a_stft_dense_f32 / b2a_stft_large_f32 computed with the same
 *                                (T, n_fft, hop, window, pad, right_pad, pad_mode, drop_edge): per frame
 *                                w[n] sum_k Re(G_k e^{2 pi i kn/n_fft}), overlap-added without envelope division over the
 *                                padded range, folded back through both paddings (each padded position's gradient is
 *                                added to the sample it was read from).  amatrix: the kind 2 matrix of b2a_dft_matrix_f32,
 *                                required on B2A_ROUTE_DENSE, else unused.
 *                                ws: b2a_stft_backward_workspace_bytes(...) bytes, 8-byte aligned.
 *   b2a_istft_backward_f32       grad_out [rows, out_len] -> grad_spec [rows, n_fft/2+1, n_frames] for the inverse that
 *                                b2a_istft_f32 computed with the same arguments: grad_out / envelope framed with the
 *                                window, forward real FFT, bin k scaled by c_k / n_fft (c = 1 at DC and Nyquist, else
 *                                2), imaginary parts of DC / Nyquist 0.  matrix: the kind 0 (forward) matrix
 *                                of b2a_dft_matrix_f32, required on B2A_ROUTE_DENSE.  ws: b2a_istft_backward_workspace_bytes.
 *   b2a_mel_backward_f32         grad_mel [rows, n_mels, n_frames] -> grad_stft [rows, F, n_frames] (re,im) from the
 *                                complex STFT `stft` the mel came from: recomputes mel from the banded filters, applies the
 *                                post-op's derivative (B2A_POST_LOG10: post_power / (ln10 mel) where mel >= post_eps, else
 *                                0; B2A_POST_LN: 1 / (mel + post_eps)), projects back through fb^T and multiplies by
 *                                X / |X| (0 where |X| = 0).  bin_lo / bin_hi [F] int32: the filters m that may hold bin k
 *                                lie in [bin_lo[k], bin_hi[k]) (mel_lo[m] <= k < mel_hi[m] is checked per filter).
 * The mfcc DCT's backward is b2a_mel_dct_f32 with the transposed basis; the gain's is b2a_gain_f32. */
size_t b2a_stft_backward_workspace_bytes(int64_t rows, int64_t T, int n_fft, int hop, int pad, int right_pad,
                                         int drop_edge);
int b2a_stft_backward_f32(const float* grad_spec, int64_t rows, int64_t T, int n_fft, int hop, const float* window,
                          const float* amatrix, int pad, int right_pad, int pad_mode, int drop_edge, float* grad_x,
                          void* ws, size_t ws_bytes, void* stream);
size_t b2a_istft_backward_workspace_bytes(int64_t rows, int64_t out_len);
int b2a_istft_backward_f32(const float* grad_out, int64_t rows, int64_t n_frames, int n_fft, int hop,
                           const float* window, const float* matrix, int pad_frames, int64_t start, int64_t out_len,
                           float* grad_spec, void* ws, size_t ws_bytes, void* stream);
int b2a_mel_backward_f32(const float* stft, int64_t rows, int F, int64_t n_frames, const float* mel_fb,
                         const int32_t* mel_lo, const int32_t* mel_hi, int n_mels, const int32_t* bin_lo,
                         const int32_t* bin_hi, int post, float post_eps, float post_power, const float* grad_mel,
                         float* grad_stft, void* stream);

/* ---- spectral L1 losses with their gradient (csrc/loss.cu) --------------------------------------------------------
 * One scale of MultiScaleSTFTLoss / MelSpectrogramLoss with loss_fn = nn.L1Loss() (audiotools/metrics/spectral.py:70-95,
 * 159-192) for the estimate x and the target y [rows, T] of the same geometry (the framing arguments of
 * b2a_spectral_f32, no gain), with lg(v) = log10(max(v, clamp_eps)^pow):
 *   mel_fb == NULL   L = log_weight mean |lg|X| - lg|Y|| + mag_weight mean ||X| - |Y||        over [rows, F, n_frames]
 *   mel_fb != NULL   the same over mel = fb |.| [rows, n_mels, n_frames]; mel_lo / mel_hi: the band table of
 *                    b2a_spectral_f32, bin_lo / bin_hi: the transposed one of b2a_mel_backward_f32.
 *   loss_out         one device float, written by a second one-warp launch that adds per-CTA partials in a fixed order
 *                    (float64): no atomics, reruns are bit-identical.
 *   grad_x / grad_y  nullable [rows, F, n_frames] (re,im): dL/dX, dL/dY of the two STFTs with torch's derivatives
 *                    (sign(0) = 0, the gradient passes the clamp where v >= clamp_eps, X / |X| is 0 at X = 0); feed them
 *                    to b2a_stft_backward_f32.  A weight of 0 removes its term and its gradient.
 *   b2a_spectral_loss_supported  (n_fft, hop, n_mels; 0 for the STFT loss): n_fft a power of two in [64, 2048],
 *                                1 <= hop <= n_fft, and the launch fits shared memory.
 *   workspace        b2a_spectral_loss_workspace_bytes(n_fft, hop, n_mels) bytes, 8-byte aligned (the partials). */
int b2a_spectral_loss_supported(int n_fft, int hop, int n_mels);
size_t b2a_spectral_loss_workspace_bytes(int n_fft, int hop, int n_mels);
int b2a_spectral_loss_f32(const float* x, const float* y, int64_t rows, int64_t T, int n_fft, int hop,
                          const float* window, int pad, int right_pad, int pad_mode, int drop_edge, const float* mel_fb,
                          const int32_t* mel_lo, const int32_t* mel_hi, const int32_t* bin_lo, const int32_t* bin_hi,
                          int n_mels, float clamp_eps, float pow, float log_weight, float mag_weight, float* loss_out,
                          float* grad_x, float* grad_y, void* workspace, size_t workspace_bytes, void* stream);

/* ---- SpecAugment band masks on a complex STFT, in place -------------------------------------------------
 * DSPMixin.mask_frequencies / mask_timesteps (audiotools/core/dsp.py:217-306): cells whose axis value v satisfies
 * lo[item] <= v < hi[item] (float32, as the reference compares) become fill = val * exp(1j * val); all other
 * cells are left as they are.  spec [rows, F, N] complex64; axis 0 = frequency (axis_vals [F] = the reference's
 * linspace(0, sr/2, F)), 1 = time (axis_vals [N] = linspace(0, duration, N)); lo, hi [rows / rows_per_item]. */
int b2a_spec_band_mask_f32(float* spec, int64_t rows, int F, int N, const float* axis_vals, const float* lo,
                           const float* hi, int rows_per_item, int axis, float fill_re, float fill_im, void* stream);
/* DSPMixin.shift_phase (dsp.py:335-351): spec *= exp(1j * shift) in place; shift [items] (per_cell 0) or
 * [items * cells_per_item] (per_cell 1: CorruptPhase's per-cell noise).  spec viewed as [items, cells_per_item]. */
int b2a_spec_rotate_f32(float* spec, int64_t items, int64_t cells_per_item, const float* shift, int per_cell,
                        void* stream);
/* DSPMixin.mask_low_magnitudes (dsp.py:308-333) with log_magnitude()'s arithmetic (audio_signal.py:1457-1487):
 * db = max(10 log10(max(|X|^2, amin_sq)), max over the WHOLE tensor - top_db); cells with db < db_cutoff[item] get
 * magnitude `val` and keep their phase.  ws: 4 bytes of device scratch (4-byte aligned). */
int b2a_spec_mask_low_f32(float* spec, int64_t items, int64_t cells_per_item, const float* db_cutoff, float amin_sq,
                          float top_db, float val, void* ws, void* stream);

/* Spectral noise gate (audiotools/ml/layers/spectral_gate.py:60-129, transforms.SpectralDenoising): per-bin threshold
 * mean_t + n_std * std_t of the noise STFT's dB magnitudes (20 log10 max(|X|, 1e-4)); boolean (signal dB < threshold),
 * smoothed by the zero-padded separable kernel smooth_f (x) smooth_t / sum (the reference's conv2d with the outer
 * product of two triangles); out = spec * (1 - amount[item] * smoothed).  spec / out [rows, F, N] complex64 (out must
 * not alias spec), nz_spec [nz_rows, F, nz_N] with nz_rows 1 or rows, amount [rows / rows_per_item] device,
 * smooth_f_h / smooth_t_h HOST vectors of odd length <= 17, ws >= nz_rows * F floats. */
int b2a_spec_gate_f32(const float* spec, int64_t rows, int F, int64_t N, const float* nz_spec, int64_t nz_rows,
                      int64_t nz_N, float n_std, const float* amount, int rows_per_item, const float* smooth_f_h,
                      int n_f, const float* smooth_t_h, int n_t, float* out, void* ws, void* stream);

/* ---- gradients of the spectral masks and the spectral gate (differentiable through torch in the reference) -------
 * A complex gradient is G = dL/dRe + i dL/dIm (torch's convention).  The forwards of the gradient path write a new
 * tensor (one read and one write per cell, `out` must not alias `spec`); the backwards recompute each mask decision
 * from the forward's input `spec` with the forward's arithmetic.  No atomics in any backward.
 *   b2a_spec_band_mask_out_f32       b2a_spec_band_mask_f32 into `out`: out = fill in the band, spec elsewhere.
 *   b2a_spec_band_mask_backward_f32  grad_spec = 0 in the band and where spec == 0 (|X| and angle(X) both
 *                                    backpropagate 0 there), grad_out elsewhere.  Same arguments as the forward.
 *   b2a_spec_mask_low_out_f32        b2a_spec_mask_low_f32 into `out`; ws (4 bytes) then holds the maximum |X|^2 and is
 *                                    passed unchanged to the backward.
 *   b2a_spec_mask_low_backward_f32   unmasked cells: grad_out (0 where spec == 0); masked cells (magnitude := val, phase
 *                                    kept): val (g - Re(g conj u) u) / |X| with u = X / |X|, 0 where spec == 0.
 *   b2a_spec_gate_backward_f32       grad_spec = grad_out * (1 - amount[item] * smoothed), the mask recomputed from spec
 *                                    and the thresholds `thresh` [nz_rows, F] that b2a_spec_gate_f32 left in its ws.
 *                                    Arguments as b2a_spec_gate_f32; grad_spec must not alias spec. */
int b2a_spec_band_mask_out_f32(const float* spec, float* out, int64_t rows, int F, int N, const float* axis_vals,
                               const float* lo, const float* hi, int rows_per_item, int axis, float fill_re,
                               float fill_im, void* stream);
int b2a_spec_band_mask_backward_f32(const float* grad_out, const float* spec, int64_t rows, int F, int N,
                                    const float* axis_vals, const float* lo, const float* hi, int rows_per_item,
                                    int axis, float* grad_spec, void* stream);
int b2a_spec_mask_low_out_f32(const float* spec, float* out, int64_t items, int64_t cells_per_item,
                              const float* db_cutoff, float amin_sq, float top_db, float val, void* ws, void* stream);
int b2a_spec_mask_low_backward_f32(const float* grad_out, const float* spec, int64_t items, int64_t cells_per_item,
                                   const float* db_cutoff, float amin_sq, float top_db, float val, const void* ws,
                                   float* grad_spec, void* stream);
int b2a_spec_gate_backward_f32(const float* grad_out, const float* spec, int64_t rows, int F, int64_t N,
                               const float* thresh, int64_t nz_rows, const float* amount, int rows_per_item,
                               const float* smooth_f_h, int n_f, const float* smooth_t_h, int n_t, float* grad_spec,
                               void* stream);

/* ---- integrated loudness (ITU-R BS.1770 / LUFS) ----------------------------------------
 * Replaces Meter.integrated_loudness with the IIR semantics of apply_filter_cpu
 * (audiotools/core/loudness.py:102-126, 164-247) and the pad / clamp shell of
 * LoudnessMixin.loudness (:268-320); optionally also produces normalize()'s gain
 * (audiotools/core/effects.py:214-217).
 *
 *   x [B, C, T];  T_padded >= T is the zero-extended length (loudness.py:302-305)
 *   sos_h   [n_stage][6] float64 host: b0 b1 b2 a0 a1 a2 per biquad stage, in application order
 *           (pyloudnorm K-weighting: high-shelf then high-pass); coefficients are rounded to
 *           float32 exactly as the reference does (:118-119); stage_gain_h [n_stage] passband gains
 *   chan_gain_h [C] float64 host (G = [1,1,1,1.41,1.41], :49-50)
 *   block_s  gating block in seconds (0.4): K = int(block_s*rate), stride = int(block_s*rate*0.25)
 *   z_blocks nullable [B, C, nblk] float32 block energies before gating (:214)
 *   lufs_out [B] float32: integrated loudness, NOT clamped (may be -inf for silence)
 *   loud_out nullable [B]: max(lufs, -70)            (:315-320)
 *   target_db nullable [n_target] (n_target 1 or B), gain_out nullable [B]:
 *            gain = exp((target_db - loud) * ln(10)/20)
 *   ws: b2a_lufs_workspace_bytes(...) bytes of scratch, contents irrelevant on entry.
 */
int64_t b2a_lufs_num_blocks(int64_t T_padded, double rate, double block_s);
size_t b2a_lufs_workspace_bytes(int64_t B, int C, int64_t T_padded, double rate, double block_s);
int b2a_lufs_f32(const float* x, int64_t B, int C, int64_t T, int64_t T_padded, double rate,
                 const double* sos_h, const double* stage_gain_h, int n_stage, double block_s,
                 const double* chan_gain_h, float* z_blocks, float* lufs_out, float* loud_out,
                 const float* target_db, int n_target, float* gain_out,
                 void* ws, size_t ws_bytes, void* stream);

/* ---- per-item gain ---------------------------------------------------------------------
 * x[b, :, :] * gain[b]  (EffectMixin.normalize / volume_change, effects.py:219,237).
 * out may alias x.  per_item = C*T. */
int b2a_gain_f32(const float* x, float* out, int64_t B, int64_t per_item, const float* gain, void* stream);

/* ---- FIR / circular convolution by partitioned overlap-save FFT convolution -------------------
 * out[row][n] = post_scale[f] * sum_{k<L} g[f][k] * xv[row][n - k + offset0 + offset[f]],  f = row / rows_per_filt,
 * n in [0, T), where xv extends x[row] by pad_mode: 1 zeros, 2 replicate (edge), 3 circular (period T).
 * With subtract_from_input != 0 the result is x - (that).   g: [n_filt, L] row-major taps (zero-pad
 * shorter filters); offset / post_scale: nullable [n_filt].   out must not alias x.
 * bypass: nullable [n_filt] int32 -- the rows of a filter with bypass != 0 are copied through unchanged (out = x,
 * exactly): how a transform applies itself to the items its mask selects without gathering / scattering the batch
 * (audiotools/data/transforms.py:133-166).  The same argument exists on b2a_fir_direct_f32 (stride 1) and
 * b2a_circconv_f32.
 * Replaces julius.LowPassFilter / HighPassFilter (audiotools/core/dsp.py:153-215), julius.SplitBands +
 * the weighted band sum (audiotools/core/effects.py:386-433) -- each collapsed to one FIR per item. */
size_t b2a_fftconv_workspace_bytes(int64_t rows, int64_t T, int64_t n_filt, int64_t L);
int b2a_fftconv_f32(const float* x, int64_t rows, int64_t T, const float* g, int64_t n_filt, int64_t L,
                    int rows_per_filt, const int32_t* offset, int offset0, int pad_mode,
                    const float* post_scale, int subtract_from_input, const int32_t* bypass, float* out, void* ws,
                    size_t ws_bytes, void* stream);

/* Direct (time-domain) strided FIR for short filters, correlation form:
 *   out[row][m] = sum_{k<K} taps[f][k] * xv[row][m*stride + k - left0 - left[f]],  f = row / rows_per_filt, m < out_len
 * xv = x extended by zeros (pad_mode 1) or edge replication (2).  Used for short julius.LowPassFilter /
 * HighPassFilter taps (stride 1, left = half; subtract_from_input gives x - y) and for julius.resample_frac when
 * the reduced new rate is 1 (stride = old rate, left = width).  b2a_fir_direct_supported tells whether
 * (K, stride) fits the kernel's shared memory; longer filters go through b2a_fftconv_f32. */
int b2a_fir_direct_supported(int64_t T, int K, int stride);
int b2a_fir_direct_f32(const float* x, int64_t rows, int64_t T, const float* taps, int64_t n_filt, int K,
                       int rows_per_filt, const int32_t* left, int left0, int stride, int64_t out_len,
                       int pad_mode, int subtract_from_input, const int32_t* bypass, float* out, void* stream);

/* Replicate-padding fold of a stride-1 FIR's gradient.  For the correlation form y[m] = sum_k taps[f][k] *
 * xv[m + k - left0 - left[f]] with replicate padding, the gradient is the zero-padded correlation with the reversed
 * taps (b2a_fftconv_f32, pad_mode 1) PLUS what the padded positions carry back to the edge samples; this adds that
 * part to grad_x in place:
 *   grad_x[0]   += sum_{n < l}           (taps[0] + .. + taps[min(l-1-n, K-1)]) grad_out[n]          (l = left0 + left[f])
 *   grad_x[T-1] += sum_{n > T + l - K}   (taps[T+l-n] + .. + taps[K-1]) grad_out[n]
 * valid for any T (also T < K).  Rows of a filter with bypass != 0 are left alone (their gradient is the copy).
 * ws: b2a_fir_pad_fold_workspace_bytes() bytes (prefix / suffix sums of every filter, computed on the device). */
size_t b2a_fir_pad_fold_workspace_bytes(int64_t n_filt, int K);
int b2a_fir_pad_fold_f32(const float* grad_out, int64_t rows, int64_t T, const float* taps, int64_t n_filt, int K,
                         int rows_per_filt, const int32_t* left, int left0, const int32_t* bypass, float* grad_x,
                         void* ws, size_t ws_bytes, void* stream);

/* EffectMixin.convolve (audiotools/core/effects.py:66-123): CIRCULAR convolution (period T) of each row with
 * its item's impulse response, the IR rolled so that max|ir| sits at t = 0 (roll_to_peak) and the result
 * scaled by 1 / max(max|ir|, 1e-5).   ir: [n_ir, L] with L <= T (truncate first, as the reference does). */
size_t b2a_circconv_workspace_bytes(int64_t rows, int64_t T, int64_t n_ir, int64_t L);
int b2a_circconv_f32(const float* x, int64_t rows, int64_t T, const float* ir, int64_t n_ir, int64_t L,
                     int rows_per_ir, int roll_to_peak, const int32_t* bypass, float* out, void* ws, size_t ws_bytes,
                     void* stream);
/* Gradient of b2a_circconv_f32 with respect to x (same arguments; the IR is a constant): with the forward
 * y[n] = s sum_j h[j] x[(n - j + idx) mod T], grad_x[m] = s sum_j h[j] grad_out[(m + j - idx) mod T] -- a circular
 * correlation, run on the same engine with reversed taps.  Bypassed rows: grad_x = grad_out.  grad_x must not alias
 * grad_out. */
size_t b2a_circconv_backward_workspace_bytes(int64_t rows, int64_t T, int64_t n_ir, int64_t L);
int b2a_circconv_backward_f32(const float* grad_out, int64_t rows, int64_t T, const float* ir, int64_t n_ir, int64_t L,
                              int rows_per_ir, int roll_to_peak, const int32_t* bypass, float* grad_x, void* ws,
                              size_t ws_bytes, void* stream);

/* ---- windowed-sinc polyphase resampling ------------------------------------------------------
 * AudioSignal.resample (audiotools/core/audio_signal.py:716-736 -> julius.resample_frac): old_r/new_r are
 * the gcd-reduced rates, kernel_t the per-phase kernels transposed to [K = 2*width + old_r][new_r]
 * (julius.ResampleFrac._init_kernels: zeros 24, rolloff 0.945, each phase renormalised to sum 1).
 * out: [rows, b2a_resample_out_len(T, old_r, new_r)] = floor(new_r*T/old_r) samples per row. */
int64_t b2a_resample_out_len(int64_t T, int old_r, int new_r);
int b2a_resample_f32(const float* x, int64_t rows, int64_t T, int old_r, int new_r, int width,
                     const float* kernel_t, float* out, void* stream);
/* Gradient of the resampling with respect to x (either forward route: the polyphase kernel above, or
 * b2a_fir_direct_f32 when new_r == 1): grad_out [rows, out_len] -> grad_x [rows, T],
 *   grad_x_ext[u] = sum_{m, i} kernel_t[u + width - m*old_r][i] grad_out[m*new_r + i]   (0 <= u + width - m*old_r < K),
 * with the replicate padding folded back: grad_x[0] also takes u in [-width, 0), grad_x[T-1] u in [T, T + width + old_r).
 * Fixed summation order (no atomics): reruns are bit-identical. */
int b2a_resample_backward_f32(const float* grad_out, int64_t rows, int64_t T, int old_r, int new_r, int width,
                              const float* kernel_t, float* grad_x, void* stream);

/* ---- pitch shift ---------------------------------------------------------------------------------
 * EffectMixin.pitch_shift (audiotools/core/effects.py:247-277; SoX `pitch -q` + `rate` there): WSOLA
 * time-scale modification by r = 2^(semitones/12) (search -> overlap-add into the workspace) + band-limited
 * rate change by 1/r (windowed sinc, cutoff 0.95*min(1,1/r), 8 zero crossings), output length == T.
 * ws: 16-byte aligned, b2a_pitch_shift_workspace_bytes() bytes (frame positions + the stretched rows). */
size_t b2a_pitch_shift_workspace_bytes(int64_t rows, int64_t T, int sr, float semitones);
int b2a_pitch_shift_f32(const float* x, int64_t rows, int64_t T, int sr, float semitones, float* out, void* ws,
                        size_t ws_bytes, void* stream);
/* Several shifts in one launch (a batch whose items drew different shifts, e.g. a PitchShift transform):
 * semitones_h HOST [n_groups] (n_groups <= 8 distinct values, 0 = copy the row), row_group DEVICE [rows] int32
 * in [0, n_groups) (nullable when n_groups == 1).  Rows of all groups share every launch, so the one-CTA-per-row
 * search fills the GPU with the whole batch instead of one group at a time. */
size_t b2a_pitch_shift_multi_workspace_bytes(int64_t rows, int64_t T, int sr, const float* semitones_h, int n_groups);
int b2a_pitch_shift_multi_f32(const float* x, int64_t rows, int64_t T, int sr, const float* semitones_h, int n_groups,
                              const int32_t* row_group, float* out, void* ws, size_t ws_bytes, void* stream);

/* EffectMixin.time_stretch (audiotools/core/effects.py:279-309; SoX `tempo factor` + `rate` there): the WSOLA stages of
 * the pitch shifter on their own: out [rows, out_len] with out_len = b2a_time_stretch_out_len(T, factor) = round(T / factor),
 * pitch unchanged; factor in [0.25, 4], factor == 1 copies. */
/* number of WSOLA frames J of a row for this shift: the splice positions chosen by the search are the first
 * rows * J int32 of the workspace after the call (row-major [rows, J]); exposed so that tests can compare them with
 * the oracle (oracle/pitch_spec.py) exactly */
int b2a_pitch_shift_num_frames(int64_t T, int sr, float semitones);
int64_t b2a_time_stretch_out_len(int64_t T, double factor);
size_t b2a_time_stretch_workspace_bytes(int64_t rows, int64_t T, int sr, double factor);
int b2a_time_stretch_f32(const float* x, int64_t rows, int64_t T, int sr, double factor, float* out, void* ws,
                         size_t ws_bytes, void* stream);

/* ---- element-wise / per-row-peak effects (csrc/effects.cu; audiotools/core/effects.py:27-64,181-198,435-523) -------
 * One pass over the waveform each; x, out: [B or rows, per_item or T] float32 contiguous, device pointers.
 *   b2a_row_absmax_f32   peak[row] = max |x[row, :]|  (ensure_max_of_audio :194, apply_ir's peak restore :155,176)
 *   b2a_limit_peak_f32   out = x * (peak[row] > max_abs ? max_abs / peak[row] : 1)          (:181-198)
 *   b2a_mix_f32          out = x + other_gain[item] * other   (other_gain nullable = 1)       (:27-64: the
 *                        normalize() multiply of the noise and the addition, in one pass)
 *   b2a_quantize_f32     mulaw = 0: linear quantisation to channels[item] levels (:463-491); 1: mu-law (:493-523);
 *                        the reference's float32 operation order, including out = x - (x - q)
 *   b2a_order_stats_f32  out[i] = the k[i]-th smallest value (0-based) of row[0..T): exact 4-pass radix selection;
 *                        k: device int64 [nk].  torch.quantile's sorted gather for clip_distortion (:452-453)
 *   b2a_clamp_items_f32  out = min(max(x, lo[item]), hi[item])                                 (:459) */
int b2a_row_absmax_f32(const float* x, int64_t rows, int64_t T, float* peak, void* stream);
int b2a_limit_peak_f32(const float* x, float* out, int64_t rows, int64_t T, const float* peak, float max_abs, void* stream);
/* Gradient of the per-row peak rescales, one CTA per row (first arg-max and dot(grad_out, y) in a fixed order):
 *   x_ref == NULL  ensure_max_of_audio, y' = y p with p = max_abs / peak where peak = max|y| > max_abs, else 1:
 *                  grad_y = p g - [peak > max_abs] (max_abs / peak^2) dot(g, y) sign(y_b) e_b
 *   x_ref != NULL  apply_ir's peak restore, y' = y S, S = clamp(max|x_ref|, 1e-8) / clamp(max|y|, 1e-8):
 *                  grad_y = S g - [My >= 1e-8] S dot(g, y) / My sign(y_b) e_b,
 *                  grad_x_ref = [Mx >= 1e-8] dot(g, y) / clamp(My, 1e-8) sign(x_a) e_a (zero elsewhere, written whole);
 *                  bypass: nullable [rows] int32, non-zero = S was 1: grad_y = g, grad_x_ref = 0.
 * e_a, e_b: the first index of the row's maximum.  [rows, T] float32 each. */
int b2a_peak_scale_backward_f32(const float* grad_out, const float* y, const float* x_ref, int64_t rows, int64_t T,
                                float max_abs, const int32_t* bypass, float* grad_y, float* grad_x_ref, void* stream);
int b2a_clamp_items_f32(const float* x, float* out, int64_t B, int64_t per_item, const float* lo, const float* hi,
                        void* stream);
int b2a_mix_f32(const float* x, const float* other, const float* other_gain, float* out, int64_t B, int64_t per_item,
                void* stream);
int b2a_quantize_f32(const float* x, float* out, int64_t B, int64_t per_item, const float* channels, int mulaw,
                     void* stream);
int b2a_order_stats_f32(const float* row, int64_t T, const int64_t* k, int nk, float* out, void* stream);

/* ImpulseResponseMixin.alter_drr (audiotools/core/effects.py:540-647: decompose_ir + solve_alpha + the re-weighted sum +
 * ensure_max_of_audio) in ONE launch, one CTA per impulse-response row.  ir / out [rows = B*C, T] (out must not alias
 * ir), t0 = int(sample_rate * 0.0025), drr [B] target direct-to-reverberant ratios in dB, max_abs = 1. */
int b2a_alter_drr_f32(const float* ir, float* out, int64_t rows, int64_t T, int C, int t0, const float* drr,
                      float max_abs, void* stream);

/* ---- ragged signals -> one padded / truncated batch (csrc/collate.cu; AudioSignal.batch, audiotools/core/audio_signal.py:
 * 380-470, called by util.collate, core/util.py:426-479; excerpt gathering of salient_excerpt, audio_signal.py:227-286)
 * item i = C rows of src_len[i] samples at src_ptrs[i], consecutive rows src_stride[i] samples apart;
 * out[i, c, t] = row c's sample t + src_off[i] when that index is inside [0, src_len[i]), else 0 (zero padding,
 * truncation at T_out).  src_ptrs / src_len / src_stride / src_off (nullable = 0) are DEVICE arrays of n_items entries. */
int b2a_pack_rows_f32(const float* const* src_ptrs, const int64_t* src_len, const int64_t* src_stride,
                      const int64_t* src_off, int64_t n_items, int C, int64_t T_out, float* out, void* stream);

/* 1 when b2a_spectral_f32 runs a launch of this geometry on the tensor-core kernel (csrc/spectral_tc.cu: wgmma,
 * accumulators in registers): window_length 2048, hop <= 512, mel / log-mel output without the complex STFT, and
 * the path switched on with b2a_spectral_tc_enable(1).  It is opt-in: the FP32 warp kernel of
 * spectral.cu is the default; every other launch uses the FP32 kernels. */
int b2a_spectral_uses_tensor_cores(int n_fft, int hop, int want_mel, int want_stft);
/* Switch the tensor-core path on / off for this process (A/B measurements, parity tests of both kernels); returns the
 * previous setting. */
int b2a_spectral_tc_enable(int on);

/* ---- STOI / extended STOI (csrc/stoi.cu; metrics.quality.stoi, audiotools/metrics/quality.py:11-57, which calls
 * pystoi.stoi(references[i, 0], estimates[i, 0], sample_rate, extended) per item after to_mono).
 *   est, ref   [batch, channels, T] float32; mixed to mono (mean over channels) inside the first launch
 *   taps       [n_taps] float64, n_taps odd: scipy.signal.resample_poly's filter for up / down (the gcd-reduced
 *              10000 / sample_rate), already multiplied by up -- pystoi's Octave Kaiser design, normalised to unit sum,
 *              times up.  At 10 kHz: up = down = 1 and taps = {1}.
 *   out        [batch] float64 scores; 1e-5 where fewer than 30 STFT frames survive the silence removal
 *   kept_out   [batch] int32 frames kept by the silence removal (the STFT then has kept_out - 1 frames)
 *   short_out  [batch] int32, 1 where the score is the 1e-5 of a short item
 *   ws         b2a_stoi_workspace_bytes(batch, T, up, down) bytes
 * B2A_E_INVALID when the signal has no full 256-sample frame at 10 kHz.  Four launches, no atomics: bit-identical
 * reruns.  The extended mode leaves out pystoi's EPS-scale random noise (deterministic). */
size_t b2a_stoi_workspace_bytes(int64_t batch, int64_t T, int up, int down);
int b2a_stoi_f32(const float* est, const float* ref, int64_t batch, int channels, int64_t T, int extended,
                 const double* taps, int n_taps, int up, int down, double* out, int32_t* kept_out, int32_t* short_out,
                 void* ws, size_t ws_bytes, void* stream);

/* ---- one-sided statistics exchange between the GPUs of a node (NVLink peer memory) --------------------
 * The path shards by batch item with no data-path collective; the one exchange is the per-item loudness vector for
 * whole-batch statistics (the reference has no multi-GPU code of its own: SURVEY.md 8e).  Every rank owns a small
 * buffer (b2a_peer_buffer_create: cudaMalloc + cudaIpc handle), maps its peers' buffers (b2a_peer_buffer_open on
 * the 64-byte handles, exchanged by the host side), then per step
 *   b2a_peer_put_f32      stores src[0..n) into its slot of EVERY rank's buffer and publishes `seq` (system-scope
 *                         release); no rendezvous, no NCCL kernel, NEVER waits for another rank;
 *   b2a_peer_latest_f32   reads from the LOCAL buffer the newest complete vector of every rank -> out [world, n] and
 *                         the sequence number each row carries -> seqs_out [world] (0 + NaN row: nothing published
 *                         yet).  Never waits: a rank that is behind shows an older sequence number;
 *   b2a_peer_collect_f32  the lock-step form: waits (bounded spin) until every rank published exactly `seq`, gathers
 *                         [world, n]; seqs_out (nullable) [world] = seq, or -(what was seen) + a NaN row for a rank
 *                         that died or lapped the slot.  For validation / exact-step statistics, on a side stream.
 * seq >= 1 grows by one per step; slots rotate over 4 sequence numbers and are seqlock-protected (invalidate, data,
 * publish), so readers never accept a torn or overwritten vector whatever the skew between ranks.
 * b2a_peer_status copies the buffer's status word (last sequence number a collect gave up on, 0 = none) to
 * status_out (device int32). */
size_t b2a_peer_buffer_bytes(int world, int n_max);
int b2a_peer_buffer_create(int world, int n_max, void** dev_ptr, unsigned char* handle_out /*[64]*/);
int b2a_peer_buffer_open(const unsigned char* handle /*[64]*/, void** peer_ptr);
int b2a_peer_buffer_close(void* peer_ptr);
int b2a_peer_buffer_destroy(void* dev_ptr);
int b2a_peer_put_f32(const float* src, int n, void* const* peer_bufs_h /*host [world]*/, int world, int rank,
                     int n_max, int seq, void* stream);
int b2a_peer_latest_f32(const void* local_buf, int world, int n, int n_max, float* out, int32_t* seqs_out,
                        void* stream);
int b2a_peer_collect_f32(const void* local_buf, int world, int n, int n_max, int seq, float* out, int32_t* seqs_out,
                         void* stream);
int b2a_peer_status(const void* local_buf, int world, int n_max, int32_t* status_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B2A_H_ */
