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

/* Kernels the library has launched in this process, over all entry points, devices, streams and threads.  Every
 * kernel launch adds one (a relaxed atomic add on the host); memsets and copies are not counted.  A caller that reads
 * it before and after an entry point gets the kernels that call launched, provided no other thread launched in
 * between.  It is a variable rather than a function so that reading it costs no foreign-function call. */
extern int64_t b2a_kernel_launches;

/* ---- STFT / mel ---------------------------------------------------------------------
 * Replaces the device work of AudioSignal.stft (audiotools/core/audio_signal.py:1123-1212:
 * F.pad(pad, pad+right_pad, padding_type) -> torch.stft(center=True, reflect) -> optional
 * drop of 2+2 edge frames) and AudioSignal.mel_spectrogram (:1333-1369: |X| @ mel_basis.T),
 * on the route b2a_stft_route(n_fft, hop, 0), with the same framing and bit-exact frame indexing on every route:
 *   FFT           one fused pass over x: framing -> window -> real FFT -> |.| -> banded mel -> post-op.
 *   LARGE / DENSE the gain pass (b2a_gain_f32) if gain != NULL, the STFT of all frames (fft_large.cu's per-frame FFT /
 *                 dft.cu's dense DFT), then |X| -> banded mel -> post-op from that STFT if mel_out != NULL: up to
 *                 3 launches (the gain pass takes rows / rows_per_gain <= 65535, the mel pass rows <= 65535).
 *                 The STFT and the scaled signal go to ws when the caller does not ask for them.
 *
 *   x        [rows, T]
 *   window   [n_fft]              (AudioSignal.get_window, :1009-1039)
 *   matrix   nullable; on DENSE the kind 0 matrix of b2a_dft_matrix_f32
 *   n_fft/hop                     any pair whose forward route is not B2A_ROUTE_NONE
 *   pad/right_pad/pad_mode        compute_stft_padding (:1089-1121); 0/0 when !match_stride
 *   drop_edge                     frames dropped at each end (2 when match_stride, else 0)
 *   gain     nullable [rows/rows_per_gain]: x is multiplied by gain[row / rows_per_gain] first
 *            (EffectMixin.normalize's x*gain, effects.py:219) and, if y_out != NULL, the scaled
 *            waveform is written there ([rows, T]); on FFT by the same pass, which needs pad == right_pad ==
 *            drop_edge == 0 for y_out.  On LARGE / DENSE rows_per_gain divides rows.
 *   mel_fb   nullable [n_mels, F] row-major dense filterbank (get_mel_filters, :1298-1331);
 *   mel_lo/mel_hi  [n_mels] int32: mel_fb[m, k] == 0 outside mel_lo[m] <= k < mel_hi[m]
 *            (the caller derives them from the actual non-zeros, so the banded sum equals the
 *            dense matmul exactly for ANY matrix).
 *   mel_packed_len  floats of the kernel's shared-memory band table (0: read the weights from global):
 *            with n4[m] = (ceil4(mel_hi[m]) - floor4(mel_lo[m]))/4, 4 * sum over filters m of
 *            even(max(n4[m'] : m' in {4g .. 4g + 3})) where g = m / 4, even(v) = (v+1) & ~1
 *            (the 4 consecutive filters one warp projects in one step share a trip count; the loop is unrolled by two).
 *            Used on FFT only.
 *   mel_out  nullable [rows, n_mels, n_frames]    stft_out  nullable [rows, F, n_frames] (re,im); at least one of them
 *   n_frames = 1 + (T + 2*pad + right_pad)/hop - 2*drop_edge,  F = n_fft/2 + 1
 *   ws       b2a_spectral_workspace_bytes(..., stft_out == NULL, gain != NULL && y_out == NULL) bytes, 8-byte aligned:
 *            the STFT when stft_out is NULL, then the scaled signal when y_out is NULL.  0 on FFT, where ws may be NULL.
 */
int64_t b2a_stft_num_frames(int64_t T, int n_fft, int hop, int pad, int right_pad, int drop_edge);
size_t b2a_spectral_workspace_bytes(int64_t rows, int64_t T, int n_fft, int hop, int pad, int right_pad, int drop_edge,
                                    int stft_scratch, int scaled_scratch);
int b2a_spectral_f32(const float* x, int64_t rows, int64_t T, int n_fft, int hop, const float* window,
                     const float* matrix, int pad, int right_pad, int pad_mode, int drop_edge,
                     const float* gain, int rows_per_gain, float* y_out,
                     const float* mel_fb, const int32_t* mel_lo, const int32_t* mel_hi, int n_mels,
                     int mel_packed_len, int post, float post_eps, float post_power,
                     float* mel_out, float* stft_out, void* ws, size_t ws_bytes, void* stream);

/* ---- the one route table: which kernel family runs an STFT of (n_fft, hop) -------------------------------------
 * inverse 0: the forward STFT, b2a_spectral_f32.  inverse 1: b2a_istft_f32 and both backward passes.  Each of these
 * routes by the table itself.  Everything not in the table is B2A_ROUTE_NONE.
 *                      FFT                          LARGE                          DENSE
 *   inverse 0, hop>=1  power of two in [32, 4096]   power of two in [8192, 32768]  any other length in [2, 8192]
 *   inverse 1, hop in  power of two in [64, 2048]   power of two in [4096, 32768]  any other length in [2, 8192]
 *   [1, n_fft]                                                                     (incl. 32)
 * LARGE serves the default window of AudioSignal.stft_params, 2^ceil(log2(0.032 sr)), at high rates: 8192 at 176.4 /
 * 192 kHz (and the inverse of 4096 at 88.2 / 96 kHz); 16384 / 32768 serve fine frequency resolution.  It needs no
 * matrix and no table. */
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
 *                          for b2a_spectral_f32, inverse 1 -> c_k/n_fft . w[n] exp(-2 pi i nk/n_fft) (c = 1 for DC and
 *                          Nyquist, else 2) for b2a_istft_f32, inverse 2 -> the layout of 1 with weight 1 on every
 *                          bin for b2a_stft_backward_f32; `matrix`: b2a_dft_matrix_floats(n_fft, inverse)
 *                          floats, 16-byte aligned; angles reduced in integers (nk mod n_fft), evaluated in float64 */
size_t b2a_dft_matrix_floats(int n_fft, int inverse);
int b2a_dft_matrix_f32(const float* window, int n_fft, int inverse, float* matrix, void* stream);
/* AudioSignal.mfcc's `log-mel^T @ create_dct(n_mfcc, n_mels, "ortho")` (audio_signal.py:1420-1426):
 * out[row][j][n] = sum_m dct[m][j] * logmel[row][m][n];  logmel [rows, n_mels, n_frames], dct [n_mels, n_mfcc] row-major. */
int b2a_mel_dct_f32(const float* logmel, int64_t rows, int n_mels, int64_t n_frames, const float* dct, int n_mfcc,
                    float* out, void* stream);

/* ---- backward passes of the spectral front end (csrc/grad.cu) ---------------------------------------------------
 * Gradients of AudioSignal.stft / istft / mel_spectrogram / mfcc (audiotools/core/audio_signal.py:1123-1296, 1333-1426;
 * differentiable through torch there, tests/core/test_grad.py).  A complex gradient is G = dL/dRe + i dL/dIm (torch's
 * convention); every pass is deterministic (no atomics, fixed summation order).  Both backward passes exist where
 * b2a_stft_route(n_fft, hop, 1) is not B2A_ROUTE_NONE, and run on that route.
 *   b2a_stft_backward_f32        grad_spec [rows, n_fft/2+1, n_frames] (re,im) -> grad_x [rows, T], for the STFT that
 *                                b2a_spectral_f32 computed with the same (T, n_fft, hop, window, pad, right_pad,
 *                                pad_mode, drop_edge) and no gain: per frame
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

/* ---- gradient of the integrated loudness (K21) -------------------------------------------
 * grad_x [B, C, T] float32 = grad_loud[b] d loud_b / d x, loud = max(lufs, -70) of b2a_lufs_f32, for the same
 * x [B, C, T], T_padded, rate, sos_h, stage_gain_h, n_stage, block_s and chan_gain_h as that call:
 *   d loud / d x_c = K^T u_c,  u_c[t] = (10 / ln 10) G_c scale gain / (E n) * 2 y_c[t] * m[t]
 * y_c = K x_c on the row zero-extended to T_padded (K: the cascade, float32 coefficients as b2a_lufs_f32 rounds them),
 * scale = float32(1 / (block_s rate)), J the blocks that passed both gates, n = |J|, E = sum_c G_c zavg_c, m[t] the
 * number of blocks of J that contain t, K^T the cascade run backwards in time over [0, T_padded), cropped to [0, T).
 *   grad_loud [B] float32 on the device.
 *   gain nullable [B]: the forward measured float32(gain[b] x) (a deferred normalize() gain); grad_x is then with
 *        respect to x.
 *   z_blocks [B, C, nblk], lufs [B]: the z_blocks and lufs_out of the forward call.  The gate decisions are rebuilt
 *        from them by the forward's own functions; they are constants of the backward (piecewise-constant).
 *   An item with lufs <= -70 gets an exactly zero row; an item with a non-finite block energy (a NaN or inf sample)
 *   gets an all-NaN row.  Other items are unaffected; reruns and batch-versus-single calls are bit-identical.
 *   ws: b2a_lufs_backward_workspace_bytes(B, C, T_padded, rate, block_s) bytes of scratch.
 * Seven launches (one per-item gate kernel, two three-launch passes of csrc/iir.cu), no host sync. */
size_t b2a_lufs_backward_workspace_bytes(int64_t B, int C, int64_t T_padded, double rate, double block_s);
int b2a_lufs_backward_f32(const float* grad_loud, const float* x, const float* gain, int64_t B, int C, int64_t T,
                          int64_t T_padded, double rate, const double* sos_h, const double* stage_gain_h,
                          int n_stage, double block_s, const double* chan_gain_h, const float* z_blocks,
                          const float* lufs, float* grad_x, void* ws, size_t ws_bytes, void* stream);

/* ---- EBU R128 loudness statistics ------------------------------------------------------
 * The six numbers of audiotools/core/ffmpeg.py:13-62 (r128stats) for every item, in one
 * K-weighting pass of the GPU instead of one ffmpeg process per item.  BS.1770 arithmetic of
 * b2a_lufs_f32 (block 0.4 s), not ffmpeg's quantised gating histogram.  Arguments as b2a_lufs_f32.
 *   stats_out [B, 6] float32: I (== b2a_lufs_f32's lufs_out, -inf for silence), I Threshold (the
 *            relative gate, -inf when no block passes -70), LRA, LRA Threshold, LRA Low, LRA High
 *   momentary_out nullable [B, nblk]: -0.691 + 10 log10(sum_c G_c z_c) per 400 ms block
 *   short_term_out nullable [B, n_st]: 3 s short-term loudness S_i over strides i .. i+29,
 *            n_st = (T_padded - 30 stride) / stride + 1 (0 when T_padded < 30 stride)
 *   LRA fields from S: absolute gate S > -70, LRA Threshold = power mean of those - 20 LU,
 *   relative gate S > LRA Threshold, nearest-rank 10 % / 95 % percentiles (Low / High) of the
 *   kept S, LRA = High - Low; LRA = 0 and the other three -inf when no S passes -70.
 *   ws: b2a_loudness_stats_workspace_bytes(...) bytes of scratch, contents irrelevant on entry.
 */
int64_t b2a_loudness_stats_num_short_term(int64_t T_padded, double rate);
size_t b2a_loudness_stats_workspace_bytes(int64_t B, int C, int64_t T_padded, double rate);
int b2a_loudness_stats_f32(const float* x, int64_t B, int C, int64_t T, int64_t T_padded, double rate,
                           const double* sos_h, const double* stage_gain_h, int n_stage,
                           const double* chan_gain_h, float* stats_out, float* momentary_out,
                           float* short_term_out, void* ws, size_t ws_bytes, void* stream);

/* ---- true-peak level (ITU-R BS.1770 Annex 2 structure, this package's interpolator; csrc/truepeak.cu) -----------
 * The largest |value| of each row oversampled by L with a 12-tap Hann-windowed-sinc polyphase FIR:
 *   b2a_true_peak_factor   L for a sample rate: 4 below 96 kHz, 2 below 192 kHz, else 1 (host only; B2A_E_INVALID for
 *                          a rate that is not positive and finite)
 *   b2a_true_peak_taps     the float taps the kernel uses (host only): taps_h [(factor - 1) * 12], phase p = 1 .. L-1
 *                          at [(p - 1) * 12], tap d = -6 .. 5 at [+ d + 6]; h_p[d] = float(sinc(u) (1 + cos(pi u / 6)) / 2)
 *                          with u = d + p / L, designed in double.  No per-phase renormalisation.
 *   b2a_true_peak_f32      x [B, C, T]; the instants are every (n, p) with n < T - 1 plus (T - 1, 0), where phase 0 is
 *                          x[n] itself and phase p >= 1 is sum_{d=-6..5} h_p[d] x[n - d] (x = 0 outside [0, T)).
 *                          row_peak [B * C] linear max |y| over those instants (>= max |x|, bit for bit; NaN or +inf
 *                          for a row with a non-finite sample); item_db nullable [B]: 20 log10 of the channel maximum
 *                          (-inf for silence).  factor 1, 2 or 4.  Two launches (one without item_db) and a memset; the
 *                          maximum is exact and order-independent: reruns are bit-identical.  Not the Annex's coefficient table:
 *                          values are not those of ffmpeg / libebur128. */
int b2a_true_peak_factor(double rate);
int b2a_true_peak_taps(int factor, float* taps_h);
int b2a_true_peak_f32(const float* x, int64_t B, int C, int64_t T, int factor, float* row_peak, float* item_db,
                      void* stream);

/* ---- look-ahead true-peak limiter (csrc/limiter.cu) ----------------------------------------------------------------
 * One gain series per item that keeps the true-peak envelope of b2a_true_peak_f32's interpolator under a ceiling and is
 * exactly 1 away from the overs.  x [B, C, T]; gain nullable [B] (x means float(gain[b] x) below); ceiling [B] linear;
 * lookahead = A samples, 0 .. 1024; release_a = exp(-1 / (release seconds * rate)) in [0, 1); factor 1, 2 or 4.
 *   e[n]  = max over the channels of max(|x[n]|, max_p |y[n, p]|, max_p |y[n - 1, p]|), y and its instants as in
 *           b2a_true_peak_f32
 *   q[n]  = 0 where e[n] <= ceiling, else 1 - ceiling / e[n] (NaN where e[n] is not finite)
 *   h[n]  = max q[j], |j - n| <= A;  d[n] = max(h[n], a d[n - 1]), then d < 2^-26 counts as 0
 *   r[n]  = mean d[j], |j - n| <= A, over the j inside [0, T);  out[b, c, n] = x[b, c, n] (1 - r[n])
 * out [B, C, T] may alias x; reduction nullable [B, T] receives r.  Where r = 0 out equals x bit for bit.  A NaN or inf
 * sample makes r NaN from at most 2 A + 6 samples before it to the end of that item; other items are unaffected.
 * ws: b2a_limiter_workspace_bytes(B, C, T) bytes of scratch (0 for a bad shape), contents irrelevant on entry.  Three
 * launches, no host sync; reruns and batch-versus-single calls are bit-identical. */
size_t b2a_limiter_workspace_bytes(int64_t B, int C, int64_t T);
int b2a_limiter_f32(const float* x, const float* gain, int64_t B, int C, int64_t T, int factor, const float* ceiling,
                    int lookahead, float release_a, float* out, float* reduction, void* ws, void* stream);

/* ---- per-item IIR biquad cascades (csrc/iir.cu) ---------------------------------------------------------------------
 * scipy.signal.sosfilt with zero initial state, per item.  x [B, C, T]; gain nullable [B] (x means float(gain[b] x));
 * sos [sos_items, S, 6] float32, rows b0 b1 b2 a0 a1 a2, used as b / a0 and a / a0 in float32; sos_items 1 (one set
 * for the batch) or B (set b for item b, all its channels); 1 <= S <= 8 sections, run in order, each in the transposed
 * direct form II, in double (each output rounded to float32 once).  reverse != 0 reads and writes every row back to front (the adjoint of the forward filter).
 * A section that fails |a2| < 1 and |a1| < 1 + a2 makes its item's output all NaN; a NaN or inf sample makes its row
 * non-finite from that sample on; other rows and items are unaffected.  out [B, C, T] may alias x.
 * ws: b2a_sos_filter_workspace_bytes(B, C, T, S) bytes of scratch (0 for a bad shape).  Three launches, no host sync;
 * reruns and batch-versus-single calls are bit-identical. */
size_t b2a_sos_filter_workspace_bytes(int64_t B, int C, int64_t T, int S);
int b2a_sos_filter_f32(const float* x, const float* gain, int64_t B, int C, int64_t T, const float* sos,
                       int64_t sos_items, int S, int reverse, float* out, void* ws, void* stream);

/* scipy.signal.sosfilt(sos, x, zi=zi), per item: as b2a_sos_filter_f32 (reverse = 0), started from zi [S, B, C, 2]
 * float64 (scipy's layout for x [B, C, T]); zf nullable [S, B, C, 2] float64 receives the state after sample T - 1
 * (NaN for an unstable item).  The state is carried in double, so chaining zf into the next segment's zi gives one
 * pass over the whole row.  ws: b2a_sos_filter_workspace_bytes(B, C, T, S) bytes.  Three launches, no host sync. */
int b2a_sos_filter_zi_f32(const float* x, const float* gain, int64_t B, int C, int64_t T, const float* sos,
                          int64_t sos_items, int S, const double* zi, float* out, double* zf, void* ws, void* stream);

/* scipy.signal.sosfiltfilt(sos, x, padtype, padlen), method "pad", per item; x, gain and sos as b2a_sos_filter_f32.
 * padtype 0 (None: no extension), 1 (odd), 2 (even) or 3 (constant); padlen >= 0, or -1 for scipy's default per item,
 * 3 (2S + 1 - min(#{b2 = 0}, #{a2 = 0})).  The row is extended by padlen samples on either side in the loads, filtered
 * forwards from sosfilt_zi(sos) ext[0] into a float32 intermediate, backwards from sosfilt_zi(sos) times its last
 * sample, and cropped.  T must exceed the padding: padlen, or 3 (2S + 1) with the default.  An unstable item is all
 * NaN; a NaN or inf sample makes its whole row non-finite.  out may alias x.
 * ws: b2a_sos_filtfilt_workspace_bytes(B, C, T, S, padtype, padlen) bytes (0 for a bad shape or padding), shared with
 * the backward.  Six launches, no host sync. */
size_t b2a_sos_filtfilt_workspace_bytes(int64_t B, int C, int64_t T, int S, int padtype, int64_t padlen);
int b2a_sos_filtfilt_f32(const float* x, const float* gain, int64_t B, int C, int64_t T, const float* sos,
                         int64_t sos_items, int S, int padtype, int64_t padlen, float* out, void* ws, void* stream);
/* The gradient of b2a_sos_filtfilt_f32 with respect to x for the upstream gradient grad_y [B, C, T]: the adjoints of
 * the two passes, the rank-one terms of their start states and the fold of the edge extension.  Same arguments and
 * workspace; grad_x may alias grad_y.  Seven launches, no host sync. */
int b2a_sos_filtfilt_backward_f32(const float* grad_y, const float* gain, int64_t B, int C, int64_t T,
                                  const float* sos, int64_t sos_items, int S, int padtype, int64_t padlen,
                                  float* grad_x, void* ws, void* stream);

/* ---- shoebox-room impulse responses by the image-source method (csrc/rir.cu) ----------------------------------------
 * The impulse responses from item b's source to its microphone c (DESIGN.md K20), in K octave bands; K = 1 is the
 * frequency-flat room.  Geometry is float64 on the device: room [B, 3] (Lx, Ly, Lz, metres), src [B, 3],
 * mics [B, C, 3], beta [B, 6, K] (reflection coefficients of the walls x = 0, x = Lx, y = 0, y = Ly, z = 0, z = Lz;
 * band k, centred on 125 2^k Hz, uses beta[b, :, k]).  fs in [125, 384000] Hz, c > 0 m/s; max_order >= 0 keeps images
 * of at most that order, -1 keeps every image that reaches the first L samples.  Each image adds g h(i - d) at the
 * Tw = 2 floor(0.004 fs + 1/2) samples around its distance d (samples), h a Hann-windowed sinc.
 *
 * air [B, K] (dB/m, float64) or null: every image of band k is also scaled by 10^(-air[b, k] d / 20) (d in metres)
 * and the tail's envelope by 10^(-air[b, k] (c n / fs) / 10).
 *
 * t_d [B] (float64 seconds > 0) and seed [B] (uint64), both on the device or both null, add a diffuse late tail
 * (DESIGN.md K20, "Hybrid"): the images with floor(d) < min(L, n_d), n_d = ceil(t_d[b] fs), then, at every sample
 * n >= n_d - Tw/2, w(n) sqrt(E_b(n)) xi(seed[b], c, n): E_b the expected energy per sample of the image arrivals of
 * item b's room, w a raised-cosine ramp over the Tw samples centred on n_d, xi a standard normal from a stateless
 * counter-based generator (SplitMix64, Box-Muller) shared by the bands.  Every image order is kept: max_order must be
 * -1 with a tail.
 *
 * Only the first K' = b2a_rir_bands_kept(K, fs) bands are computed: those whose lower crossover 125 2^(k - 1/2) Hz is
 * below fs / 2 (DESIGN.md K20, "Bands").  out [K', B, C, L] float32, band-major: row k < K' - 1 holds r_k - r_{k+1},
 * row K' - 1 holds r_{K'-1}, r_k the band's response before the crossovers.  The images are enumerated once for all
 * bands; with equal bands and no air the differences are exactly 0 and r_{K'-1} is the K = 1 output, bit for bit.
 *
 * 1 <= K <= 8, B C K <= 65535, L <= 2^30; the arguments are not checked against each other (positions inside the room,
 * beta in [0, 1]): core/room.py does that.  One launch, two with a tail; no host sync, no atomics: reruns and a batch
 * against its items one at a time are bit-identical. */
int b2a_rir_bands_kept(int K, double fs);
int b2a_rir_f32(const double* room, const double* src, const double* mics, const double* beta, const double* air,
                const double* t_d, const uint64_t* seed, int64_t B, int C, int K, int64_t L, double fs, double c,
                int max_order, float* out, void* stream);
/* b2a_rir_f32 with first-order directivity (DESIGN.md K20, "Directivity"); with both tables null it is
 * b2a_rir_f32, bit for bit and through the same kernels.  mic_dir [B, C, 4] and src_dir [B, 4] (float64 on the device,
 * each null for an omnidirectional end) hold (p, v_x, v_y, v_z): the pattern p in [0, 1] and a unit orientation v.  Its
 * amplitude gain for a unit direction u is D(u) = p + (1 - p) u.v (p = 1: omni, 1/2: cardioid, 0: figure-eight; it
 * may be negative).  An image with offset (X, Y, Z) = image - microphone and parities (q, j, k) (odd numbers of
 * reflections on the x, y, z walls) is scaled by D_m((X, Y, Z) / d) D_s(-((1-2q) X, (1-2j) Y, (1-2k) Z) / d), the
 * microphone's pattern at the direction the sound arrives from and the source's at the direction it left in, the same
 * in every band; the tail's envelope becomes the expected energy of those scaled arrivals.  The tables are not read on
 * the host, so their sizes and the p and unit-vector conditions are the caller's (core/room.py checks them).  The
 * same launches as b2a_rir_f32. */
int b2a_rir_directional_f32(const double* room, const double* src, const double* mics, const double* beta,
                            const double* air, const double* t_d, const uint64_t* seed, const double* mic_dir,
                            const double* src_dir, int64_t B, int C, int K, int64_t L, double fs, double c,
                            int max_order, float* out, void* stream);

/* y[b, c] = bands[n_conv, b, c] + sum_{k < n_conv} conv[k, b, c] (added in k order): the crossover outputs of the
 * octave-band differences added to the last band (bands [n_conv + 1, B, C, L] from b2a_rir_f32, conv [n_conv, B,
 * C, L]).  Samples before the first one any band can reach through crossovers of half-length `half` (the direct path's
 * window, or with t_d the tail's start, less half and one sample) are written as 0.  1 <= n_conv < 8.  One launch. */
int b2a_rir_band_sum_f32(const double* src, const double* mics, const double* t_d, int64_t B, int C, int64_t L,
                         double fs, double c, int half, const float* bands, const float* conv, int n_conv, float* out,
                         void* stream);

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
/* A moving impulse response: b2a_circconv_f32 along a path of K waypoints, waypoint k at sample tau_k = k hop.
 *   out[row][t] = s sum_k v_k(t) sum_j h_{i,k}[j] x[row][(t - j + idx) mod T],   i = row / rows_per_ir,
 * v_k(t) = max(0, 1 - |t - tau_k| / hop), except v_{K-1}(t) = 1 for t >= tau_{K-1}: the weights sum to 1.  idx and s
 * are b2a_circconv_f32's roll and scale of waypoint 0's IR and serve the whole path, so a change in delay along it
 * is kept.  ir: [items][K][ir_channels][L] with items = rows / (rows_per_ir ir_channels) and IR i = item ir_channels
 * + c, so h_{i,k} = ir[item][k][c]; L <= T; hop >= 1024 (the engine's block: a block then meets at most 3
 * waypoints); K = (T - 1) / hop + 1 exactly; K <= 65535 and K ir_channels L < 2^31.  bypass: nullable
 * [rows / rows_per_ir], rows copied through.  No host sync, no atomics: rows are independent and reruns are
 * bit-identical.  With K = 1 and L > 1024 the output is b2a_circconv_f32's bit for bit.  out must not alias x.
 * ws: b2a_circconv_path_workspace_bytes() bytes. */
size_t b2a_circconv_path_workspace_bytes(int64_t rows, int64_t T, int64_t K, int64_t L, int rows_per_ir,
                                         int ir_channels, int hop);
int b2a_circconv_path_f32(const float* x, int64_t rows, int64_t T, const float* ir, int64_t K, int64_t L,
                          int rows_per_ir, int ir_channels, int hop, int roll_to_peak, const int32_t* bypass,
                          float* out, void* ws, size_t ws_bytes, void* stream);

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
 * One call takes one shift or several (a batch whose items drew different shifts, e.g. a PitchShift transform):
 * semitones_h HOST [n_groups] (n_groups <= 8 distinct values, 0 = copy the row), row_group DEVICE [rows] int32
 * in [0, n_groups) (nullable when n_groups == 1).  Rows of all groups share every launch, so the one-CTA-per-row
 * search fills the GPU with the whole batch instead of one group at a time.  Four launches.
 * ws: 16-byte aligned, b2a_pitch_shift_multi_workspace_bytes() bytes (frame positions + the stretched rows). */
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

/* Stub left from the removed tensor-core spectral kernel, which was slower and less accurate than the FP32 kernel.
 * bench.py --tc still calls it.  Returns 0 for on == 0 and B2A_E_UNSUPPORTED for any other value; b2a_spectral_f32
 * runs the FP32 kernels either way. */
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

/* ---- backward of b2a_stoi_f32 with respect to the estimates (metrics.quality.STOILoss; the references are constants)
 *   grad_score  [batch] float64 dL/dscore
 *   fwd_ws      the workspace b2a_stoi_f32 filled for the same est, ref, batch, channels, T, taps, up, down and left
 *               untouched since (its 10 kHz signals, kept-frame lists and counts and band envelopes are read);
 *               fwd_ws_bytes >= b2a_stoi_workspace_bytes(batch, T, up, down)
 *   grad_est    [batch, channels, T] float32 dL/dest; exactly 0 for an item scored 1e-5 (fewer than 30 STFT frames)
 *               and for samples that only dropped (silent) frames cover
 *   ws          b2a_stoi_backward_workspace_bytes(batch, T, up, down) bytes.  With n10 = ceil(T up / down) and
 *               n_fr = ceil((n10 - 256) / 128) (0 when n10 <= 256), each part rounded up to 256 bytes:
 *                 1800 batch n_fr   (per-cell derivatives, float [n_fr][15][30])
 *               +  120 batch n_fr   (dL/d band envelope, float64 [15][n_fr])
 *               +    4 batch n_fr   (frame -> kept position, int32)
 *               + 1024 batch n_fr   (dL/d STOI frame, float [n_fr][256])
 *               +    4 batch n10    (dL/d 10 kHz estimate, float)
 * Arguments are checked as b2a_stoi_f32 checks them (messages prefixed "stoi_backward:"), plus the forward workspace's
 * size; B2A_E_UNSUPPORTED when the transposed FIR's tile (1024 inputs) needs more than 200 KB of shared memory.  Four
 * launches (three when n10 <= 384), no atomics: bit-identical reruns. */
size_t b2a_stoi_backward_workspace_bytes(int64_t batch, int64_t T, int up, int down);
int b2a_stoi_backward_f32(const double* grad_score, const void* fwd_ws, size_t fwd_ws_bytes, int64_t batch,
                          int channels, int64_t T, int extended, const double* taps, int n_taps, int up, int down,
                          float* grad_est, void* ws, size_t ws_bytes, void* stream);

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
