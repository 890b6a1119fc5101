"""Float64 references and the per-sample / per-block error model of the time-domain accuracy tests
(tests/test_gpu_timedomain_accuracy.py on the H100, tests/test_sim_timedomain_accuracy.py on the simulator).

Every reference takes the kernel's exact float32 inputs (samples, taps, coefficients) and evaluates the formula in the
kernel's header in float64: direct sums where affordable, numpy's float64 FFT for long filters (its ~1e-15 relative
error is far below any budget here).  Errors are measured where they arise, never over a whole tensor:

* direct sums (``fir_direct_kernel``, ``resample_kernel``): e_n = |y^_n - y_n| / a_n with a_n = sum_k |h_k| |x_{n,k}|,
  the sum of the magnitudes of the products the output adds up.  Any FP32 summation order keeps e_n <= gamma_K ~ K u;
  rounding errors of random sign give ~ sqrt(K) u.  Budget C u sqrt(K).
* overlap-save (``fftconv``, circconv): per 1024-sample output block, max |y^ - y| / (||h||_2 rms(x over the span the
  block reads)).  Budget C u log2(2048) sqrt(P) with P the number of 1024-tap partitions.
* K-weighting: per 400 ms block, |z^_j - z_j| / z_j, with z_j floored at 1e-6 of the row's loudest block (-60 dB).
  Budget ``kweight_budget(rate, signal)`` u, and at most KW_VS_SEQ32 times the error of the sequential float32 cascade (the
  reference's torchaudio ``lfilter``) on the same input.

u = 2^-24.  The constants C are set once from the H100 measurement in DESIGN.md ("Time-domain accuracy") with about 2x
headroom over the worst case measured there and on the simulator."""
import math

import numpy as np
import scipy.signal as ss
import torch

U = 2.0 ** -24

BUDGET_C = {
    "fir_direct": 2.0,  # e_n / (u sqrt K)
    "resample": 2.0,    # e_n / (u sqrt K)
    "fftconv": 5.0,     # block error / (u log2 2048 sqrt P)
    "circconv": 5.0,    # as fftconv
}
# K-weighting per-block budget in u by kind of signal, up to 48 kHz; above, it grows as rate^2 (a state error is
# amplified by the high-pass's ~1 / (1 - rho)^2, and 1 - rho ~ 1 / rate).  About 2x the worst measured on the H100 (and
# on the simulator, which rounds as the GPU does): noise 11 u; DC steps and 20-60 Hz tones 596 u (DC, 44.1 kHz); a row
# falling by 100 dB 45 130 u (44.1 kHz: the block that starts at the drop holds only the filter's ringing, ~1e-5 of the
# loud blocks, against the loud part's rounding; the sequential float32 cascade: 31 415 u).
KW_BUDGET = {"noise": 24.0, "bass": 1280.0, "drop": 98304.0}
# ours / the sequential float32 cascade, worst block of a row: measured <= 1.0 on noise, DC steps and 20-60 Hz tones at
# every rate.  The exception is the block that starts at a 100 dB drop: it holds only the ringing (~1e-5 of the loud
# blocks), and the lane start states after the drop carry float32 rounding of the loud state summed over the scan;
# measured up to 11.7x (22.05 kHz, drop at 0.6 s), 1.4x at 44.1 kHz.  It gets its own factor.
KW_VS_SEQ32 = 2.0
KW_DROP_VS_SEQ32 = 24.0
KW_FLOOR = 1e-6  # blocks below -60 dB of the row's loudest block are measured against that floor

DIRECT_FIR_MAX_TAPS = 320
FFT_BLOCK = 1024


# --------------------------------------------------------------------------- routes
def fir_route(lib, T: int, K: int, stride: int = 1) -> str:
    """The kernel ``Engine.sinc_filter`` launches for a K-tap filter on rows of T samples (stride 1)."""
    return "fir_direct" if K <= DIRECT_FIR_MAX_TAPS and lib.b2a_fir_direct_supported(T, K, stride) else "fftconv"


def resample_route(lib, T: int, old_sr: int, new_sr: int) -> str:
    """The kernel ``Engine.resample`` launches: the decimating ``fir_direct`` when the reduced new rate is 1."""
    g = math.gcd(old_sr, new_sr)
    old, new = old_sr // g, new_sr // g
    K = 2 * resample_width(old_sr, new_sr) + old
    return "fir_direct" if new == 1 and lib.b2a_fir_direct_supported(T, K, old) else "resample"


def resample_width(old_sr: int, new_sr: int, zeros: int = 24, rolloff: float = 0.945) -> int:
    g = math.gcd(old_sr, new_sr)
    old, new = old_sr // g, new_sr // g
    return math.ceil(zeros * old / (min(new, old) * rolloff))


# --------------------------------------------------------------------------- extension of a row
def extend_index(idx: np.ndarray, T: int, pad_mode: str):
    """(index into x, valid mask) of xv[idx] for xv = x extended by ``pad_mode``."""
    if pad_mode == "replicate":
        return np.clip(idx, 0, T - 1), np.ones(idx.shape, bool)
    if pad_mode == "circular":
        return np.mod(idx, T), np.ones(idx.shape, bool)
    assert pad_mode == "constant", pad_mode
    return np.clip(idx, 0, T - 1), (idx >= 0) & (idx < T)


def _np64(t):
    return t.detach().cpu().double().numpy() if isinstance(t, torch.Tensor) else np.asarray(t, np.float64)


# --------------------------------------------------------------------------- direct sums
def fir_direct64(x, taps, rows_per_filt: int, left=None, left0: int = 0, stride: int = 1, out_len=None,
                 pad_mode: str = "replicate", subtract: bool = False, bypass=None):
    """(y, a) [rows, out_len] float64 of fir.cu:3,
    out[row][m] = sum_k taps[f][k] xv[row][m stride + k - left0 - left[f]]   (x - out when ``subtract``),
    and a = sum_k |taps[f][k]| |xv[...]| (plus |x| when ``subtract``).  Bypassed filters copy their rows."""
    x = _np64(x)
    x = x.reshape(-1, x.shape[-1])
    taps = _np64(taps)
    rows, T = x.shape
    n_filt, K = taps.shape
    out_len = T if out_len is None else out_len
    left = np.zeros(n_filt, np.int64) if left is None else _np64(left).astype(np.int64).reshape(-1)
    y = np.zeros((rows, out_len))
    a = np.zeros((rows, out_len))
    m = np.arange(out_len)
    for r in range(rows):
        f = r // rows_per_filt
        if bypass is not None and bypass[f]:
            y[r], a[r] = x[r, :out_len], np.abs(x[r, :out_len])
            continue
        idx = m[:, None] * stride + np.arange(K)[None, :] - left0 - left[f]
        i, ok = extend_index(idx, T, pad_mode)
        xv = np.where(ok, x[r][i], 0.0)
        y[r] = xv @ taps[f]
        a[r] = np.abs(xv) @ np.abs(taps[f])
        if subtract:
            y[r] = x[r, :out_len] - y[r]
            a[r] += np.abs(x[r, :out_len])
    return y, a


def resample64(x, old_sr: int, new_sr: int, kt):
    """(y, a) [rows, out_len] float64 of resample.cu:5 with the engine's float32 kernel ``kt`` [K, new]:
    out[m new + i] = sum_k kernel[i][k] x[clamp(m old + k - width, 0, T-1)], the first floor(new T / old) kept."""
    g = math.gcd(old_sr, new_sr)
    old, new = old_sr // g, new_sr // g
    width = resample_width(old_sr, new_sr)
    kern = _np64(kt).T  # [new, K]
    x = _np64(x)
    x = x.reshape(-1, x.shape[-1])
    T = x.shape[-1]
    out_len = new * T // old
    n = np.arange(out_len)
    mm, ii = n // new, n % new
    idx = np.clip(mm[:, None] * old + np.arange(kern.shape[1])[None, :] - width, 0, T - 1)
    xv = x[:, idx]                       # [rows, out_len, K]
    w = kern[ii]                          # [out_len, K]
    return np.einsum("rnk,nk->rn", xv, w), np.einsum("rnk,nk->rn", np.abs(xv), np.abs(w))


def direct_errors(got, y, a):
    """e_n = |y^_n - y_n| / a_n (0 where a_n = 0 and the output is exact, inf where it is not)."""
    d = np.abs(_np64(got).reshape(y.shape) - y)
    return np.where(a > 0, d / np.maximum(a, 1e-300), np.where(d > 0, np.inf, 0.0))


def direct_budget(route: str, K: int) -> float:
    return BUDGET_C[route] * U * math.sqrt(K)


# --------------------------------------------------------------------------- overlap-save
def fftconv64(x, taps, rows_per_filt: int, offset=None, offset0: int = 0, pad_mode: str = "replicate",
              post_scale=None, subtract: bool = False, bypass=None):
    """(y, scale) [rows, T] float64 of fftconv.cu:13,
    out[row][n] = post[f] sum_k g[f][k] xv[row][n - k + offset0 + offset[f]]   (x - out when ``subtract``),
    by numpy's float64 FFT of the extended span; ``scale`` [rows, n_blocks] = ||g_f||_2 |post_f| rms(xv over the
    samples the transform frames behind block b read) (+ rms of x over the block when ``subtract``)."""
    x = _np64(x)
    x = x.reshape(-1, x.shape[-1])
    g = _np64(taps)
    rows, T = x.shape
    n_filt, L = g.shape
    off = np.zeros(n_filt, np.int64) if offset is None else _np64(offset).astype(np.int64).reshape(-1)
    post = np.ones(n_filt) if post_scale is None else _np64(post_scale).reshape(-1)
    nb = (T + FFT_BLOCK - 1) // FFT_BLOCK
    y = np.zeros((rows, T))
    scale = np.zeros((rows, nb))
    nfft = 1 << (T + L - 1).bit_length()
    for r in range(rows):
        f = r // rows_per_filt
        if bypass is not None and bypass[f]:
            y[r] = x[r]
            scale[r] = [np.sqrt(np.mean(x[r, b * FFT_BLOCK:(b + 1) * FFT_BLOCK] ** 2)) for b in range(nb)]
            continue
        c = offset0 + off[f]
        # xv[j + c - (L-1)], j in [0, T + L - 1): out[n] = sum_k g[k] xv[n + (L-1) - k + c - (L-1)]
        i, ok = extend_index(np.arange(T + L - 1) + c - (L - 1), T, pad_mode)
        xv = np.where(ok, x[r][i], 0.0)
        full = np.fft.irfft(np.fft.rfft(xv, nfft) * np.fft.rfft(g[f], nfft), nfft)
        y[r] = post[f] * full[L - 1:L - 1 + T]
        hn = np.sqrt(np.sum(g[f] ** 2)) * abs(post[f])
        # the 2048-sample transform frames behind block b also read the 1024 samples in front of its span and the
        # extension past the row's end
        i, ok = extend_index(np.arange(-FFT_BLOCK, (nb + 1) * FFT_BLOCK + L - 1) + c - (L - 1), T, pad_mode)
        xe = np.where(ok, x[r][i], 0.0)
        for b in range(nb):
            span = xe[b * FFT_BLOCK:(b + 2) * FFT_BLOCK + L - 1]
            scale[r, b] = hn * np.sqrt(np.mean(span ** 2))
        if subtract:
            y[r] = x[r] - y[r]
            scale[r] += [np.sqrt(np.mean(x[r, b * FFT_BLOCK:(b + 1) * FFT_BLOCK] ** 2)) for b in range(nb)]
    return y, scale


def block_errors(got, y, scale):
    """[rows, n_blocks]: max |y^ - y| over each 1024-sample output block / the block's scale."""
    d = np.abs(_np64(got).reshape(y.shape) - y)
    rows, T = y.shape
    nb = scale.shape[1]
    dp = np.zeros((rows, nb * FFT_BLOCK))
    dp[:, :T] = d
    m = dp.reshape(rows, nb, FFT_BLOCK).max(-1)
    return np.where(scale > 0, m / np.maximum(scale, 1e-300), np.where(m > 0, np.inf, 0.0))


def fft_budget(route: str, L: int) -> float:
    P = max(1, (L + FFT_BLOCK - 1) // FFT_BLOCK)
    return BUDGET_C[route] * U * math.log2(2 * FFT_BLOCK) * math.sqrt(P)


def circconv_filters64(x, ir, roll_to_peak: bool = True):
    """The convolution taps circconv applies (fftconv.cu:338): the IR truncated to T, rolled so that its first peak
    (the first index of max |ir|) lands on sample 0, scaled by 1 / max(max |ir|, 1e-5); [n_ir, L] float64 with the
    offset [n_ir] that places the roll."""
    ir = _np64(ir)
    T = x.shape[-1]
    ir = ir.reshape(-1, ir.shape[-1])[:, :T]
    peak = np.abs(ir).max(-1)
    idx = np.argmax(np.abs(ir), -1) if roll_to_peak else np.zeros(ir.shape[0], np.int64)
    return ir / np.maximum(peak, 1e-5)[:, None], idx


def circconv64(x, ir, rows_per_ir: int, roll_to_peak: bool = True):
    """(y, scale) of the reference's convolve(): out[n] = sum_k ir_s[k] x[(n - k + idx) mod T]."""
    g, idx = circconv_filters64(x, ir, roll_to_peak)
    return fftconv64(x, g, rows_per_ir, offset=idx, pad_mode="circular")


# --------------------------------------------------------------------------- K-weighting
def kweight_coef(rate: float):
    """(b0, b1, b2, a1, a2) float64 arrays [NS] of the kernel's float32-rounded, a0-normalised coefficients with the
    stage gain folded into b (lufs.cu, ``run``)."""
    from audiotools_b200.core import kweighting

    sos, sg = kweighting.design(float(rate))
    f = np.float32
    cols = [[], [], [], [], []]
    for c, gs in zip(sos, sg):
        a0, g = f(c[3]), f(gs)
        for i in range(3):
            cols[i].append(float(f(f(f(c[i]) / a0) * g)))
        cols[3].append(float(f(f(c[4]) / a0)))
        cols[4].append(float(f(f(c[5]) / a0)))
    return tuple(np.array(c) for c in cols)


def kweight64(x, coef):
    """The biquad cascade in float64 along the last axis of x."""
    b0, b1, b2, a1, a2 = coef
    y = _np64(x)
    for s in range(len(b0)):
        y = ss.lfilter([b0[s], b1[s], b2[s]], [1.0, a1[s], a2[s]], y, axis=-1)
    return y


def kweight_seq32(x, coef):
    """The sequential float32 cascade of the reference (torchaudio ``lfilter`` per stage, clamp=False)."""
    import torchaudio

    b0, b1, b2, a1, a2 = coef
    y = torch.as_tensor(np.asarray(x, np.float32))
    for s in range(len(b0)):
        a = torch.tensor([1.0, a1[s], a2[s]], dtype=torch.float32)
        b = torch.tensor([b0[s], b1[s], b2[s]], dtype=torch.float32)
        y = torchaudio.functional.lfilter(y, a, b, clamp=False)
    return y.double().numpy()


def kweight_geometry(Tp: int, rate: float, block_s: float = 0.4):
    """(K, stride, nblk) of lufs.cu:503: K = int(block_s rate), stride = int(block_s rate / 4)."""
    kf = block_s * rate
    K, stride = int(kf), int(kf * 0.25)
    nblk = (max(Tp, K) - K + stride - 1) // stride + 1
    return K, stride, nblk


def kweight_blocks64(x, rate: float, Tp: int = None, filtered=None, block_s: float = 0.4):
    """z [..., nblk] float64: the energy of the K-weighted row (zero-padded to Tp) over each block / (block_s rate)."""
    x = _np64(x)
    T = x.shape[-1]
    Tp = T if Tp is None else Tp
    K, stride, nblk = kweight_geometry(Tp, rate, block_s)
    xp = np.zeros(x.shape[:-1] + (Tp,))
    xp[..., :T] = x
    y = kweight64(xp, kweight_coef(rate)) if filtered is None else filtered
    # the filtered row is zero-padded to the last block (julius.core.unfold)
    y = np.concatenate([y, np.zeros(y.shape[:-1] + (max(0, (nblk - 1) * stride + K - y.shape[-1]),))], -1)
    c = np.concatenate([np.zeros(y.shape[:-1] + (1,)), np.cumsum(y * y, -1)], -1)
    j = np.arange(nblk) * stride
    return (c[..., np.minimum(j + K, c.shape[-1] - 1)] - c[..., j]) / (block_s * rate)


def kweight_budget(rate: float, signal: str) -> float:
    """The per-block bound in u for a signal of tests/test_gpu_timedomain_accuracy.py ``kw_signals`` at a rate."""
    kind = "noise" if signal.startswith("noise") else ("drop" if signal.startswith("loud_then") else "bass")
    return KW_BUDGET[kind] * max(1.0, (rate / 48000.0) ** 2)


def kweight_vs_seq32(signal: str) -> float:
    """The allowed factor of the sequential float32 cascade's worst block for a signal of ``kw_signals``."""
    return KW_DROP_VS_SEQ32 if signal.startswith("loud_then") else KW_VS_SEQ32


def kweight_block_errors(got, z):
    """|z^_j - z_j| / max(z_j, KW_FLOOR max_j z_j) per block."""
    z = np.asarray(z)
    den = np.maximum(z, KW_FLOOR * z.max(-1, keepdims=True))
    return np.abs(_np64(got).reshape(z.shape) - z) / np.maximum(den, 1e-300)


def kweight_state_maps(coef, L2: int = 64):
    """(A, Wa): the cascade's state transition matrix [D, D] on (y1, y2) per stage, and the zero-state end state of a
    chunk of L2 samples as a linear map of its L2 + 2 inputs (two history samples first) [L2 + 2, D], float64."""
    b0, b1, b2, a1, a2 = coef
    NS = len(b0)
    D = 2 * NS

    def run(state, inputs):
        y1 = [state[2 * s] for s in range(NS)]
        y2 = [state[2 * s + 1] for s in range(NS)]
        for i in range(2, len(inputs)):
            in0, in1, in2 = inputs[i], inputs[i - 1], inputs[i - 2]
            for s in range(NS):
                y0 = b0[s] * in0 + b1[s] * in1 + b2[s] * in2 - a1[s] * y1[s] - a2[s] * y2[s]
                in0, in1, in2 = y0, y1[s], y2[s]
                y2[s], y1[s] = y1[s], y0
        return np.array([v for s in range(NS) for v in (y1[s], y2[s])])

    A = np.stack([run(np.eye(D)[k], np.zeros(3)) for k in range(D)], 1)
    Wa = np.stack([run(np.zeros(D), np.eye(L2 + 2)[j]) for j in range(L2 + 2)], 0)
    return A, Wa


def kweight_basis(coef):
    """P [D, D]: the kernel's state basis w = P (y1, y2), per stage (y1 - rho y2, y2) with rho the stage's largest
    pole radius rounded to float32 (lufs.cu, ``build_tables``)."""
    b0, b1, b2, a1, a2 = coef
    NS = len(b0)
    P = np.eye(2 * NS)
    for s in range(NS):
        P[2 * s, 2 * s + 1] = -float(np.float32(np.max(np.abs(np.roots([1.0, a1[s], a2[s]])))))
    return P


# --------------------------------------------------------------------------- adjoints
def _scatter_adjoint(g, idx, w, T):
    """(gx, a) [rows, T]: gx[j] = sum over (n, k) with idx[n, k] = j of w[n, k] g[n], a the same sum of magnitudes."""
    g = _np64(g).reshape(-1, idx.shape[0])
    gx = np.zeros((g.shape[0], T))
    a = np.zeros((g.shape[0], T))
    flat = idx.reshape(-1)
    for r in range(g.shape[0]):
        p = (g[r][:, None] * w).reshape(-1)
        np.add.at(gx[r], flat, p)
        np.add.at(a[r], flat, np.abs(p))
    return gx, a


def resample_backward64(g, T: int, old_sr: int, new_sr: int, kt):
    """(gx, a) [rows, T]: the adjoint of ``resample64`` applied to g [rows, out_len]."""
    gc = math.gcd(old_sr, new_sr)
    old, new = old_sr // gc, new_sr // gc
    width = resample_width(old_sr, new_sr)
    kern = _np64(kt).T
    n = np.arange(new * T // old)
    idx = np.clip((n // new)[:, None] * old + np.arange(kern.shape[1])[None, :] - width, 0, T - 1)
    return _scatter_adjoint(g, idx, kern[n % new], T)


def fir_backward64(g, taps, rows_per_filt: int, left0: int):
    """(gx, a) [rows, T]: the adjoint of the stride-1 replicate-padded correlation of ``fir_direct64`` (what
    ``equalizer_backward`` computes with ``fftconv`` + ``fir_pad_fold``)."""
    g = _np64(g)
    g = g.reshape(-1, g.shape[-1])
    taps = _np64(taps)
    rows, T = g.shape
    K = taps.shape[1]
    idx = np.clip(np.arange(T)[:, None] + np.arange(K)[None, :] - left0, 0, T - 1)
    out = [_scatter_adjoint(g[r:r + 1], idx, np.broadcast_to(taps[r // rows_per_filt], (T, K)), T) for r in range(rows)]
    return np.concatenate([o[0] for o in out]), np.concatenate([o[1] for o in out])


def circconv_backward64(g, ir, rows_per_ir: int, roll_to_peak: bool = True):
    """(gx, scale): the adjoint of ``circconv64``, gx[j] = sum_k ir_s[k] g[(j + k - idx) mod T], as the convolution
    with the reversed taps."""
    gs, idx = circconv_filters64(g, ir, roll_to_peak)
    L = gs.shape[1]
    return fftconv64(g, gs[:, ::-1].copy(), rows_per_ir, offset=L - 1 - idx, pad_mode="circular")
