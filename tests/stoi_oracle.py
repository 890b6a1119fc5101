"""Float64 restatement of pystoi's ``stoi`` [3P-recall]: the arithmetic of pystoi (``stoi.py`` and ``utils.py`` of
its public source), restated in numpy because pystoi is not a dependency of this project.  It calls the real
``scipy.signal.resample_poly``, ``np.kaiser`` and ``np.hanning``.  It is the checker of ``metrics.quality.stoi``
(csrc/stoi.cu), never the thing shipped.

One deliberate difference: pystoi's extended mode adds ``EPS * randn`` to the segments before each normalisation of
``row_col_normalize``.  This restatement leaves that noise out, as the CUDA port does, so results are deterministic;
the noise only matters for a row or column that is exactly constant (there both give NaN instead of noise).
"""
import warnings

import numpy as np
from scipy.signal import resample_poly

EPS = np.finfo("float").eps
FS = 10000        # the rate STOI works at
N_FRAME = 256     # frame length (and the silence-removal frame)
HOP = N_FRAME // 2
NFFT = 512
NUMBAND = 15      # third-octave bands
MINFREQ = 150     # centre of the lowest band
N = 30            # frames per segment (384 ms)
BETA = -15.0      # lower SDR bound of the clipping
DYN_RANGE = 40    # dB below the loudest frame that still count as speech


def thirdoct(fs=FS, nfft=NFFT, num_bands=NUMBAND, min_freq=MINFREQ):
    """[num_bands, nfft/2 + 1] 0/1 matrix of the third-octave bands, and the centre frequencies."""
    f = np.linspace(0, fs, nfft + 1)[: nfft // 2 + 1]
    k = np.arange(num_bands).astype(float)
    cf = 2.0 ** (k / 3) * min_freq
    lo = min_freq * 2.0 ** ((2 * k - 1) / 6)
    hi = min_freq * 2.0 ** ((2 * k + 1) / 6)
    obm = np.zeros((num_bands, len(f)))
    for i in range(num_bands):
        a = np.argmin(np.square(f - lo[i]))
        b = np.argmin(np.square(f - hi[i]))
        obm[i, a:b] = 1
    return obm, cf


OBM, CF = thirdoct()


def band_edges():
    """The 16 bin edges of the contiguous bands: band k covers bins [edges[k], edges[k + 1])."""
    lo = [int(np.argmax(r)) for r in OBM]
    hi = [int(len(r) - np.argmax(r[::-1])) for r in OBM]
    assert lo[1:] == hi[:-1], "the bands are contiguous"
    return lo + [hi[-1]]


def resample_window_oct(p, q):
    """The anti-aliasing filter of Octave's ``resample`` for the ratio p / q (60 dB Kaiser-windowed sinc)."""
    g = np.gcd(p, q)
    p, q = p // g, q // g
    stopband_cutoff_f = 1.0 / (2 * max(p, q))
    roll_off_width = stopband_cutoff_f / 10
    rejection_db = 60.0
    L = np.ceil((rejection_db - 8) / (28.714 * roll_off_width))
    t = np.arange(-L, L + 1)
    ideal = 2 * p * stopband_cutoff_f * np.sinc(2 * stopband_cutoff_f * t)
    return np.kaiser(2 * L + 1, 0.1102 * (rejection_db - 8.7)) * ideal


def resample_oct(x, p, q):
    h = resample_window_oct(p, q)
    return resample_poly(x, p, q, window=h / h.sum())


def _frames(x):
    w = np.hanning(N_FRAME + 2)[1:-1]
    return np.array([w * x[i:i + N_FRAME] for i in range(0, len(x) - N_FRAME, HOP)])


def remove_silent_frames(x, y):
    """(x, y with the frames more than DYN_RANGE dB below x's loudest removed, overlap-added; kept-frame count)."""
    xf, yf = _frames(x), _frames(y)
    if len(xf) == 0:
        raise ValueError("stoi: the signal has no full 256-sample frame at 10 kHz")
    e = 20 * np.log10(np.linalg.norm(xf, axis=1) + EPS)
    mask = (np.max(e) - DYN_RANGE - e) < 0
    xf, yf = xf[mask], yf[mask]
    n = (len(xf) - 1) * HOP + N_FRAME
    xs, ys = np.zeros(n), np.zeros(n)
    for i in range(len(xf)):
        xs[i * HOP:i * HOP + N_FRAME] += xf[i]
        ys[i * HOP:i * HOP + N_FRAME] += yf[i]
    return xs, ys, int(mask.sum()), e


def _row_col_normalize(x):
    x = x - x.mean(axis=-1, keepdims=True)
    x = x / np.sqrt(np.sum(x ** 2, axis=-1, keepdims=True))
    x = x - x.mean(axis=1, keepdims=True)
    return x / np.sqrt(np.sum(x ** 2, axis=1, keepdims=True))


def stoi_detail(x, y, fs_sig, extended=False):
    """pystoi.stoi(x, y, fs_sig, extended) with x the clean signal -> (score, kept frames, STFT frames M)."""
    x, y = np.asarray(x), np.asarray(y)
    if x.shape != y.shape:
        raise ValueError(f"stoi: x and y should have the same length, found {x.shape} and {y.shape}")
    if fs_sig != FS:
        x, y = resample_oct(x, FS, fs_sig), resample_oct(y, FS, fs_sig)
    x, y, kept, _ = remove_silent_frames(x, y)
    xf, yf = _frames(x), _frames(y)
    M = len(xf)
    if M < N:
        warnings.warn("Not enough STFT frames to compute intermediate intelligibility measure after removing silent "
                      "frames. Returning 1e-5. Please check you wav files", RuntimeWarning)
        return 1e-5, kept, M
    x_tob = np.sqrt(OBM @ np.square(np.abs(np.fft.rfft(xf, n=NFFT).T)))
    y_tob = np.sqrt(OBM @ np.square(np.abs(np.fft.rfft(yf, n=NFFT).T)))
    xs = np.array([x_tob[:, m - N:m] for m in range(N, M + 1)])
    ys = np.array([y_tob[:, m - N:m] for m in range(N, M + 1)])
    if extended:
        xn, yn = _row_col_normalize(xs), _row_col_normalize(ys)
        return float(np.sum(xn * yn / N) / xn.shape[0]), kept, M
    c = np.linalg.norm(xs, axis=2, keepdims=True) / (np.linalg.norm(ys, axis=2, keepdims=True) + EPS)
    yp = np.minimum(ys * c, xs * (1 + 10 ** (-BETA / 20)))
    yp = yp - yp.mean(axis=2, keepdims=True)
    xs = xs - xs.mean(axis=2, keepdims=True)
    yp /= np.linalg.norm(yp, axis=2, keepdims=True) + EPS
    xs /= np.linalg.norm(xs, axis=2, keepdims=True) + EPS
    return float(np.sum(yp * xs) / (xs.shape[0] * xs.shape[1])), kept, M


def stoi(x, y, fs_sig, extended=False):
    """pystoi.stoi: the STOI (or extended STOI) of the processed signal y against the clean signal x."""
    return stoi_detail(x, y, fs_sig, extended)[0]


def batch_stoi(estimates, references, sample_rate, extended=False):
    """The reference's ``metrics.quality.stoi`` on [B, C, T] float32 tensors or arrays: to_mono (float32 mean over
    channels), then this module's ``stoi_detail`` per item in a Python loop -> (scores [B], kept [B], M [B])."""
    est = np.asarray(estimates, dtype=np.float32).mean(axis=1, dtype=np.float32)
    ref = np.asarray(references, dtype=np.float32).mean(axis=1, dtype=np.float32)
    out = [stoi_detail(ref[i], est[i], sample_rate, extended) for i in range(est.shape[0])]
    return tuple(np.array(v) for v in zip(*out))


class _Module:
    """``sys.modules["pystoi"]`` for running the reference's wrapper against this restatement."""
    stoi = staticmethod(stoi)
