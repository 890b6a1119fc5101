"""Float64 oracle of ``AudioSignal.apply_moving_ir`` / ``b2a_circconv_path_f32`` (DESIGN.md K22), written from the
definition: K circular convolutions of period T, every one with the roll and scale of the row's first waypoint
(``EffectMixin.convolve``'s rule), crossfaded in receiver time,

    y[t] = sum_k v_k(t) (h~_k (*)_T x)(t),   v_k(t) = max(0, 1 - |t - k hop| / hop),   v_{K-1}(t) = 1 for t >= (K-1) hop.

Each convolution is one length-T FFT product of x with the rolled IR wrapped onto the period, so long paths stay cheap.
"""
import numpy as np

from tests import timedomain64 as td


def path_weights(T: int, K: int, hop: int) -> np.ndarray:
    """v [K, T] float64: the crossfade weights of the waypoints."""
    t = np.arange(T)[None, :]
    tau = (np.arange(K) * hop)[:, None]
    v = np.maximum(0.0, 1.0 - np.abs(t - tau) / hop)
    v[K - 1, t[0] >= (K - 1) * hop] = 1.0
    return v


def _periodic_energy(x: np.ndarray):
    """S(n) = sum of x^2 over [0, n) of the T-periodic extension of the row x, for integer arrays n."""
    T = x.shape[-1]
    cs = np.concatenate([[0.0], np.cumsum(x ** 2)])
    return lambda n: (n // T) * cs[T] + cs[n % T]


def moving_ir64(x, irs, hop: int, roll_to_peak: bool = True, bypass=None):
    """(y, scale) [rows, T] / [rows, n_blocks] float64 for x [B, C, T] and irs [B, K, C or 1, L].

    ``scale`` is what ``timedomain64.fft_budget("circconv", min(L, T))`` is measured against: per waypoint, the
    overlap-save scale of ``timedomain64.fftconv64`` (the filter's 2-norm times the rms of the samples the transform
    frames behind the block read), times the waypoint's largest weight on the block, summed over the waypoints."""
    x = td._np64(x)
    irs = td._np64(irs)
    B, C, T = x.shape
    _, K, n_ch, L = irs.shape
    L = min(L, T)
    irs = irs[..., :L]
    rows_per_ir = 1 if n_ch == C else C
    first = irs[:, 0].reshape(B * n_ch, L)
    peak = np.maximum(np.abs(first).max(-1), 1e-5)
    idx = np.argmax(np.abs(first), -1) if roll_to_peak else np.zeros(B * n_ch, np.int64)
    v = path_weights(T, K, hop)
    nb = (T + td.FFT_BLOCK - 1) // td.FFT_BLOCK
    vp = np.zeros((K, nb * td.FFT_BLOCK))
    vp[:, :T] = v
    vmax = vp.reshape(K, nb, td.FFT_BLOCK).max(-1)  # [K, nb]
    xr = x.reshape(B * C, T)
    y = np.zeros((B * C, T))
    scale = np.zeros((B * C, nb))
    for r in range(B * C):
        i = r // rows_per_ir
        if bypass is not None and bypass[r // C]:
            y[r] = xr[r]
            continue
        X = np.fft.rfft(xr[r])
        energy = _periodic_energy(xr[r])
        # the transform frames behind block b read x[(b - 1) 1024 - (L - 1) + idx, (b + 1) 1024 + idx) (circular)
        start = (np.arange(nb) - 1) * td.FFT_BLOCK - (L - 1) + idx[i]
        n = 2 * td.FFT_BLOCK + L - 1
        rms = np.sqrt((energy(start + n) - energy(start)) / n)
        for k in range(K):
            g = irs[i // n_ch, k, i % n_ch] / peak[i]
            h = np.zeros(T)
            np.add.at(h, (np.arange(L) - idx[i]) % T, g)  # y[t] = sum_j g[j] x[(t - j + idx) mod T]
            y[r] += v[k] * np.fft.irfft(X * np.fft.rfft(h), T)
            scale[r] += vmax[k] * np.sqrt(np.sum(g ** 2)) * rms
    return y, scale


def keep_peak64(x, y):
    """apply_ir's last step: every row of y scaled back to the peak of the same row of x."""
    x = td._np64(x).reshape(y.shape)
    return y * np.maximum(np.abs(x).max(-1, keepdims=True), 1e-8) / np.maximum(np.abs(y).max(-1, keepdims=True), 1e-8)
