"""Float64 restatement of the true-peak level of csrc/truepeak.cu (DESIGN.md K17), the oracle of
tests/test_sim_true_peak.py and tests/test_gpu_true_peak.py.

For a row x[0..T-1] at rate sr: L = 4 below 96 kHz, 2 below 192 kHz, else 1.  Phase 0 is the sample itself; phase
p = 1 .. L-1 is y[n, p] = sum_{d=-6..5} h_p[d] x[n - d] (x = 0 outside the row) with
h_p[d] = sinc(u) (1 + cos(pi u / 6)) / 2, u = d + p / L.  The instants are every (n, p) with n < T - 1 plus (T - 1, 0);
the row's true peak is max |y| over them, the item's 20 log10 of the channel maximum."""
import numpy as np


def factor(sr: float) -> int:
    return 4 if sr < 96000 else 2 if sr < 192000 else 1


def design(L: int) -> np.ndarray:
    """[L - 1, 12] float64 taps: phase p at row p - 1, tap d = -6 .. 5 at column d + 6."""
    u = np.arange(-6, 6)[None, :] + np.arange(1, L)[:, None] / L
    return np.sinc(u) * 0.5 * (1.0 + np.cos(np.pi * u / 6.0))


def row_peaks(x: np.ndarray, taps: np.ndarray) -> np.ndarray:
    """Linear true peak of every row of x [..., T] (float64) with the taps [L - 1, 12] (the library's float32 taps,
    promoted, for the kernel comparisons)."""
    x = np.asarray(x, dtype=np.float64)
    shape, T = x.shape[:-1], x.shape[-1]
    rows = x.reshape(-1, T)
    out = np.abs(rows).max(axis=1)  # phase 0; NaN propagates
    if T > 1:
        for h in np.asarray(taps, dtype=np.float64):
            # y[n] = sum_m h[m] x[n + 6 - m] = full convolution at n + 6, n = 0 .. T - 2
            y = np.stack([np.convolve(r, h)[6:6 + T - 1] for r in rows])
            out = np.maximum(out, np.abs(y).max(axis=1))
    return out.reshape(shape)


def item_db(peaks: np.ndarray) -> np.ndarray:
    """[B, C] linear row peaks -> [B] dBTP."""
    with np.errstate(divide="ignore"):
        return 20.0 * np.log10(np.max(peaks, axis=1))


def true_peak_db(x: np.ndarray, sr: float) -> np.ndarray:
    """[B, C, T] -> [B] dBTP with the float64 design (the definition, for the accuracy checks)."""
    return item_db(row_peaks(x, design(factor(sr))))


def faded_sine(sr: float, f_rel: float, phase: float, amp: float = 1.0, seconds: float = 0.25,
               fade: float = 0.05) -> np.ndarray:
    """amp sin(2 pi f_rel n + phase) with raised-cosine fades of ``fade`` s at both ends (no edge ringing)."""
    T = int(seconds * sr)
    n = np.arange(T)
    x = amp * np.sin(2 * np.pi * f_rel * n + phase)
    nf = int(fade * sr)
    ramp = 0.5 * (1 - np.cos(np.pi * np.arange(nf) / nf))
    x[:nf] *= ramp
    x[T - nf:] *= ramp[::-1]
    return x
