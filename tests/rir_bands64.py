"""Float64 oracle of the octave bands of ``core.room.image_source_ir(..., bands=K, air_absorption=)`` (csrc/rir.cu,
DESIGN.md K20 "Bands"), written from the definition: per band, ``tests/rir64.py``'s images and
``tests/rir_diffuse64.py``'s tail with the band's beta, every image gain times 10^(-a_k d / 20) (d in metres) and the
tail's envelope times 10^(-a_k (c n / fs) / 10); then y = r_{K'-1} + sum_{k < K'-1} LP_k * (r_k - r_{k+1}) with LP_k
the zero-phase low-pass at e_k = 125 2^(k + 1/2) Hz, the signal zero outside [0, L).

``combine`` takes the taps as given: the tests pass the library's float32 taps cast to float64, which separates the
kernels' error from the tap design; ``lowpass64`` is the float64 design those taps are checked against.
"""
import math

import numpy as np

from tests import rir64
from tests import rir_diffuse64 as D

U = rir64.U


def crossover(k: int) -> float:
    """e_k in Hz: the crossover between bands k and k + 1."""
    return 125.0 * 2.0 ** (k + 0.5)


def kept(K: int, fs: float) -> int:
    """K': band 0 and the bands whose lower crossover e_{k-1} is below fs / 2."""
    return 1 + sum(1 for k in range(1, K) if crossover(k - 1) < fs / 2)


def half0(fs: float) -> int:
    """The crossovers' shared half-length: julius.SplitBands(zeros=8) for its lowest cutoff e_0 / fs."""
    return int(8 / (crossover(0) / fs) / 2)


def lowpass64(fs: float, n: int) -> np.ndarray:
    """[n, 2 half0 + 1] float64 correlation taps of the windowed-sinc low-passes at e_k / fs, k < n, each normalised
    to a unit sum (julius.LowPassFilters' design)."""
    h = half0(fs)
    t = np.arange(-h, h + 1, dtype=np.float64)
    win = 0.5 - 0.5 * np.cos(2 * math.pi * np.arange(2 * h + 1) / (2 * h))
    out = []
    for k in range(n):
        c = crossover(k) / fs
        f = 2 * c * win * np.sinc(2 * c * t)
        out.append(f / f.sum())
    return np.array(out).reshape(n, 2 * h + 1)


def band_images(room, src, mic, beta_k, air_k: float, fs: float, L: int, max_order: int = -1, c: float = 343.0):
    """(d, g) of one band's images with floor(d) < L: rir64's gains times 10^(-air_k d_m / 20)."""
    d, g, _ = rir64.images(room, src, mic, beta_k, fs, L, max_order, c)
    return d, g * 10.0 ** (-air_k * (d * c / fs) / 20.0)


def band(room, src, mic, beta_k, air_k: float, fs: float, L: int, max_order: int = -1, td=None, seed=None,
         ch: int = 0, c: float = 343.0):
    """(r [L], G [L], tail [L], tail scale [L]) of one band of one microphone: r = images (+ tail); G the images'
    per-sample bound (rir64.bound); the tail and sqrt(E) times the Box-Muller radius, both with the air's factor."""
    Tw = rir64.window(fs)
    lim = L if td is None else min(L, D.n_diffuse(td, fs))
    d, g = band_images(room, src, mic, beta_k, air_k, fs, lim, max_order, c)
    r, G = rir64.render(d, g, Tw, L), rir64.bound(d, g, Tw, L)
    tail, scale = np.zeros(L), np.zeros(L)
    if td is not None:
        tail, scale = D.tail(room, beta_k, fs, L, td, seed, ch, c)
        att = 10.0 ** (-air_k * (np.arange(L) * c / fs) / 20.0)
        tail, scale = tail * att, scale * att
    return r + tail, G, tail, scale


def conv_centred(x: np.ndarray, f: np.ndarray) -> np.ndarray:
    """y[n] = sum_j f[j] x[n + j - h] (correlation taps f of length 2h + 1), x zero outside [0, L)."""
    h = (len(f) - 1) // 2
    L = len(x)
    return np.convolve(x, f[::-1], mode="full")[h:h + L]


def combine(r: np.ndarray, taps: np.ndarray) -> np.ndarray:
    """y = r[-1] + sum_k conv_centred(r[k] - r[k + 1], taps[k]) for r [K', L] and correlation taps [K' - 1, 2h + 1]."""
    y = r[-1].copy()
    for k in range(len(r) - 1):
        y += conv_centred(r[k] - r[k + 1], taps[k])
    return y


def spread(w: np.ndarray, taps: np.ndarray) -> np.ndarray:
    """The per-sample bound of ``combine`` for per-band bounds w [K', L]: sum_k |LP_k| * (w_k + w_{k+1}) + w_{K'-1}."""
    out = w[-1].copy()
    for k in range(len(w) - 1):
        out += conv_centred(w[k] + w[k + 1], np.abs(taps[k]))
    return out


def first_zero_end(src, mic, fs: float, td=None, c: float = 343.0) -> float:
    """Samples n below this are exactly 0: the direct path's distance - Tw/2 - half0 (or the tail's first sample -
    half0 when earlier), less one sample for the rounding of the distance."""
    Tw, h = rir64.window(fs), half0(fs)
    d = float(np.linalg.norm((np.asarray(src, np.float64) - np.asarray(mic, np.float64)) * fs / c))
    z = d - Tw // 2 - h - 1
    if td is not None:
        z = min(z, max(D.n_diffuse(td, fs) - Tw // 2, 0) - h - 1)
    return z
