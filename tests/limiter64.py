"""Float64 restatement of the look-ahead true-peak limiter of csrc/limiter.cu (DESIGN.md K18), the oracle of
tests/test_sim_limiter.py and tests/test_gpu_limiter.py.  Sequential recursion, nothing shared with the kernels.

Input x [B, C, T] float32 (after the optional per-item gain: x = float32(g0 x)), the linear ceiling c [B], the
look-ahead A in samples, the release coefficient a (the float32 the library is given, promoted), and the true-peak
taps [L - 1, 12] of tests/truepeak64.py (the library's float32 taps, promoted, for the kernel comparisons).

1. envelope   y[n, p] as in truepeak64 (between samples n and n + 1; only n in [0, T - 1) exists);
              e_c[n] = max(|x[n]|, max_p |y[n, p]|, max_p |y[n - 1, p]|), e[n] = max_c e_c[n]
2. reduction  q[n] = 0 where e[n] <= c, else 1 - c / e[n]; NaN where e[n] is not finite
3. hold       h[n] = max of q[j] over |j - n| <= A, j in [0, T)
4. release    d[n] = max(h[n], a d[n - 1]), d[-1] = 0; afterwards d < 2^-26 counts as 0
5. attack     r[n] = mean of d[j] over |j - n| <= A, j in [0, T)  (divided by the number of such j)
6. output     out[c, n] = x[c, n] float32(1 - r[n])

Every maximum propagates NaN.  So a sample that is NaN or inf makes e non-finite at the samples whose interpolated
neighbours it reaches (at most 6 before, 6 after), h NaN from A before those, d NaN from there to the end of the row,
and r (hence every channel of the item's output) NaN from 2 A + 6 samples before the bad sample, at the earliest, on.
Other items are unaffected."""
import numpy as np

from tests import truepeak64 as tp

TINY = 2.0 ** -26
CHUNK = 4096  # samples of an item per CTA work item in csrc/limiter.cu


def envelope(x: np.ndarray, taps: np.ndarray) -> np.ndarray:
    """[B, C, T] -> e [B, T] float64."""
    x = np.asarray(x, dtype=np.float64)
    B, C, T = x.shape
    e = np.abs(x)
    taps = np.asarray(taps, dtype=np.float64)
    if T > 1 and len(taps):
        with np.errstate(invalid="ignore"):
            m = np.zeros((B, C, T - 1))
            for h in taps:
                y = np.stack([np.convolve(r, h)[6:6 + T - 1] for r in x.reshape(-1, T)]).reshape(B, C, T - 1)
                m = np.maximum(m, np.abs(y))
        e[..., :-1] = np.maximum(e[..., :-1], m)
        e[..., 1:] = np.maximum(e[..., 1:], m)
    out = e[:, 0]
    for c in range(1, C):
        out = np.maximum(out, e[:, c])
    return out


def reduction_needed(e: np.ndarray, c: np.ndarray) -> np.ndarray:
    c = np.asarray(c, dtype=np.float64).reshape(-1, 1)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(e <= c, 0.0, 1.0 - c / e)
    q[~np.isfinite(e)] = np.nan
    return q


def hold(q: np.ndarray, A: int) -> np.ndarray:
    """Centred maximum over 2 A + 1 samples, zeros outside the row (q >= 0)."""
    B, T = q.shape
    w = 2 * A + 1
    m = np.concatenate([np.zeros((B, A)), q, np.zeros((B, A))], axis=1)  # m[i] = q[i - A]
    L = 1
    while 2 * L <= w:  # m[i] = max over [i, i + L)
        m = np.maximum(m[:, :-L], m[:, L:])
        L *= 2
    n = np.arange(T)
    return np.maximum(m[:, n], m[:, n + w - L])


def release(h: np.ndarray, a: float) -> np.ndarray:
    a = float(a)
    d = np.empty_like(h)
    for b in range(h.shape[0]):
        prev, row = 0.0, []
        for v in h[b].tolist():
            t = a * prev
            prev = v if (v >= t or v != v) else t
            row.append(prev)
        d[b] = row
    with np.errstate(invalid="ignore"):
        d[d < TINY] = 0.0
    return d


def attack(d: np.ndarray, A: int) -> np.ndarray:
    B, T = d.shape
    P = np.concatenate([np.zeros((B, 1)), np.cumsum(d, axis=1)], axis=1)
    n = np.arange(T)
    lo, hi = np.maximum(n - A, 0), np.minimum(n + A, T - 1)
    with np.errstate(invalid="ignore"):
        r = (P[:, hi + 1] - P[:, lo]) / (hi - lo + 1)
    return np.maximum(r, 0.0)  # the prefix difference's rounding; NaN stays


def limit(x: np.ndarray, taps: np.ndarray, c, A: int, a: float, gain=None):
    """-> (out [B, C, T] float64, r [B, T] float64)."""
    x = np.asarray(x, dtype=np.float32)
    if gain is not None:
        x = x * np.asarray(gain, dtype=np.float32).reshape(-1, 1, 1)  # a float32 product, as the gain kernel's
    B = x.shape[0]
    c = np.broadcast_to(np.asarray(c, dtype=np.float64).reshape(-1), (B,))
    r = attack(release(hold(reduction_needed(envelope(x, taps), c), A), a), A)
    g = (1.0 - r).astype(np.float32).astype(np.float64)
    return x.astype(np.float64) * g[:, None, :], r


def params(sr: float, lookahead: float = 0.0015, release_s: float = 0.05):
    """(A, a): the look-ahead in samples and the float32 release coefficient."""
    return int(round(lookahead * sr)), float(np.float32(np.exp(-1.0 / (release_s * sr))))


def limit_db(x, sr, ceiling_db=-1.0, lookahead=0.0015, release_s=0.05, gain=None):
    """The definition end to end with the float64 design of the taps (the overshoot study)."""
    A, a = params(sr, lookahead, release_s)
    c = np.float32(10.0 ** (np.asarray(ceiling_db, dtype=np.float64) / 20.0))
    return limit(x, tp.design(tp.factor(sr)), c, A, a, gain)


# --------------------------------------------------------------------------- the test signals (closed form or seeded)
def clicks_on_noise(sr: float, seconds: float, n_clicks: int, seed: int, noise_db: float = -26.0,
                    click: float = 0.9) -> np.ndarray:
    """Gaussian noise at ``noise_db`` RMS with ``n_clicks`` single-sample clicks of alternating sign."""
    rng = np.random.default_rng(seed)
    T = int(seconds * sr)
    x = 10 ** (noise_db / 20) * rng.standard_normal(T)
    pos = rng.choice(T, n_clicks, replace=False)
    x[pos] = click * np.where(np.arange(n_clicks) % 2 == 0, 1.0, -1.0)
    return x


def am_noise(sr: float, seconds: float, seed: int, rate_hz: float = 3.0, depth: float = 0.8) -> np.ndarray:
    """Unit-RMS-ish Gaussian noise, amplitude-modulated by 1 + depth sin(2 pi rate t)."""
    rng = np.random.default_rng(seed)
    T = int(seconds * sr)
    t = np.arange(T) / sr
    return rng.standard_normal(T) * (1 + depth * np.sin(2 * np.pi * rate_hz * t)) / 3.0


def clipped_sine(T: int, f_rel: float = 0.21, phase: float = 0.3, amp: float = 1.5) -> np.ndarray:
    return np.clip(amp * np.sin(2 * np.pi * f_rel * np.arange(T) + phase), -1, 1)


def quarter_rate_sine(T: int, amp: float = 1.0) -> np.ndarray:
    """fs/4 at 45 degrees, unfaded: starts and ends at full level; sample peak amp / sqrt 2, true peak amp."""
    return amp * np.sin(2 * np.pi * 0.25 * np.arange(T) + np.pi / 4)
