"""Float64 oracle of ``core.room.image_source_ir`` (csrc/rir.cu, DESIGN.md K20), written from the definition of the
image-source method, not from the kernel.

* ``images``: every image of one (room, source, microphone) with floor(d) < L (and order <= max_order when >= 0):
  its distance d in samples, its gain g and its order, enumerated over |m| <= ceil(L / (2 L_axis)) + 1 per axis.
* ``render``: y[i] = sum over images of g h_n at i = floor(d) - Tw/2 + 1 + n, n = 0 .. Tw - 1, with
  h_n = 1/2 (1 - cos(2 pi (n + 1 - f) / Tw)) sinc(pi (n + 1 - f - Tw/2)), f = d - floor(d); taps outside [0, L) dropped.
* ``bound``: G[i] = sum |g| min(1, 1 / (pi |i - d|)) over the images reaching sample i, and ``reached``: whether any
  does.  A float32 evaluation of the taps is held to |y - y64| <= K u G.
* ``sabine_beta`` and ``highpass_sos``: Sabine's wall coefficient and Allen & Berkley's 100 Hz high-pass section.
"""
import math

import numpy as np

U = 2.0 ** -24


def window(fs: float) -> int:
    """Tw = 2 round(0.004 fs), halves rounded up."""
    return 2 * int(math.floor(0.004 * fs + 0.5))


def sabine_beta(room, rt60, c: float = 343.0) -> float:
    lx, ly, lz = (float(v) for v in room)
    if rt60 == 0:
        return 0.0
    alpha = 24.0 * math.log(10.0) * lx * ly * lz / (c * 2.0 * (lx * ly + lx * lz + ly * lz) * rt60)
    assert alpha <= 1.0
    return math.sqrt(1.0 - alpha)


def highpass_sos(fs: float) -> np.ndarray:
    w = 2.0 * math.pi * 100.0 / fs
    r = math.exp(-w)
    return np.array([[1.0, -(1.0 + r), r, 1.0, -2.0 * r * math.cos(w), r * r]])


def images(room, src, mic, beta, fs: float, L: int, max_order: int = -1, c: float = 343.0):
    """(d [n], g [n], order [n]) of the images used for an IR of L samples."""
    ks = fs / c
    room = np.asarray(room, np.float64) * ks
    src = np.asarray(src, np.float64) * ks
    mic = np.asarray(mic, np.float64) * ks
    beta = np.asarray(beta, np.float64)
    axes = []
    for a in range(3):
        M = int(math.ceil(L / (2.0 * room[a]))) + 1
        m = np.arange(-M, M + 1, dtype=np.float64)
        off, order, gain = [], [], []
        for p in (0, 1):
            off.append((1 - 2 * p) * src[a] - mic[a] + 2.0 * m * room[a])
            order.append(np.abs(2 * m - p))
            gain.append(beta[2 * a] ** np.abs(m - p) * beta[2 * a + 1] ** np.abs(m))
        axes.append((np.concatenate(off), np.concatenate(order), np.concatenate(gain)))
    (X, ox, gx), (Y, oy, gy), (Z, oz, gz) = axes
    ds, gs, os_ = [], [], []
    for i in range(len(X)):  # chunked over the x images
        d = np.sqrt(X[i] ** 2 + Y[:, None] ** 2 + Z[None, :] ** 2)
        o = ox[i] + oy[:, None] + oz[None, :]
        keep = np.floor(d) < L
        if max_order >= 0:
            keep &= o <= max_order
        if not keep.any():
            continue
        g = gx[i] * gy[:, None] * gz[None, :] / (4.0 * math.pi * d / ks)
        ds.append(d[keep])
        gs.append(g[keep])
        os_.append(o[keep])
    if not ds:
        return np.zeros(0), np.zeros(0), np.zeros(0)
    return np.concatenate(ds), np.concatenate(gs), np.concatenate(os_)


def _scatter(d, vals_fn, Tw: int, L: int, chunk_taps: int = 1 << 23) -> np.ndarray:
    out = np.zeros(L)
    n = np.arange(Tw, dtype=np.float64)
    step = max(1, chunk_taps // Tw)
    for s in range(0, len(d), step):
        dd = d[s:s + step]
        fl = np.floor(dd)
        idx = (fl[:, None] - Tw // 2 + 1 + n).astype(np.int64)
        v = vals_fn(s, s + step, dd, fl, n)
        ok = (idx >= 0) & (idx < L)
        out += np.bincount(idx[ok], weights=v[ok], minlength=L)
    return out


def render(d, g, Tw: int, L: int) -> np.ndarray:
    """The IR of the images (d, g) before the high-pass, float64 [L]."""
    def taps(a, b, dd, fl, n):
        f = (dd - fl)[:, None]
        h = 0.5 * (1.0 - np.cos(2.0 * math.pi * (n + 1 - f) / Tw)) * np.sinc(n + 1 - f - Tw / 2)
        return g[a:b, None] * h
    return _scatter(d, taps, Tw, L)


def bound(d, g, Tw: int, L: int) -> np.ndarray:
    """G[i] = sum |g| min(1, 1 / (pi |i - d|)) over the images whose window holds sample i."""
    def terms(a, b, dd, fl, n):
        t = np.abs(fl[:, None] - Tw // 2 + 1 + n - dd[:, None])
        return np.abs(g[a:b, None]) * np.minimum(1.0, 1.0 / (math.pi * np.maximum(t, 1e-300)))
    return _scatter(d, terms, Tw, L)


def reached(d, Tw: int, L: int) -> np.ndarray:
    """[L] bool: some image's window holds the sample."""
    return _scatter(d, lambda a, b, dd, fl, n: np.ones((len(dd), Tw)), Tw, L) > 0


def ir(room, src, mic, beta, fs, L, max_order=-1, c=343.0):
    """(y64 [L], G [L], reached [L], n_images) for one microphone."""
    d, g, _ = images(room, src, mic, beta, fs, L, max_order, c)
    Tw = window(fs)
    return render(d, g, Tw, L), bound(d, g, Tw, L), reached(d, Tw, L), len(d)
