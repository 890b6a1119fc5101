"""Float64 oracle of the directivity of ``core.room.image_source_ir(..., mic_pattern=, mic_orientation=,
source_pattern=, source_orientation=)`` (csrc/rir.cu, DESIGN.md K20 "Directivity"), written from the definition, not
from the kernel.

* ``images``: every image with floor(d) < L (order <= max_order when >= 0) with its offset (X, Y, Z) = image -
  microphone, its parities (q, j, k) and its gain g; ``gains`` scales g by D_m(u_m) D_s(w), D(u) = p + (1 - p) u.v,
  u_m = (X, Y, Z) / d, w = -((1 - 2q) X, (1 - 2j) Y, (1 - 2k) Z) / d.  ``tests/rir64.py`` renders them and bounds them.
* ``envelope``: the tail's expected energy per sample with directivity,
    E(n) = c / (4 pi V fs) (1/4pi) int D_m(u)^2 <D_s(-s u)^2>_s exp(-n sum_a lambda_a |u_a|) dOmega(u),
  <.>_s the mean over the eight sign vectors s (the parity classes), by its own tanh-sinh rule over each of the eight
  octants of the full sphere: nothing of the kernel's reduction to one octant is assumed.
* ``band``: one band of one microphone (images, air, tail), as ``tests/rir_bands64.py``'s ``band``.
"""
import math

import numpy as np

from tests import rir64
from tests import rir_diffuse64 as D

OMNI = (1.0, np.zeros(3))


def gain(p: float, v, u) -> np.ndarray:
    """D(u) = p + (1 - p) u.v for unit directions u [..., 3]."""
    return p + (1.0 - p) * (np.asarray(u) @ np.asarray(v, np.float64))


def images(room, src, mic, beta, fs: float, L: int, max_order: int = -1, c: float = 343.0):
    """(d [n], g [n], off [n, 3] in samples, parity [n, 3]) of the images used for an IR of L samples."""
    ks = fs / c
    room = np.asarray(room, np.float64) * ks
    src = np.asarray(src, np.float64) * ks
    mic = np.asarray(mic, np.float64) * ks
    beta = np.asarray(beta, np.float64)
    axes = []
    for a in range(3):
        M = int(math.ceil(L / (2.0 * room[a]))) + 1
        m = np.arange(-M, M + 1, dtype=np.float64)
        off, order, g, par = [], [], [], []
        for p in (0, 1):
            off.append((1 - 2 * p) * src[a] - mic[a] + 2.0 * m * room[a])
            order.append(np.abs(2 * m - p))
            g.append(beta[2 * a] ** np.abs(m - p) * beta[2 * a + 1] ** np.abs(m))
            par.append(np.full(len(m), p))
        axes.append(tuple(np.concatenate(v) for v in (off, order, g, par)))
    (X, ox, gx, px), (Y, oy, gy, py), (Z, oz, gz, pz) = axes
    out = []
    for i in range(len(X)):
        d = np.sqrt(X[i] ** 2 + Y[:, None] ** 2 + Z[None, :] ** 2)
        keep = np.floor(d) < L
        if max_order >= 0:
            keep &= ox[i] + oy[:, None] + oz[None, :] <= max_order
        if not keep.any():
            continue
        iy, iz = np.nonzero(keep)
        dd = d[keep]
        g = gx[i] * gy[iy] * gz[iz] / (4.0 * math.pi * dd / ks)
        off = np.stack([np.full(len(iy), X[i]), Y[iy], Z[iz]], axis=1)
        par = np.stack([np.full(len(iy), px[i]), py[iy], pz[iz]], axis=1)
        out.append((dd, g, off, par))
    if not out:
        return np.zeros(0), np.zeros(0), np.zeros((0, 3)), np.zeros((0, 3))
    return tuple(np.concatenate(v) for v in zip(*out))


def gains(d, g, off, par, mic_pv=OMNI, src_pv=OMNI) -> np.ndarray:
    """g D_m(u_m) D_s(w) per image."""
    u = off / d[:, None]
    w = -(1.0 - 2.0 * par) * u
    return g * gain(*mic_pv, u) * gain(*src_pv, w)


def ir(room, src, mic, beta, fs, L, mic_pv=OMNI, src_pv=OMNI, max_order=-1, c=343.0):
    """(y64 [L], G [L]) of one microphone: G the per-sample bound of rir64.bound with |g D_m D_s|."""
    d, g, off, par = images(room, src, mic, beta, fs, L, max_order, c)
    gd = gains(d, g, off, par, mic_pv, src_pv)
    Tw = rir64.window(fs)
    return rir64.render(d, gd, Tw, L), rir64.bound(d, gd, Tw, L)


_SIGNS = np.array([[sx, sy, sz] for sx in (1, -1) for sy in (1, -1) for sz in (1, -1)], np.float64)


def direction_mean(lam, n, mic_pv=OMNI, src_pv=OMNI, K: int = 48) -> np.ndarray:
    """(1/4pi) int D_m(u)^2 <D_s(-s u)^2>_s exp(-n sum lambda_a |u_a|) dOmega over the full sphere, per octant a
    tanh-sinh rule in u_z (uniform: Archimedes) and in the azimuth."""
    x, w = D._tanh_sinh(K)
    pts, wts = [], []
    for zs in (1.0, -1.0):
        for quad in range(4):
            z = zs * x
            phi = 0.5 * math.pi * (quad + x)
            rho = np.sqrt(np.maximum(0.0, 1.0 - z * z))
            u = np.stack([rho[:, None] * np.cos(phi)[None, :], rho[:, None] * np.sin(phi)[None, :],
                          np.broadcast_to(z[:, None], (len(x), len(x)))], axis=-1).reshape(-1, 3)
            pts.append(u)
            # dOmega = dz dphi: per octant the z- and phi-rules' weights, times (1/4pi)
            wts.append((w[:, None] * (0.5 * math.pi * w)[None, :]).reshape(-1) / (4.0 * math.pi))
    u, wt = np.concatenate(pts), np.concatenate(wts)
    dm2 = gain(*mic_pv, u) ** 2
    ds2 = np.mean([gain(*src_pv, -s * u) ** 2 for s in _SIGNS], axis=0)
    sig = np.abs(u) @ np.asarray(lam, np.float64)
    wt = wt * dm2 * ds2
    n = np.asarray(n, np.float64)
    out = np.empty(len(n))
    for s in range(0, len(n), 256):
        out[s:s + 256] = np.exp(-n[s:s + 256, None] * sig[None, :]) @ wt
    return out


def envelope(room, beta, fs: float, n, mic_pv=OMNI, src_pv=OMNI, c: float = 343.0, K: int = 48) -> np.ndarray:
    lam = D.rates(room, beta, fs, c)
    n = np.asarray(n, np.float64)
    if lam is None:
        return np.zeros(len(n))
    vol = float(np.prod(np.asarray(room, np.float64)))
    return c / (4.0 * math.pi * vol * fs) * direction_mean(lam, n, mic_pv, src_pv, K)


def tail(room, beta, fs: float, L: int, t_d: float, seed: int, mic: int, mic_pv=OMNI, src_pv=OMNI,
         c: float = 343.0):
    """(tail [L], sqrt(E) * radius [L]) of microphone ``mic`` with the weighted envelope."""
    Tw = rir64.window(fs)
    n_d = D.n_diffuse(t_d, fs)
    n = np.arange(max(0, n_d - Tw // 2), L)
    out, scale = np.zeros(L), np.zeros(L)
    if len(n):
        sq = np.sqrt(envelope(room, beta, fs, n, mic_pv, src_pv, c))
        x, r = D.xi(seed, mic, n)
        out[n] = D.ramp(n, n_d, Tw) * sq * x
        scale[n] = sq * r
    return out, scale


def band(room, src, mic, beta_k, air_k: float, fs: float, L: int, mic_pv=OMNI, src_pv=OMNI, max_order: int = -1,
         td=None, seed=None, ch: int = 0, c: float = 343.0):
    """(r [L], G [L], tail [L], tail scale [L]) of one band: directional images times 10^(-air_k d_m / 20), and with
    ``td`` the tail under the weighted envelope times 10^(-air_k (c n / fs) / 20)."""
    Tw = rir64.window(fs)
    lim = L if td is None else min(L, D.n_diffuse(td, fs))
    d, g, off, par = images(room, src, mic, beta_k, fs, lim, max_order, c)
    gd = gains(d, g, off, par, mic_pv, src_pv) * 10.0 ** (-air_k * (d * c / fs) / 20.0)
    r, G = rir64.render(d, gd, Tw, L), rir64.bound(d, gd, Tw, L)
    t, sc = np.zeros(L), np.zeros(L)
    if td is not None:
        t, sc = tail(room, beta_k, fs, L, td, seed, ch, mic_pv, src_pv, c)
        att = 10.0 ** (-air_k * (np.arange(L) * c / fs) / 20.0)
        t, sc = t * att, sc * att
    return r + t, G, t, sc
