"""Float64 oracle of the diffuse late tail of ``core.room.image_source_ir(..., diffuse_after=t_d, seed=s)``
(csrc/rir.cu, DESIGN.md K20 "Hybrid"), written from the definition, not from the kernel; the early part is
``tests/rir64.py``'s images with floor(d) < min(L, n_d), n_d = ceil(t_d fs).

* ``envelope``: the expected energy per sample of the image arrivals at sample n,
    E(n) = c / (4 pi V fs) (1/4pi) int exp(-n sum_a lambda_a |u_a|) dOmega(u),
    lambda_a = -(ln beta_a0 + ln beta_a1) / L_a  (L_a in samples),
  written with u_z uniform on [0, 1] (Archimedes) over one octant and evaluated by a tanh-sinh rule in z and in the
  azimuth, fine enough to be converged (``test_sim_rir_diffuse`` checks it against one twice as fine).  A wall with
  beta = 0 gives E = 0.
* ``xi_bits`` / ``xi``: the counter-based normal generator.  key = mix(mix(seed) + c), z = mix(key + n gamma) (mod
  2^64, gamma = 0x9E3779B97F4A7C15, mix the SplitMix64 finaliser); u1 = (z >> 32 + 1/2) 2^-32, u2 = (z mod 2^32)
  2^-32; xi = sqrt(-2 ln u1) cos(2 pi u2) (Box-Muller).
* ``ramp``: w(n) = sqrt(1/2 (1 - cos(pi x))), x = (n - n_d + Tw/2 + 1/2) / Tw over the Tw samples centred on n_d,
  then 1: w^2 at n_d - Tw/2 + k and at n_d + Tw/2 - 1 - k add to 1.
* ``tail``: w(n) sqrt(E(n)) xi(seed, c, n) for n >= n_d - Tw/2, else 0.
"""
import math

import numpy as np

from tests import rir64

GAMMA = 0x9E3779B97F4A7C15
_M64 = (1 << 64) - 1


def _mix(z: np.ndarray) -> np.ndarray:
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def xi_bits(seed: int, c: int, n) -> np.ndarray:
    """The 64-bit word of sample(s) n of microphone c under ``seed``."""
    with np.errstate(over="ignore"):
        key = _mix(_mix(np.uint64(seed)) + np.uint64(c))
        return _mix(key + np.asarray(n, dtype=np.uint64) * np.uint64(GAMMA))


def xi(seed: int, c: int, n):
    """(xi, radius sqrt(-2 ln u1)) of sample(s) n."""
    z = xi_bits(seed, c, n)
    u1 = ((z >> np.uint64(32)).astype(np.float64) + 0.5) * 2.0 ** -32
    u2 = (z & np.uint64(0xFFFFFFFF)).astype(np.float64) * 2.0 ** -32
    r = np.sqrt(-2.0 * np.log(u1))
    return r * np.cos(2.0 * math.pi * u2), r


def rates(room, beta, fs: float, c: float = 343.0):
    """lambda [3] per sample, or None when a wall has beta = 0."""
    beta = np.asarray(beta, np.float64)
    if np.any(beta == 0):
        return None
    L = np.asarray(room, np.float64) * fs / c
    return -(np.log(beta[0::2]) + np.log(beta[1::2])) / L


def _tanh_sinh(K: int, kmax: float = 3.2):
    """Nodes and weights of a (2K + 1)-point tanh-sinh rule on [0, 1]."""
    h = kmax / K
    t = np.arange(-K, K + 1) * h
    x = 0.5 * (1.0 + np.tanh(0.5 * math.pi * np.sinh(t)))
    w = 0.25 * math.pi * h * np.cosh(t) / np.cosh(0.5 * math.pi * np.sinh(t)) ** 2
    return x, w


def direction_mean(lam, n, K: int = 64) -> np.ndarray:
    """(1/4pi) int exp(-n sum_a lambda_a |u_a|) dOmega for samples n [N] (float64)."""
    x, w = _tanh_sinh(K)
    z, wz = x, w
    phi, wp = 0.5 * math.pi * x, 0.5 * math.pi * w
    rho = np.sqrt(1.0 - z * z)
    sig = (lam[2] * z[:, None] + rho[:, None] * (lam[0] * np.cos(phi)[None, :] + lam[1] * np.sin(phi)[None, :]))
    sig, wt = sig.reshape(-1), (wz[:, None] * wp[None, :]).reshape(-1) * (2.0 / math.pi)
    n = np.asarray(n, np.float64)
    out = np.empty(len(n))
    for s in range(0, len(n), 256):
        out[s:s + 256] = np.exp(-n[s:s + 256, None] * sig[None, :]) @ wt
    return out


def envelope(room, beta, fs: float, n, c: float = 343.0, K: int = 64) -> np.ndarray:
    """E(n) [N] for samples n of one item."""
    lam = rates(room, beta, fs, c)
    n = np.asarray(n, np.float64)
    if lam is None:
        return np.zeros(len(n))
    vol = float(np.prod(np.asarray(room, np.float64)))
    return c / (4.0 * math.pi * vol * fs) * direction_mean(lam, n, K)


def n_diffuse(t_d: float, fs: float) -> int:
    return int(math.ceil(t_d * fs))


def ramp(n, n_d: int, Tw: int) -> np.ndarray:
    n = np.asarray(n, np.float64)
    x = np.clip((n - n_d + Tw // 2 + 0.5) / Tw, 0.0, 1.0)
    return np.sqrt(0.5 * (1.0 - np.cos(math.pi * x)))


def tail(room, beta, fs: float, L: int, t_d: float, seed: int, mic: int, c: float = 343.0):
    """(tail [L], sqrt(E) * radius [L]) of microphone ``mic``: 0 before n_d - Tw/2."""
    Tw = rir64.window(fs)
    n_d = n_diffuse(t_d, fs)
    n = np.arange(max(0, n_d - Tw // 2), L)
    out, scale = np.zeros(L), np.zeros(L)
    if len(n):
        sq = np.sqrt(envelope(room, beta, fs, n, c))
        x, r = xi(seed, mic, n)
        out[n] = ramp(n, n_d, Tw) * sq * x
        scale[n] = sq * r
    return out, scale


def early(room, src, mic, beta, fs: float, L: int, t_d: float, c: float = 343.0):
    """(y64 [L], G [L]) of the images with floor(d) < min(L, n_d)."""
    d, g, _ = rir64.images(room, src, mic, beta, fs, min(L, n_diffuse(t_d, fs)), -1, c)
    Tw = rir64.window(fs)
    return rir64.render(d, g, Tw, L), rir64.bound(d, g, Tw, L)
