"""Float64 oracle of ``AudioSignal.sos_filter`` / ``parametric_eq`` (csrc/iir.cu, DESIGN.md K19).

* ``coefficients``: the kernel's inputs, every section divided by its a0 in float64 and rounded to float32 once.
* ``reference``: ``scipy.signal.sosfilt`` in float64 on the float32 input (times the gain, rounded to float32) with
  those coefficients, per item; an item with a section outside the triangle |a2| < 1, |a1| < 1 + a2 is all NaN.
* ``baseline``: the same call in float32 -- the sequential float32 cascade the kernel's error is compared with.
* ``block_error``: per row, the worst 1024-sample block's max |error| over the block's float64 RMS (floored at 1e-3
  of the row's loudest block), in units of u = 2^-24.
* ``cookbook``: a numpy restatement of the RBJ Audio EQ Cookbook, written from the cookbook's own formulas, not from
  ``core/biquad.py``; ``response`` evaluates |H(e^{jw})| of a cascade.
"""
import numpy as np
from scipy import signal as sps

U = 2.0 ** -24
BLOCK = 1024


def coefficients(sos, B: int) -> np.ndarray:
    """[S, 6] or [1 or B, S, 6] -> [B, S, 6] float32, normalised by a0 in float64."""
    s = np.asarray(sos, dtype=np.float64)
    if s.ndim == 2:
        s = s[None]
    s = (s / s[..., 3:4]).astype(np.float32)
    return np.broadcast_to(s, (B,) + s.shape[1:])


def stable(sos32) -> np.ndarray:
    """[B] bool: every section passes the triangle test in float32."""
    a1, a2 = sos32[..., 4], sos32[..., 5]
    return ((np.abs(a2) < 1) & (np.abs(a1) < 1 + a2)).all(axis=-1)


def _run(x, sos32, dtype, gain=None, reverse=False):
    x = np.asarray(x, dtype=np.float32)
    if gain is not None:
        x = (x * np.asarray(gain, np.float32)[:, None, None]).astype(np.float32)
    if reverse:
        x = x[..., ::-1]
    out = np.empty(x.shape, dtype=np.float64)
    ok = stable(sos32)
    for b in range(x.shape[0]):
        if not ok[b]:
            out[b] = np.nan
            continue
        out[b] = sps.sosfilt(sos32[b].astype(dtype), x[b].astype(dtype), axis=-1)
    return out[..., ::-1] if reverse else out


def reference(x, sos32, gain=None, reverse=False) -> np.ndarray:
    return _run(x, sos32, np.float64, gain, reverse)


def baseline(x, sos32, gain=None, reverse=False) -> np.ndarray:
    return _run(x, sos32, np.float32, gain, reverse)


def block_error(got, ref, block: int = BLOCK) -> np.ndarray:
    """[rows] worst-block error in u (see the module docstring); rows of [..., T] flattened."""
    got = np.asarray(got, np.float64).reshape(-1, np.shape(got)[-1])
    ref = np.asarray(ref, np.float64).reshape(-1, np.shape(ref)[-1])
    T = ref.shape[-1]
    nb = (T + block - 1) // block
    pad = nb * block - T
    e = np.pad(np.abs(got - ref), ((0, 0), (0, pad))).reshape(len(ref), nb, block).max(axis=-1)
    sq = np.pad(ref * ref, ((0, 0), (0, pad))).reshape(len(ref), nb, block).sum(axis=-1)
    n = np.full(nb, block, dtype=np.float64)
    n[-1] = block - pad
    rms = np.sqrt(sq / n)
    floor = 1e-3 * rms.max(axis=1, keepdims=True)
    denom = np.maximum(rms, floor)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(e == 0, 0.0, e / np.where(denom > 0, denom, np.inf))
    r = np.where((denom == 0) & (e > 0), np.inf, r)
    return r.max(axis=1) / U


# --------------------------------------------------------------------------- the cookbook
def cookbook(kind: str, freq: float, gain_db: float, q: float, sr: float) -> np.ndarray:
    """One section [6] (b0 b1 b2 a0 a1 a2), float64, from the RBJ Audio EQ Cookbook."""
    A = 10.0 ** (gain_db / 40.0)
    w0 = 2.0 * np.pi * freq / sr
    cs, sn = np.cos(w0), np.sin(w0)
    alpha = sn / (2.0 * q)
    if kind == "peaking":
        return np.array([1 + alpha * A, -2 * cs, 1 - alpha * A, 1 + alpha / A, -2 * cs, 1 - alpha / A])
    if kind == "low_shelf":
        t = 2 * np.sqrt(A) * alpha
        return np.array([A * ((A + 1) - (A - 1) * cs + t), 2 * A * ((A - 1) - (A + 1) * cs),
                         A * ((A + 1) - (A - 1) * cs - t), (A + 1) + (A - 1) * cs + t,
                         -2 * ((A - 1) + (A + 1) * cs), (A + 1) + (A - 1) * cs - t])
    if kind == "high_shelf":
        t = 2 * np.sqrt(A) * alpha
        return np.array([A * ((A + 1) + (A - 1) * cs + t), -2 * A * ((A - 1) + (A + 1) * cs),
                         A * ((A + 1) + (A - 1) * cs - t), (A + 1) - (A - 1) * cs + t,
                         2 * ((A - 1) - (A + 1) * cs), (A + 1) - (A - 1) * cs - t])
    a = [1 + alpha, -2 * cs, 1 - alpha]
    b = {"low_pass": [(1 - cs) / 2, 1 - cs, (1 - cs) / 2],
         "high_pass": [(1 + cs) / 2, -(1 + cs), (1 + cs) / 2],
         "band_pass": [alpha, 0.0, -alpha],
         "notch": [1.0, -2 * cs, 1.0],
         "all_pass": [1 - alpha, -2 * cs, 1 + alpha]}[kind]
    return np.array(b + a)


def response(sos, f, sr: float) -> np.ndarray:
    """|H| of the cascade ``sos`` [S, 6] at the frequencies ``f`` (Hz)."""
    z = np.exp(-1j * 2 * np.pi * np.asarray(f, np.float64) / sr)
    h = np.ones_like(z)
    for b0, b1, b2, a0, a1, a2 in np.asarray(sos, np.float64):
        h *= (b0 + b1 * z + b2 * z * z) / (a0 + a1 * z + a2 * z * z)
    return np.abs(h)
