"""Float64 oracle of the stateful and zero-phase cascades (``core.iir.sosfilt(..., zi)`` / ``sosfiltfilt``,
``AudioSignal.sos_filter(zero_phase=True)``; csrc/iir.cu, DESIGN.md K19), next to ``tests/iir64.py``.

* ``reference_filtfilt``: ``scipy.signal.sosfiltfilt`` in float64 on the float32 samples (times the gain, rounded to
  float32) and the float32 coefficients of ``iir64.coefficients``, per item; an unstable item is all NaN.
* ``baseline_filtfilt``: scipy's same steps in float32 -- the edge extension, ``sosfilt_zi`` cast to float32, two
  float32 ``sosfilt`` passes -- the sequential float32 error the kernels are compared with.
* ``reference_state`` / ``baseline_state``: ``scipy.signal.sosfilt(..., zi=zi)`` in float64 / float32 -> (y, zf).
* ``default_padlen``: scipy's rule, 3 (2S + 1 - min(#{b2 == 0}, #{a2 == 0})), per item.
"""
import numpy as np
from scipy import signal as sps

from tests import iir64


def default_padlen(sos32) -> np.ndarray:
    S = sos32.shape[-2]
    nb = (sos32[..., 2] == 0).sum(-1)
    na = (sos32[..., 5] == 0).sum(-1)
    return 3 * (2 * S + 1 - np.minimum(nb, na))


def _gained(x, gain):
    x = np.asarray(x, dtype=np.float32)
    if gain is not None:
        x = (x * np.asarray(gain, np.float32)[:, None, None]).astype(np.float32)
    return x


def _extend(x, padtype, n):
    """scipy's odd / even / constant extension of the last axis by n, in x's dtype."""
    if padtype is None or n == 0:
        return x
    left, right = x[..., 1:n + 1][..., ::-1], x[..., -n - 1:-1][..., ::-1]
    if padtype == "even":
        return np.concatenate([left, x, right], axis=-1)
    x0, x1 = x[..., :1], x[..., -1:]
    if padtype == "constant":
        return np.concatenate([np.repeat(x0, n, -1), x, np.repeat(x1, n, -1)], axis=-1)
    two = x.dtype.type(2)
    return np.concatenate([two * x0 - left, x, two * x1 - right], axis=-1)


def reference_filtfilt(x, sos32, gain=None, padtype="odd", padlen=None) -> np.ndarray:
    x = _gained(x, gain)
    ok = iir64.stable(sos32)
    out = np.empty(x.shape, dtype=np.float64)
    for b in range(x.shape[0]):
        if not ok[b]:
            out[b] = np.nan
            continue
        out[b] = sps.sosfiltfilt(sos32[b].astype(np.float64), x[b].astype(np.float64), axis=-1, padtype=padtype,
                                 padlen=padlen)
    return out


def baseline_filtfilt(x, sos32, gain=None, padtype="odd", padlen=None) -> np.ndarray:
    x = _gained(x, gain)
    ok = iir64.stable(sos32)
    out = np.empty(x.shape, dtype=np.float64)
    T = x.shape[-1]
    for b in range(x.shape[0]):
        if not ok[b]:
            out[b] = np.nan
            continue
        s = sos32[b].astype(np.float32)
        n = 0 if padtype is None else int(default_padlen(s) if padlen is None else padlen)
        ext = _extend(x[b], padtype, n)
        zi = sps.sosfilt_zi(s.astype(np.float64)).astype(np.float32)[:, None, :]  # [S, 1, 2] over the channels
        y = sps.sosfilt(s, ext, axis=-1, zi=zi * ext[None, :, :1])[0].astype(np.float32)
        y = sps.sosfilt(s, y[:, ::-1], axis=-1, zi=zi * y[None, :, -1:])[0][:, ::-1].astype(np.float32)
        out[b] = y[:, n:n + T]
    return out


def _state(x, sos32, zi, dtype, gain=None):
    x = _gained(x, gain)
    ok = iir64.stable(sos32)
    y = np.empty(x.shape, dtype=np.float64)
    zf = np.empty(np.shape(zi), dtype=np.float64)
    for b in range(x.shape[0]):
        if not ok[b]:
            y[b] = np.nan
            zf[:, b] = np.nan
            continue
        yb, zb = sps.sosfilt(sos32[b].astype(dtype), x[b].astype(dtype), axis=-1,
                             zi=np.asarray(zi)[:, b].astype(dtype))
        y[b], zf[:, b] = yb, zb
    return y, zf


def reference_state(x, sos32, zi, gain=None):
    return _state(x, sos32, zi, np.float64, gain)


def baseline_state(x, sos32, zi, gain=None):
    return _state(x, sos32, zi, np.float32, gain)
