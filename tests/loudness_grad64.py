"""Float64 oracle of ``metrics.LoudnessLoss``'s gradient (``b2a_lufs_backward_f32``, csrc/lufs.cu + csrc/iir.cu, DESIGN.md
K21) for tests/test_gpu_loudness_grad.py and tests/test_sim_loudness_grad.py.

* ``forward64``: loud = max(lufs, -70) in float64 from the K-weighting with the kernels' float32-rounded coefficients
  (tests/timedomain64.py ``kweight_coef``), the 400 ms blocks of the row zero-extended to Tp, both gates.  Also the
  blocks' loudness, the gates and the kept set J.
* ``grad64``: d loud / d x by the float64 adjoint, K^T u over [0, Tp) cropped to [0, T), with
  u_c[t] = (10 / ln 10) G_c / (E n) * 2 y_c[t] * m[t] / (0.4 rate) and m[t] the blocks of J that contain t.
* ``baseline32``: the same formula with the J of float64 and everything else a sequential float32 cascade -- the error
  the kernel's is compared with.
* ``interval_error``: per row, the worst 100 ms interval's max |error| over the interval's float64 RMS (floored at
  1e-3 of the row's loudest interval), in units of u = 2^-24; intervals masked out are skipped.
"""
import math

import numpy as np
from scipy import signal as sps

from tests import timedomain64 as td

U = 2.0 ** -24
DB_PER_REL = 10.0 / math.log(10.0)
GATE_A = -70.0


def _sos(rate, dtype):
    b0, b1, b2, a1, a2 = td.kweight_coef(rate)
    return np.stack([b0, b1, b2, np.ones_like(b0), a1, a2], axis=1).astype(dtype)


def _zext(x, Tp):
    x = np.asarray(x, np.float64)
    xp = np.zeros(x.shape[:-1] + (Tp,))
    xp[..., :x.shape[-1]] = x
    return xp


def padded_length(T, rate):
    """``AudioSignal._padded_length``: rows under 0.5 s are zero-extended to 0.5 s."""
    dur = T / rate
    return T + int((0.5 - dur) * rate) if dur < 0.5 else T


def forward64(x, rate, Tp=None):
    """x [B, C, T] -> dict: loud, lufs [B]; l [B, nblk] block loudness; gamma_r [B]; keep [B, nblk] (J); y [B, C, Tp]
    the K-weighted zero-extended rows; z [B, C, nblk]; E, n [B]."""
    x = np.asarray(x, np.float64)
    B, C, T = x.shape
    Tp = T if Tp is None else Tp
    y = sps.sosfilt(_sos(rate, np.float64), _zext(x, Tp), axis=-1)
    z = td.kweight_blocks64(x, rate, Tp, filtered=y)
    G = _gains(C)
    with np.errstate(divide="ignore", invalid="ignore"):
        l = -0.691 + 10 * np.log10(np.einsum("c,bcj->bj", G, z))
        a = l > GATE_A
        na = a.sum(-1)
        za = (z * a[:, None]).sum(-1) / na[:, None]
        gamma_r = -0.691 + 10 * np.log10(np.einsum("c,bc->b", G, za)) - 10
        keep = a & (l > gamma_r[:, None])
        n = keep.sum(-1)
        zj = (z * keep[:, None]).sum(-1) / n[:, None]
        E = np.einsum("c,bc->b", G, np.nan_to_num(zj, nan=0.0))
        lufs = -0.691 + 10 * np.log10(E)
    return dict(loud=np.maximum(lufs, -70.0), lufs=lufs, l=l, gamma_r=gamma_r, keep=keep, y=y, z=z, E=E, n=n, Tp=Tp)


def _gains(C):
    from audiotools_b200.core import kweighting

    return kweighting.CHANNEL_GAINS[:C].astype(np.float64)


def block_counts(keep, T, rate, Tp):
    """m [B, Tp]: the blocks of J that contain each sample of the zero-extended row."""
    K, stride, nblk = td.kweight_geometry(Tp, rate)
    B = keep.shape[0]
    d = np.zeros((B, max(Tp, (nblk - 1) * stride + K) + 1))
    for i in range(nblk):
        d[:, i * stride] += keep[:, i]
        d[:, i * stride + K] -= keep[:, i]
    return np.cumsum(d, -1)[:, :Tp]


def _adjoint(x, rate, fw, dtype, grad_loud=None):
    B, C, T = np.shape(x)
    Tp = fw["Tp"]
    G = _gains(C)
    m = block_counts(fw["keep"], T, rate, Tp)
    gl = np.ones(B) if grad_loud is None else np.asarray(grad_loud, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        w = gl * DB_PER_REL * 2.0 / (0.4 * rate) / (fw["E"] * fw["n"])
    w = np.where(fw["lufs"] > -70, w, 0.0)
    sos = _sos(rate, dtype)
    if dtype == np.float64:
        y = fw["y"]
    else:
        y = sps.sosfilt(sos, _zext(x, Tp).astype(dtype), axis=-1)
    u = (w[:, None, None] * G[None, :, None] * m[:, None, :]).astype(dtype) * y.astype(dtype)
    g = sps.sosfilt(sos, u[..., ::-1].astype(dtype), axis=-1)[..., ::-1]
    return np.asarray(g[..., :T], np.float64)


def grad64(x, rate, Tp=None, grad_loud=None, fw=None):
    fw = forward64(x, rate, Tp) if fw is None else fw
    return _adjoint(x, rate, fw, np.float64, grad_loud)


def baseline32(x, rate, Tp=None, grad_loud=None, fw=None):
    fw = forward64(x, rate, Tp) if fw is None else fw
    return _adjoint(np.asarray(x, np.float32), rate, fw, np.float32, grad_loud)


def gate_margin(fw):
    """[B, nblk]: each block's distance in LU from the nearer gate (inf for an item with no gradient)."""
    d = np.minimum(np.abs(fw["l"] - GATE_A), np.abs(fw["l"] - fw["gamma_r"][:, None]))
    return np.where((fw["lufs"] > -70)[:, None], d, np.inf)


def near_gate_mask(fw, T, rate, margin=1e-3):
    """[B, T] bool: samples of a block within ``margin`` LU of a gate (skipped by per-interval comparisons)."""
    K, stride, nblk = td.kweight_geometry(fw["Tp"], rate)
    near = gate_margin(fw) < margin
    mask = np.zeros((near.shape[0], fw["Tp"]), bool)
    for b, i in zip(*np.nonzero(near)):
        mask[b, i * stride:i * stride + K] = True
    return mask[:, :T]


def interval_error(got, ref, rate, skip=None):
    """[rows] worst 100 ms interval error in u (module docstring); rows of [B, C, T]; skip [B, T] masks samples."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    B, C, T = ref.shape
    s = td.kweight_geometry(T, rate)[1]
    nb = (T + s - 1) // s
    pad = nb * s - T
    e = np.abs(got - ref)
    if skip is not None:
        e = np.where(skip[:, None, :], 0.0, e)
    e = np.pad(e, ((0, 0), (0, 0), (0, pad))).reshape(B, C, nb, s).max(-1)
    sq = np.pad(ref * ref, ((0, 0), (0, 0), (0, pad))).reshape(B, C, nb, s).sum(-1)
    cnt = np.full(nb, float(s))
    cnt[-1] = s - pad
    rms = np.sqrt(sq / cnt)
    den = np.maximum(rms, 1e-3 * rms.max(-1, keepdims=True))
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(e == 0, 0.0, e / np.where(den > 0, den, np.inf))
    return r.reshape(B * C, nb).max(-1) / U


def loud_of(x, rate, Tp=None):
    return forward64(x, rate, Tp)["loud"]
