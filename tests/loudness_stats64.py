"""Float64 restatement of ``AudioSignal.loudness_stats`` (EBU R128 statistics, csrc/lufs.cu ``loudness_stats_kernel``)
for tests/test_gpu_loudness_stats.py and tests/test_sim_loudness_stats.py.

* ``momentary64`` / ``short_term64``: the K-weighted energy of the zero-padded row (scipy ``lfilter`` in float64,
  tests/timedomain64.py) over 400 ms blocks / 3 s blocks (30 gating strides), 100 ms apart, in LUFS.
* ``lra64``: the four loudness-range fields from a row of short-term values, in float64: absolute gate S > -70, the
  threshold 20 LU below the power mean of those, relative gate S > threshold among them, nearest-rank 10 % / 95 %
  percentiles v[floor(p (n - 1) + 0.5)] of the kept values (libebur128's ranks), LRA = High - Low in float32 (the
  kernel's output type).  No S above -70: LRA = 0, the rest -inf.
* ``ebu3342``: the stereo 1 kHz sine sequences of EBU Tech 3342 test cases 1-4 and their expected LRA."""
import math

import numpy as np

from tests import timedomain64 as td

DB_PER_REL = 10.0 / math.log(10.0)  # d(10 log10 E) / (dE / E)


def channel_gains(C):
    from audiotools_b200.core import kweighting

    return kweighting.CHANNEL_GAINS[:C].astype(np.float64)


def _filtered(x, rate, Tp):
    x = np.asarray(x, np.float64)
    xp = np.zeros(x.shape[:-1] + (Tp,))
    xp[..., :x.shape[-1]] = x
    return td.kweight64(xp, td.kweight_coef(rate))


def stride_energies64(x, rate, Tp=None):
    """[..., C, n_strides] float64: sum of y^2 over each whole gating stride [j s, (j + 1) s) of the K-weighted row."""
    Tp = x.shape[-1] if Tp is None else Tp
    s = td.kweight_geometry(Tp, rate)[1]
    y = _filtered(x, rate, Tp)
    n = Tp // s
    return (y[..., :n * s] ** 2).reshape(y.shape[:-1] + (n, s)).sum(-1)


def num_short_term(Tp, rate):
    s = td.kweight_geometry(Tp, rate)[1]
    return (Tp - 30 * s) // s + 1 if Tp >= 30 * s else 0


def short_term64(x, rate, Tp=None):
    """[B, n_st] float64 short-term loudness of x [B, C, T]."""
    Tp = x.shape[-1] if Tp is None else Tp
    s = td.kweight_geometry(Tp, rate)[1]
    n_st = num_short_term(Tp, rate)
    e = stride_energies64(x, rate, Tp)  # [B, C, n]
    c = np.concatenate([np.zeros(e.shape[:-1] + (1,)), np.cumsum(e, -1)], -1)
    E = c[..., 30:30 + n_st] - c[..., :n_st]  # [B, C, n_st]
    G = channel_gains(x.shape[1])
    with np.errstate(divide="ignore"):
        return -0.691 + 10 * np.log10((G[None, :, None] * E).sum(1) / (30 * s))


def momentary64(x, rate, Tp=None):
    """[B, nblk] float64 loudness of every 400 ms gating block of x [B, C, T]."""
    z = td.kweight_blocks64(x, rate, Tp)
    G = channel_gains(x.shape[1])
    with np.errstate(divide="ignore"):
        return -0.691 + 10 * np.log10((G[None, :, None] * z).sum(1))


def lra64(S):
    """{"LRA", "LRA Threshold", "LRA Low", "LRA High"} of one row of float32 short-term values, with the kept count n."""
    S = np.asarray(S, np.float32).astype(np.float64)
    a = S[S > -70]
    if a.size == 0:
        return {"LRA": 0.0, "LRA Threshold": -math.inf, "LRA Low": -math.inf, "LRA High": -math.inf, "n": 0}
    thr = -0.691 + 10 * math.log10(np.mean(10.0 ** ((a + 0.691) / 10))) - 20
    v = np.sort(a[a > thr])
    n = v.size
    lo, hi = np.float32(v[math.floor(0.10 * (n - 1) + 0.5)]), np.float32(v[math.floor(0.95 * (n - 1) + 0.5)])
    return {"LRA": float(np.float32(hi - lo)), "LRA Threshold": thr, "LRA Low": float(lo), "LRA High": float(hi),
            "n": n}


def ulp32(v):
    return np.spacing(np.abs(np.asarray(v, np.float32))).astype(np.float64)


# EBU Tech 3342 (2016) cases 1-4: stereo 1 kHz sine, levels in dBFS per segment, expected LRA in LU
EBU3342 = {1: ([-20, -30], 10.0), 2: ([-20, -15], 5.0), 3: ([-40, -20], 20.0), 4: ([-50, -35, -20, -35, -50], 15.0)}


def ebu3342(case, rate, seg_s=20.0):
    """[1, 2, T] float32: the case's segments of seg_s seconds each, a 1 kHz sine of peak 10^(dBFS / 20) on both
    channels, and the expected LRA."""
    levels, want = EBU3342[case]
    n = int(round(seg_s * rate))
    t = np.arange(n * len(levels)) / rate
    amp = np.repeat([10.0 ** (l / 20.0) for l in levels], n)
    x = (amp * np.sin(2 * np.pi * 1000.0 * t)).astype(np.float32)
    return np.stack([x, x])[None], want
