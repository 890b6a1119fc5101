"""Float64 references and the per-cell error model of the spectral-mask accuracy tests (tests/test_gpu_specmask_accuracy.py
on the H100, tests/test_sim_specmask_accuracy.py on the simulator) for csrc/specmask.cu.

Every reference is written from the reference's definitions (ref:audiotools/core/dsp.py:217-370,
ref:audiotools/core/audio_signal.py log_magnitude, ref:audiotools/ml/layers/spectral_gate.py), never from the kernels,
and takes the kernels' exact float32 / complex64 inputs:

* band masks: the decision ``lo <= v < hi`` in float32 on the reference's ``torch.linspace`` grid, the fill
  ``val * exp(1j * val)`` in complex64; the backward ``band || X == 0 ? 0 : g``.  Exact: checked bit for bit.
* ``rotate``: ``X exp(1j s)`` in float64.  Per cell |out - ref| <= C_ROT u |X|.
* ``mask_low``: power |X|^2 in float64, the floor ``10 log10(max(max p, amin^2)) - top_db`` with NaN propagating as in
  ``torch.max``, a cell masked when ``max(db, floor) < cut``.  A cell within ``db_margin`` of its cut-off is undecided:
  the float32 evaluation may put it on either side.  Masked cells are ``val X / |X|`` within C_KEEP u |val|; their
  gradient ``val (g - Re(g conj w) w) / |X|`` (w = X / |X|) within C_MLBWD u |val| |g| / |X|.
* gate: thresholds ``mean + n_std std`` (unbiased) of ``20 log10(max(|X|, 1e-4))`` over the noise's frames, within
  C_TH u ``thresh_scale``; the smoothed mask is conv2d (a cross-correlation, zero padding) of the booleans against the
  KERNEL's own thresholds, evaluated twice: undecided cells counted 0 (S_lo) and 1 (S_hi).  The weights are
  non-negative, so [S_lo, S_hi] holds the exact result; the kernel's S may leave it by C_S u ``s_scale``.

u = 2^-24.  The constants C are set from the H100 measurement in DESIGN.md ("Spectral mask accuracy", printed by
tests/probes/specmask_accuracy_probe.py) with about 2x headroom over the worst case measured there and on the
simulator.  ``db_margin`` is not measured: it is the error bound of a float32 evaluation of the dB value."""
import math

import numpy as np
import torch
import torch.nn.functional as Fn

U = 2.0 ** -24

C_ROT = 6.0      # |rotate - X exp(1j s)| / (u |X|)
C_KEEP = 10.0    # |masked cell - val X / |X|| / (u |val|)
C_MLBWD = 2.0    # |masked gradient - float64| / (u |val| |g| / |X|)
C_TH = 0.15      # |thresh - float64| / (u thresh_scale)
C_S = 0.5        # distance of S from [S_lo, S_hi] / (u s_scale)
C_OUT = 0.6      # |out - mul (1 - amount S)| beyond the bracket / (u |mul| out_scale)


def db_margin(db):
    """Bound on |float32 dB - float64 dB| for ``10 log10(max(|X|^2, amin^2))`` and ``20 log10(max(|X|, 1e-4))``:
    hypotf's 3 ulp (6 u relative) doubled by the square, plus the rounding of the square, give 13 u of the power,
    4.343 x 13 u < 60 u in dB; log10f's 2 ulp and the multiply by 10 or 20 add at most 6 u |db|."""
    return U * (60.0 + 6.0 * np.abs(db))


# --------------------------------------------------------------------------- band masks
def band_fill(val):
    v = torch.tensor(float(val), dtype=torch.float32)
    return v * torch.exp(1j * v)  # complex64, the reference's arithmetic for a filled cell


def band(axis_vals, lo, hi, F, N, C, axis):
    """[B * C, F, N] bool: lo[item] <= v < hi[item] in float32, v the grid value of the cell's bin (axis 0) or frame."""
    v = axis_vals.float().cpu()
    lo = lo.float().cpu().repeat_interleave(C)[:, None, None]
    hi = hi.float().cpu().repeat_interleave(C)[:, None, None]
    v = v[None, :, None] if axis == 0 else v[None, None, :]
    return ((lo <= v) & (v < hi)).expand(-1, F, N)


def band_forward(X, m, val):
    return torch.where(m.reshape(X.shape), band_fill(val).to(torch.complex64), X)


def band_backward(g, X, m):
    zero = (X.real == 0) & (X.imag == 0)
    return torch.where(m.reshape(X.shape) | zero, torch.zeros((), dtype=torch.complex64), g)


def bits(t):
    """The bit patterns of a complex64 tensor (NaN payloads and signed zeros included)."""
    return torch.view_as_real(t.detach().cpu().contiguous()).view(torch.int32)


# --------------------------------------------------------------------------- rotate
def rotate(X, s):
    return X.detach().cpu().to(torch.complex128) * torch.exp(1j * s.detach().cpu().double())


# --------------------------------------------------------------------------- mask_low
def power(X):
    return X.detach().cpu().to(torch.complex128).abs() ** 2


def mask_low_floor(X, amin=1e-5, top_db=80.0):
    """log_magnitude()'s top_db floor of the whole batch, NaN when the batch holds a NaN (as log_spec.max())."""
    pmax = power(X).max()  # torch.max propagates NaN
    return 10.0 * torch.log10(torch.clamp(pmax, min=amin ** 2)) - top_db


def mask_low_decision(X, cut, amin=1e-5, top_db=80.0):
    """-> (masked, undecided) [shape of X]: masked by the float64 evaluation, undecided when the float32 one may differ.
    ``cut`` has one value per item."""
    B = X.shape[0]
    p = power(X)
    floor = mask_low_floor(X, amin, top_db)
    db = 10.0 * torch.log10(torch.clamp(p, min=amin ** 2))  # clamp keeps NaN
    dbf = torch.maximum(db, floor)                            # maximum propagates NaN
    c = cut.detach().cpu().double().reshape(-1).expand(B).reshape(B, *([1] * (X.ndim - 1)))
    masked = dbf < c
    marg = torch.from_numpy(db_margin(db.numpy()) + db_margin(floor.numpy()))
    with np.errstate(invalid="ignore"):
        undecided = (dbf - c).abs() <= marg
    return masked, undecided & torch.isfinite(dbf)


def unit(X):
    """X / |X| by the reference's angle: exp(1j angle X), 1 at X == 0 (angle(+0 + 0j) = 0)."""
    Xd = X.detach().cpu().to(torch.complex128)
    return torch.exp(1j * torch.angle(Xd))


def mask_low_value(X, val):
    return float(val) * unit(X)


def mask_low_grad(g, X, val):
    """d(val exp(1j angle X)) applied to g: val (g - Re(g conj w) w) / |X|."""
    Xd = X.detach().cpu().to(torch.complex128)
    gd = g.detach().cpu().to(torch.complex128)
    w = Xd / Xd.abs()
    return float(val) * (gd - (gd * w.conj()).real * w) / Xd.abs()


# --------------------------------------------------------------------------- gate
def gate_db(X):
    return 20.0 * torch.log10(torch.clamp(X.detach().cpu().to(torch.complex128).abs(), min=1e-4))


def thresholds(nz, n_std):
    """[rows, F] float64: mean + n_std * unbiased std over frames of the noise's dB (NaN for one frame, as torch.std)."""
    d = gate_db(nz).reshape(-1, nz.shape[-2], nz.shape[-1])
    if d.shape[-1] == 1:
        return torch.full(d.shape[:2], float("nan"), dtype=torch.float64)
    return d.mean(-1) + d.std(-1) * n_std


def thresh_scale(nz, n_std):
    """The error scale of gate_stats_kernel's threshold, per (row, bin): each of 32 lanes sums ceil(N / 32) dB values in
    sequence, then a 5-level shuffle tree, once for the mean and once for the squared deviations.  With A the largest
    |db|, a = 60 + 6 A the bound of one dB value (``db_margin``) and k = ceil(N / 32) + 5 the summation depth:
      mean:  m = a + k mean|db| + |mean|
      std:   (a + m + A + |mean|) sqrt(N / (N - 1)) + (k + 2) std
      total: m + |n_std| std-bound + |thresh|"""
    d = gate_db(nz).reshape(-1, nz.shape[-2], nz.shape[-1])
    N = d.shape[-1]
    k = math.ceil(N / 32) + 5
    A = d.abs().amax(-1)
    a = 60.0 + 6.0 * A
    mean = d.mean(-1)
    std = d.std(-1) if N > 1 else torch.zeros_like(mean)
    m = a + k * d.abs().mean(-1) + mean.abs()
    s = (a + m + A + mean.abs()) * math.sqrt(N / max(N - 1, 1)) + (k + 2) * std
    return m + abs(n_std) * s + (mean + n_std * std).abs()


def gate_bracket(X, th, smooth_f, smooth_t):
    """(S_lo, S_hi, undecided) [B, C, F, N] float64: the zero-padded cross-correlation of the booleans
    db(X) < th[row or 0, bin] with outer(smooth_f, smooth_t) / its sum, undecided cells counted 0 and 1.  ``th`` is
    [1 or B * C, F] (the kernel's own thresholds)."""
    B, C, F, N = X.shape
    db = gate_db(X).reshape(B * C, F, N)
    t = th.detach().cpu().double().reshape(-1, F, 1)
    below = db < t
    with np.errstate(invalid="ignore"):
        und = ((db - t).abs() <= torch.from_numpy(db_margin(db.numpy()))) & torch.isfinite(db) & torch.isfinite(t)
    rf = torch.tensor([float(v) for v in smooth_f], dtype=torch.float64)
    rt = torch.tensor([float(v) for v in smooth_t], dtype=torch.float64)
    w = torch.outer(rf, rt)
    w = (w / w.sum())[None, None]
    pad = (len(smooth_f) // 2, len(smooth_t) // 2)
    lo = Fn.conv2d((below & ~und).double()[:, None], w, padding=pad)[:, 0]
    hi = Fn.conv2d((below | und).double()[:, None], w, padding=pad)[:, 0]
    return lo.reshape(B, C, F, N), hi.reshape(B, C, F, N), und.reshape(B, C, F, N)


def s_scale(n_f, n_t, amount):
    """The error scale of the kernel's S recovered from its output: the two fmaf passes of n_t and n_f weights (S <= 1),
    and the roundings of 1 - amount S and of the product, divided by amount."""
    return n_f + n_t + 4.0 / amount


def reference_gate(X, nz, n_std, amount, smooth_f, smooth_t):
    """The reference's gate restated in float64 on the host, non-finite values included: the output factor
    1 - amount * conv2d(db(X) < thresh) per cell, [B, C, F, N].  Nothing here depends on the kernels."""
    B, C, F, N = X.shape
    nzb = nz.expand(B, C, -1, -1) if nz.shape[:2] != (1, 1) else nz
    th = thresholds(nzb, n_std).reshape(-1, F, 1)
    mask = (gate_db(X).reshape(B * C, F, N) < th).double()
    rf = torch.tensor([float(v) for v in smooth_f], dtype=torch.float64)
    rt = torch.tensor([float(v) for v in smooth_t], dtype=torch.float64)
    w = torch.outer(rf, rt)
    S = Fn.conv2d(mask[:, None], (w / w.sum())[None, None], padding=(len(smooth_f) // 2, len(smooth_t) // 2))
    amt = amount.detach().cpu().double().reshape(-1).expand(B).repeat_interleave(C)[:, None, None]
    return (1.0 - amt * S[:, 0]).reshape(B, C, F, N)
