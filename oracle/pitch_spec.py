"""CPU oracle for pitch_shift / time_stretch -- TEST INFRASTRUCTURE ONLY (imported by tests/ and nothing else).

What it pins.  The reference's ``EffectMixin.pitch_shift`` / ``time_stretch`` (ref:audiotools/core/effects.py:247-309)
hand the rows to libsox (``pitch -q <cents>`` / ``tempo -q <factor>`` + ``rate``), whose source is not under
/root/reference and whose output the reference's own tests never pin (ref:tests/core/test_effects.py:156-181 checks
batch[0] == single only).  SoX's pitch effect is WSOLA time-scale modification followed by a rate change; the product
states that construction as a written specification (header of ``audiotools_b200/csrc/pitch.cu``).  This module is an
INDEPENDENT restatement of that specification -- plain numpy, float64 accumulation, written from the prose, sharing no
code with the kernels -- so the CUDA path is compared with something other than itself:

  r = 2^(semitones / 12)   (time_stretch by ``factor``: semitones = float32(12 log2(1 / factor)), stages 1-2 only)
  geometry   W = the power of two nearest (log scale) to 0.046 sr, clamped to [64, 2048]; synthesis hop Hs = W/2;
             search radius D = W/8; Lc = W/4 correlation terms taken every 2nd sample; J = int(T r / Hs) + 2 frames
  1. search  p_0 = 0.  Frame j >= 1: nominal a_j = floor(j Hs / r + 1/2), continuation cont = p_{j-1} + Hs.
             If cont + 2 Lc <= T and a_j - D >= 0 and a_j + D + 2 Lc <= T:
               p_j = a_j + argmax_{d in [-D, D)} sum_{i < Lc} x[cont + 2 i] x[a_j + d + 2 i]
               (ties: smaller |d|, then the negative one; a NaN correlation never wins; no winner -> d = 0)
             else p_j = clamp(a_j, 0, max(T - W, 0)).
  2. overlap-add   s[u] = h x[p_J + t] + (1 - h) x[p_{J-1} + t + Hs],  J = u // Hs, t = u % Hs,
             h = 1/2 - 1/2 cos(pi t / Hs); samples outside [0, T) and frames outside [0, J) read as 0;
             u in [0, ceil(T r) + half + 2) (time_stretch: u in [0, round(T / factor)))
  3. rate    y[n] = sum_k w_k s[ip + k - half + 1] / sum_k w_k,  P = n r, ip = int(P), f = P - ip, k = 0 .. 2 half - 1,
             t_k = 1 - half - f + k,  w_k = (1/2 + 1/2 cos(pi t_k / half)) sin(pi c t_k) / t_k  (-> pi c at t_k = 0),
             c = 0.95 min(1, 1/r), half = ceil(8 / c); s[u] = 0 for u < 0.

Parity status: the SPECIFICATION is pinned by this oracle (exact splice positions wherever the arg-max is decided by
more than float32 rounding, waveforms to 1e-4); parity with libsox itself stays unpinned (no numeric pin exists in the
reference), which DESIGN.md states.
"""
import math

import numpy as np


class Geometry:
    def __init__(self, T: int, sr: int, semitones: float):
        st = float(np.float32(semitones))
        self.r = 2.0 ** (st / 12.0)
        W, target = 1, 0.046 * sr
        while W * 2 <= target * math.sqrt(2.0):
            W *= 2
        self.W = min(max(W, 64), 2048)
        self.Hs, self.D, self.Lc = self.W // 2, self.W // 8, self.W // 4
        self.J = int(T * self.r / self.Hs) + 2
        self.c = 0.95 * (1.0 / self.r if self.r > 1.0 else 1.0)
        self.half = int(math.ceil(8.0 / self.c))
        self.Ls = int(math.ceil(T * self.r)) + self.half + 2
        self.T = T


def stretch_semitones(factor: float) -> float:
    return float(np.float32(12.0 * math.log2(1.0 / factor)))


def splice_positions(x: np.ndarray, geo: Geometry):
    """Positions p_j of one row and, per searched frame, the relative margin between the best and second best
    correlation (inf for frames that were not searched): where the margin is below float32 rounding of the sum, a
    float32 implementation may legitimately pick the runner-up."""
    x = np.asarray(x, dtype=np.float64)
    T, g = len(x), geo
    pos = np.zeros(g.J, dtype=np.int64)
    margin = np.full(g.J, np.inf)
    span = 2 * g.Lc
    idx = 2 * np.arange(g.Lc)
    offs = np.arange(-g.D, g.D)
    for j in range(1, g.J):
        a = int(math.floor(j * g.Hs / g.r + 0.5))
        cont = int(pos[j - 1]) + g.Hs
        best = min(max(a, 0), max(T - g.W, 0))
        if cont + span <= T and a - g.D >= 0 and a + g.D + span <= T:
            tmpl = x[cont + idx]
            win = x[a - g.D: a + g.D + span]
            cand = np.lib.stride_tricks.sliding_window_view(win, span)[: 2 * g.D, ::2]  # [2D, Lc]
            corr = cand @ tmpl
            ok = ~np.isnan(corr)
            if ok.any():
                cm = np.where(ok, corr, -np.inf)
                top = cm.max()
                tied = np.nonzero(cm == top)[0]
                d = min((int(offs[i]) for i in tied), key=lambda v: (abs(v), v))
                best = a + d
                rest = np.delete(cm, np.nonzero(offs == d)[0][0])
                scale = float(np.abs(cand).dot(np.abs(tmpl)).max()) + 1e-300  # size of the terms being summed
                margin[j] = (top - rest.max()) / scale if rest.size else np.inf
        pos[j] = best
    return pos, margin


def overlap_add(x: np.ndarray, pos: np.ndarray, geo: Geometry, n=None) -> np.ndarray:
    """s[0 .. n), n = Ls unless given (frames outside [0, J) read as 0, so s is defined at every u >= 0)."""
    x = np.asarray(x, dtype=np.float64)
    T, g = len(x), geo
    u = np.arange(g.Ls if n is None else n)
    Jn, t = u // g.Hs, u % g.Hs
    h = 0.5 - 0.5 * np.cos(np.pi * t / g.Hs)

    def take(frame, shift):
        valid = (frame >= 0) & (frame < g.J)
        p = pos[np.clip(frame, 0, g.J - 1)] + t + shift
        valid &= (p >= 0) & (p < T)
        return np.where(valid, x[np.clip(p, 0, T - 1)], 0.0)

    return h * take(Jn, 0) + (1.0 - h) * take(Jn - 1, g.Hs)


def rate_change(s: np.ndarray, geo: Geometry) -> np.ndarray:
    g = geo
    n = np.arange(g.T)
    P = n * g.r
    ip = P.astype(np.int64)
    f = P - ip
    k = np.arange(2 * g.half)
    t = (1 - g.half - f)[:, None] + k[None, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        sinc = np.where(np.abs(t) < 1e-12, np.pi * g.c, np.sin(np.pi * g.c * t) / t)
    w = (0.5 + 0.5 * np.cos(np.pi * t / g.half)) * sinc
    src = ip[:, None] + k[None, :] - g.half + 1
    sv = np.where((src >= 0) & (src < len(s)), s[np.clip(src, 0, len(s) - 1)], 0.0)
    return (w * sv).sum(axis=1) / w.sum(axis=1)


def pitch_shift_row(x: np.ndarray, sr: int, semitones: float, positions=None):
    """One row: returns (y [T] float64, positions [J], margins [J]).  ``positions`` forces the splice positions (to
    check stages 2-3 of an implementation whose float32 arg-max legitimately differs at a near-tie)."""
    geo = Geometry(len(x), sr, semitones)
    if float(np.float32(semitones)) == 0.0:
        return np.asarray(x, dtype=np.float64).copy(), np.zeros(0, dtype=np.int64), np.zeros(0)
    pos, margin = splice_positions(x, geo)
    use = pos if positions is None else np.asarray(positions[: geo.J], dtype=np.int64)
    return rate_change(overlap_add(x, use, geo), geo), pos, margin


def time_stretch_row(x: np.ndarray, sr: int, factor: float, positions=None):
    """One row: returns (out [round(T / factor)] float64, positions, margins)."""
    T = len(x)
    out_len = int(math.floor(T / factor + 0.5))
    if factor == 1.0:
        out = np.zeros(out_len)
        out[: min(T, out_len)] = x[: min(T, out_len)]
        return out, np.zeros(0, dtype=np.int64), np.zeros(0)
    geo = Geometry(T, sr, stretch_semitones(factor))
    pos, margin = splice_positions(x, geo)
    use = pos if positions is None else np.asarray(positions[: geo.J], dtype=np.int64)
    # T r (r from float32 semitones) can fall short of T / factor: the overlap-add runs on to out_len
    return overlap_add(x, use, geo, out_len), pos, margin
