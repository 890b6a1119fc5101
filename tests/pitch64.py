"""Float64 restatement of the pitch shifter and the time stretch of csrc/pitch.cu (DESIGN.md K5) with per-frame and
per-sample error models: the oracle of tests/test_gpu_pitch_accuracy.py and tests/test_sim_pitch_accuracy.py.

The definition is oracle/pitch_spec.py's.  This module adds what the kernels' own arithmetic needs to be checked stage by
stage on their own outputs, so a near-tie that the float32 search legitimately flips does not hide the rest of the row:

* ``Geo``: the library's geometry (the stretched row's halo H and stride SL, the staged region's capacity rcap) and the
  search kernel's tiling: the 2 D candidates of a frame are summed over KS tap slices of TS taps each, TS / 8 register
  steps per slice (W 64..512: one step, the tail step only; W 1024: two; W 2048: eight, the ping-pong loop only).
* ``check_search``: every frame j >= 1 of a row against the kernel's own previous position, cont = p^_{j-1} + Hs.  A
  searched frame's correlations c_d (float64) and S_d = sum |x_cont| |x_cand| bound the float32 ones: the kernel sums TS
  products with sequential FMAs per slice and then the KS slice partials in order, so |c^_d - c_d| <= gamma S_d with
  gamma = (TS + KS + 1) u.  The kernel's choice must therefore satisfy c(p^) >= max_d c_d - gamma (S_chosen + S_best);
  where the float64 margin exceeds that bound it is the arg-max under the tie rule exactly.  A frame that is not
  searched must sit at clamp(a_j, 0, max(T - W, 0)).  ``region_of`` restates the kernel's staged region so a test can
  prove that the template was read from global memory (the continuation outside the region).
* ``ola64``: s[u] = h a + (1 - h) b from the kernel's positions, with a, b the two source samples; per sample
  |s^ - s| <= C_O u (|a| + |b|) (one ``cospif``, a product and an FMA).
* ``rate64``: y[n] = sum_k w_k s_k / sum_k w_k.  Per output e_n = |y^ - y| / (u sum_k env_k |s_k| / |sum_k w_k|) on
  the kernel's own stretched samples s^, budget C_R 2 half: the 2 half weights come from two float32 Chebyshev
  recurrences whose error grows with the tap count.  env_k = min(pi c, 1 / |t_k|) bounds |w_k| and sets the scale of
  its absolute error (|w_k| itself would not: the float64 weight at t = +-half is exactly 0, the float32 one is not).  End to end, y^ against the rate change of the float64 overlap-add is held to
  the sum of the two bounds.

Non-finite samples: NaN and inf must land where the float64 computation puts them, sample for sample.  Budgets were
measured on an NVIDIA H100 80GB HBM3 (DESIGN.md "Pitch accuracy")."""
import math

import numpy as np

from oracle import pitch_spec as ps

U = 2.0 ** -24
ST = 512     # search threads per CTA
C_O = 5.0    # overlap-add, units of u (|a| + |b|); 2.46 measured on the H100
C_R = 11.0   # rate change, units of u sum env |s| / |sum w| per tap (2 half taps); 5.37 measured on the H100

RATES = [1000, 2000, 4000, 8000, 16000, 22050, 44100, 48000, 192000]
SHIFTS = [-24.0, -12.0, -7.0, -2.0, -0.5, -0.01, 0.01, 0.5, 2.0, 7.0, 12.0, 24.0]


class Geo(ps.Geometry):
    def __init__(self, T: int, sr: int, semitones: float, min_len: int = 0):
        super().__init__(T, sr, semitones)
        self.semitones = float(np.float32(semitones))
        self.identity = self.semitones == 0.0
        self.span = 2 * self.Lc
        self.H = (self.half + 3) & ~3
        self.SL = (self.H + max(self.Ls, min_len) + 3) // 4 * 4
        drift = int(math.ceil(abs(self.Hs / self.r - self.Hs))) + 1
        self.rcap = (2 * self.D + 2 * self.Lc + drift + 48 + 63) // 64 * 64
        G = self.D >> 3
        self.KS = min(ST // (2 * G), self.Lc >> 3)
        self.TS = self.Lc // self.KS
        self.steps = self.TS >> 3
        self.gamma = (self.TS + self.KS + 1) * U
        self.nom = np.floor(np.arange(self.J) * self.Hs / self.r + 0.5).astype(np.int64)

    def searched_nominal(self, j: int) -> bool:
        """The part of frame j's search condition that does not depend on the previous position."""
        a = int(self.nom[j])
        return a - self.D >= 0 and a + self.D + self.span <= self.T


def stretch_geo(T: int, sr: int, factor: float) -> Geo:
    return Geo(T, sr, ps.stretch_semitones(factor), min_len=stretch_out_len(T, factor))


def stretch_out_len(T: int, factor: float) -> int:
    return int(math.floor(T / factor + 0.5))


def pos_bytes(rows: int, geos) -> int:
    """Bytes of the position and nominal tables in front of the stretched rows in the workspace."""
    jmax = max(g.J for g in geos)
    return ((rows + len(geos)) * jmax * 4 + 255) // 256 * 256


def workspace_bytes(rows: int, geos) -> int:
    return pos_bytes(rows, geos) + rows * max(g.SL for g in geos) * 4


def region_of(aj: int, ap: int, g: Geo):
    """The kernel's staged region [lo, lo + rn) of the frame with nominal aj after the one with nominal ap."""
    mn = min(aj - g.D, ap - g.D + g.Hs)
    mx = max(aj + g.D + g.span, ap + g.D + g.Hs + g.span)
    lo = aj - g.D - 16 * ((aj - g.D - mn + 15) >> 4)
    rn = min((mx - lo + 15) & ~15, g.rcap)
    return lo, rn


def template_always_staged(g: Geo, frames: int):
    """(ok, headroom): ok if, for frames 1 .. frames - 1, every continuation a searched frame can have lies inside its
    staged region, so the kernel's global-memory template branch is never taken; headroom = the least rcap minus the
    unclamped region length (the clamp to rcap binds nowhere if it is >= 0).  The previous frame's position is either searched,
    p in [a_{j-1} - D, a_{j-1} + D), or clamped, min(a_{j-1}, T - W) with T >= a_j + D + 2 Lc (frame j is searched),
    which lies in [a_j + D - Hs, a_{j-1}]; frame 0 sits at 0."""
    nom = np.floor(np.arange(frames) * g.Hs / g.r + 0.5).astype(np.int64)
    headroom = g.rcap
    for j in range(1, frames):
        aj, ap = int(nom[j]), int(nom[j - 1])
        lo, rn = region_of(aj, ap, g)
        mx = max(aj + g.D + g.span, ap + g.D + g.Hs + g.span)
        headroom = min(headroom, g.rcap - ((mx - lo + 15) & ~15))
        p_lo = 0 if j == 1 else min(ap - g.D, aj + g.D - g.Hs)
        p_hi = 0 if j == 1 else ap + g.D - 1
        c_lo, c_hi = p_lo + g.Hs - lo, p_hi + g.Hs - lo
        if c_lo < 0 or c_hi + g.span > rn:
            return False, headroom
    return True, headroom


def first_searched_length(g_of_T, lo: int = 1, hi: int = 1 << 16) -> int:
    """Smallest T at which frame 1 is searched (p_0 = 0, so cont = Hs); ``g_of_T(T)`` builds the geometry."""
    for T in range(lo, hi):
        g = g_of_T(T)
        if g.J > 1 and g.Hs + g.span <= T and g.searched_nominal(1):
            return T
    raise AssertionError("frame 1 is never searched")


def last_search_flips(g_of_T, T0: int, count: int = 2):
    """The first ``count`` lengths >= T0 at which the index of the last frame whose nominal search condition holds
    changes from T - 1 to T."""
    def last(T):
        g = g_of_T(T)
        return max([j for j in range(1, g.J) if g.searched_nominal(j)], default=0)

    out, prev, T = [], last(T0 - 1), T0
    while len(out) < count:
        cur = last(T)
        if cur != prev:
            out.append(T)
        prev, T = cur, T + 1
    return out


def tied_positions(g: Geo):
    """The positions when every correlation of every searched frame ties (silence, DC): d = 0 where searched, the
    clamped nominal position elsewhere."""
    pos = np.zeros(g.J, dtype=np.int64)
    for j in range(1, g.J):
        a = int(g.nom[j])
        searched = pos[j - 1] + g.Hs + g.span <= g.T and g.searched_nominal(j)
        pos[j] = a if searched else min(max(a, 0), max(g.T - g.W, 0))
    return pos


def _pick(offs, cm, top):
    tied = np.nonzero(cm == top)[0]
    return min((int(offs[i]) for i in tied), key=lambda v: (abs(v), v))


def check_search(x, pos, g: Geo, where="", j0: int = 1):
    """Every frame j >= j0 of one row against the kernel's own previous position (see the module docstring).  Returns
    {"slack": worst (c_best - c_chosen) / (gamma (S_chosen + S_best)), "searched", "fallback": frames whose template
    came from global memory, "flips": frames where the kernel chose other than the float64 arg-max}."""
    x = np.asarray(x, dtype=np.float64)
    pos = np.asarray(pos[: g.J], dtype=np.int64)
    T = len(x)
    idx = 2 * np.arange(g.Lc)
    offs = np.arange(-g.D, g.D)
    st = {"slack": 0.0, "searched": 0, "fallback": 0, "flips": 0}
    assert pos[0] == 0, (where, pos[0])
    for j in range(max(j0, 1), g.J):
        a, cont, p = int(g.nom[j]), int(pos[j - 1]) + g.Hs, int(pos[j])
        if not (cont + g.span <= T and g.searched_nominal(j)):
            want = min(max(a, 0), max(T - g.W, 0))
            assert p == want, (where, "unsearched frame", j, p, want)
            continue
        st["searched"] += 1
        lo, rn = region_of(a, int(g.nom[j - 1]), g)
        c = cont - lo
        st["fallback"] += int(c < 0 or c + g.span > rn)
        d = p - a
        assert -g.D <= d < g.D, (where, "offset outside the search", j, d)
        tmpl = x[cont + idx]
        cand = np.lib.stride_tricks.sliding_window_view(x[a - g.D: a + g.D + g.span], g.span)[: 2 * g.D, ::2]
        with np.errstate(invalid="ignore", over="ignore"):
            corr = cand @ tmpl
            S = np.abs(cand) @ np.abs(tmpl)
        ok = ~np.isnan(corr)
        if not ok.any():
            assert d == 0, (where, "every correlation is NaN: d must be 0", j, d)
            continue
        cm = np.where(ok, corr, -np.inf)
        top = cm.max()
        best = _pick(offs, cm, top)
        cp = corr[d + g.D]
        assert not np.isnan(cp), (where, "a NaN correlation won", j, d)
        st["flips"] += int(d != best)
        tol = g.gamma * (S[d + g.D] + S[best + g.D])
        if not np.isfinite(tol) or not np.isfinite(top):
            assert cp == top or np.isfinite(top), (where, "an infinite correlation lost", j, d, best)
            continue
        if S.max() == 0.0:  # every product is an exact zero: the float32 sums tie exactly, the tie rule decides
            assert d == best, (where, "exact tie broken wrongly", j, d, best)
            continue
        slack = (top - cp) / tol if tol > 0 else (0.0 if cp == top else np.inf)
        assert slack <= 1.0, (where, "frame", j, "chose", d, "float64 best", best, "slack", slack)
        st["slack"] = max(st["slack"], slack)
    return st


def ola64(x, pos, g: Geo, u0: int, u1: int):
    """s[u], a[u], b[u] for u in [u0, u1): s = h a + (1 - h) b, a = frame J's sample, b = frame J-1's (0 outside the
    row or outside frames [0, J)); the formula of pitch_spec.overlap_add on a window of u."""
    x = np.asarray(x, dtype=np.float64)
    pos = np.asarray(pos[: g.J], dtype=np.int64)
    T = len(x)
    u = np.arange(u0, u1)
    Jn, t = u // g.Hs, u % g.Hs
    h = 0.5 - 0.5 * np.cos(np.pi * t / g.Hs)

    def take(frame, shift):
        valid = (frame >= 0) & (frame < g.J)
        p = pos[np.clip(frame, 0, g.J - 1)] + t + shift
        valid &= (p >= 0) & (p < T)
        return np.where(valid, x[np.clip(p, 0, T - 1)], 0.0)

    a, b = take(Jn, 0), take(Jn - 1, g.Hs)
    with np.errstate(invalid="ignore"):
        return h * a + (1.0 - h) * b, a, b


def rate_taps(g: Geo, n):
    """Weights w [len(n), 2 half] (float64), their envelope min(pi c, 1 / |t|) (the scale of a weight's absolute
    error: the recurrences carry an error of a few u in sin(pi c t) and in the window, divided by t; a tap where the
    float64 weight is exactly 0, t = +-half, is not exact in float32) and the stretched index each tap reads."""
    P = np.asarray(n, dtype=np.int64) * g.r
    ip = P.astype(np.int64)
    f = P - ip
    k = np.arange(2 * g.half)
    t = (1 - g.half - f)[:, None] + k[None, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        sinc = np.where(np.abs(t) < 1e-12, np.pi * g.c, np.sin(np.pi * g.c * t) / t)
    w = (0.5 + 0.5 * np.cos(np.pi * t / g.half)) * sinc
    with np.errstate(divide="ignore"):
        env = np.minimum(np.pi * g.c, 1.0 / np.abs(t))
    return w, env, ip[:, None] + k[None, :] - g.half + 1


def rate64(w, env, src, s, s0: int):
    """y = sum w s / sum w with s[u] held at s[u - s0] (s = 0 for u < 0), and the error unit
    m = sum env |s| / |sum w|."""
    sv = np.where(src >= 0, s[np.clip(src - s0, 0, len(s) - 1)], 0.0)
    wsum = w.sum(axis=1)
    with np.errstate(invalid="ignore", over="ignore"):
        y = (w * sv).sum(axis=1) / wsum
        m = (env * np.abs(sv)).sum(axis=1) / np.abs(wsum)
    return y, m, sv


def _held(got, ref, unit, C, what, where, skip=None):
    """|got - ref| <= C unit per sample where ref and unit are finite; NaN and inf where ref has them, except at
    ``skip``.  Returns the worst |got - ref| / unit (0 where unit is 0, which requires got == ref)."""
    got = np.asarray(got, dtype=np.float64)
    keep = np.ones(len(ref), bool) if skip is None else ~skip
    nan_diff = (np.isnan(got) != np.isnan(ref)) & keep
    assert not nan_diff.any(), (where, what, "NaN positions differ", np.nonzero(nan_diff)[0][:8])
    inf = np.isinf(ref) & keep
    assert np.array_equal(got[inf], ref[inf]), (where, what, "inf samples differ")
    m = np.isfinite(ref) & np.isfinite(unit) & keep
    err = np.abs(got[m] - ref[m])
    z = unit[m] == 0
    assert np.all(err[z] == 0), (where, what, "nonzero error where the result is exact")
    e = np.zeros_like(err)
    e[~z] = err[~z] / unit[m][~z]
    worst = float(e.max()) if e.size else 0.0
    assert worst <= C, (where, what, "error", worst, "budget", C, "at", np.nonzero(m)[0][np.argmax(e)] if e.size else -1)
    return worst


def check_ola(x, pos, s_hat, g: Geo, u0: int, u1: int, where=""):
    """s^[u0 .. u1) (the kernel's stretched samples) per sample against ola64; returns the worst C_o."""
    s, a, b = ola64(x, pos, g, u0, u1)
    with np.errstate(invalid="ignore"):
        unit = U * (np.abs(a) + np.abs(b))
    return _held(s_hat, s, unit, C_O, "overlap-add", where)


def check_rate(x, pos, y_hat, s_hat, g: Geo, n0: int, n1: int, where=""):
    """y^[n0 .. n1) per output: against the float64 rate change of the kernel's own s^ (budget C_R 2 half, the
    returned worst is in units of 2 half), and against the rate change of the float64 overlap-add within the sum of
    both bounds.  ``s_hat`` holds the kernel's s[0 .. len(s_hat))."""
    n = np.arange(n0, n1)
    w, env, src = rate_taps(g, n)
    s_hat = np.asarray(s_hat, dtype=np.float64)
    y1, m1, sv = rate64(w, env, src, s_hat, 0)
    # a tap whose weight is within its error bound of 0 (exactly 0 at t = +-half for an integer read position, or next
    # to a zero of the sinc) has no decided sign in float32: a non-finite sample there can be inf in the kernel and NaN
    # (0 inf, or inf - inf with another tap) in float64, so those outputs' NaN and inf are not compared
    skip = ((np.abs(w) <= C_R * 2 * g.half * U * env) & ~np.isfinite(sv)).any(axis=1)
    worst = _held(y_hat, y1, U * m1, C_R * 2 * g.half, "rate change", where, skip) / (2 * g.half)
    u0 = max(0, int(src.min()))
    u1 = int(src.max()) + 1
    s, a, b = ola64(x, pos, g, u0, u1)
    y2, m2, _ = rate64(w, env, src, s, u0)
    _, mab, _ = rate64(w, env, src, np.abs(a) + np.abs(b), u0)
    with np.errstate(invalid="ignore", over="ignore"):
        unit = U * (C_R * 2 * g.half * m2 + C_O * mab)
    _held(y_hat, y2, unit, 1.0, "end to end", where, skip)
    return worst


def check_pitch_row(x, y_hat, pos, s_hat, g: Geo, where=""):
    """One row of a pitch shift: search, overlap-add and rate change.  ``s_hat`` is the kernel's stretched row with its
    halo (the workspace row, >= SL floats).  Returns the search statistics plus "C_o" and "C_r"."""
    if g.identity:
        assert np.array_equal(np.asarray(y_hat), np.asarray(x)), (where, "a shift of 0 must copy the row")
        return {"slack": 0.0, "searched": 0, "fallback": 0, "flips": 0, "C_o": 0.0, "C_r": 0.0}
    st = check_search(x, pos, g, where)
    s_row = np.asarray(s_hat[g.H: g.SL], dtype=np.float64)
    assert np.all(np.asarray(s_hat[: g.H]) == 0), (where, "the halo in front of the stretched row is not zero")
    st["C_o"] = check_ola(x, pos, s_row, g, 0, len(s_row), where)
    st["C_r"] = check_rate(x, pos, y_hat, s_row, g, 0, g.T, where)
    return st


def check_stretch_row(x, out, pos, g: Geo, where=""):
    """One row of a time stretch: search and the overlap-add, which is the output."""
    st = check_search(x, pos, g, where)
    st["C_o"] = check_ola(x, pos, out, g, 0, len(out), where)
    return st


# --------------------------------------------------------------------------- signals
def signal(kind: str, T: int, sr: int, seed: int) -> np.ndarray:
    """float32 rows: noise (at three levels), a tone under weak noise (near-tie correlations), silence, DC, an impulse
    train, and noise with one NaN or one inf."""
    rng = np.random.default_rng(abs(int(seed)))
    n = np.arange(T)
    noise = 0.3 * rng.standard_normal(T)
    if kind == "noise":
        x = noise
    elif kind == "noise_1e-3":
        x = 1e-3 * noise
    elif kind == "noise_1e-6":
        x = 1e-6 * noise
    elif kind == "tone+noise":
        x = 0.5 * np.sin(2 * np.pi * 0.0371 * n + 0.3) + 1e-3 * noise
    elif kind == "silence":
        x = np.zeros(T)
    elif kind == "dc":
        x = np.full(T, 0.25)
    elif kind == "impulses":
        x = np.where(n % 37 == 5, 0.8, 0.0)
    elif kind in ("nan", "inf"):
        x = noise.copy()
        x[T // 3] = np.nan if kind == "nan" else np.inf
    else:
        raise KeyError(kind)
    return x.astype(np.float32)


KINDS = ["noise", "tone+noise", "silence", "dc", "impulses", "noise_1e-3", "noise_1e-6", "nan", "inf"]
