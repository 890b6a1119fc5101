"""The pitch shifter and the time stretch on the H100 (``-m gpu``) against float64, per splice and per sample
(tests/pitch64.py): ``wsola_search_kernel`` per frame against the kernel's own previous position, ``wsola_ola_kernel``
per stretched sample and ``rate_kernel`` per output, at every frame size the geometry picks (W 64 .. 2048, both loop
shapes of the search), shifts from -24 to +24 semitones, lengths around a frame, the first searched frame and the last
one, silence, DC, impulses, quiet rows and non-finite samples; launches that mix eight geometries; a flat index past
2^31; and exact invariances (power-of-two scaling, negation, row independence).  tests/probes/pitch_accuracy_probe.py
prints the table of DESIGN.md "Pitch accuracy"."""
import ctypes
import math
import time

import numpy as np
import pytest
import torch

from audiotools_b200.engine import _dptr
from tests import pitch64 as p64

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


def run_pitch(eng, x, sr, shifts, groups=None):
    """x [rows, T] float32 (numpy) through ``b2a_pitch_shift_multi_f32`` with a workspace the caller keeps: returns
    (y [rows, T], positions [rows, Jmax], stretched rows with their halo [rows, SLmax], geometries per group)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    rows, T = x.shape
    sem = np.ascontiguousarray(shifts, dtype=np.float32)
    geos = [p64.Geo(T, sr, float(s)) for s in sem]
    sem_p = sem.ctypes.data_as(ctypes.c_void_p)
    ws_bytes = eng.lib.b2a_pitch_shift_multi_workspace_bytes(rows, T, sr, sem_p, len(sem))
    assert ws_bytes == p64.workspace_bytes(rows, geos), (T, sr, shifts)
    jmax, slmax, pb = max(g.J for g in geos), max(g.SL for g in geos), p64.pos_bytes(rows, geos)
    xd = torch.from_numpy(x).to(DEV)
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=DEV)
    out = torch.empty_like(xd)
    rg = None if groups is None else torch.as_tensor(np.asarray(groups, dtype=np.int32), device=DEV)
    eng._call(eng.lib.b2a_pitch_shift_multi_f32, _dptr(xd), rows, T, sr, sem_p, len(sem), _dptr(rg), _dptr(out),
              _dptr(ws), ws_bytes, eng._stream(xd))
    pos = ws[: rows * jmax * 4].view(torch.int32).reshape(rows, jmax).cpu().numpy()
    s = ws[pb: pb + rows * slmax * 4].view(torch.float32).reshape(rows, slmax).cpu().numpy()
    return out.cpu().numpy(), pos, s, geos


def run_stretch(eng, x, sr, factor):
    """x [rows, T] through ``Engine.time_stretch``: (out [rows, round(T / factor)], positions [rows, J])."""
    xd = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(DEV)
    out, pos = eng.time_stretch(xd, sr, factor, return_positions=True)
    return out.cpu().numpy(), pos.cpu().numpy()


def _merge(acc, st):
    for k, v in st.items():
        acc[k] = max(acc.get(k, 0), v) if k in ("slack", "C_o", "C_r") else acc.get(k, 0) + v
    return acc


def check_pitch(eng, sr, st, T, kinds, seed=0):
    """One launch of ``kinds`` rows of length T, every row checked; returns the merged statistics."""
    x = np.stack([p64.signal(k, T, sr, seed + i) for i, k in enumerate(kinds)])
    y, pos, s, (g,) = run_pitch(eng, x, sr, [st])
    acc = {}
    for i, k in enumerate(kinds):
        _merge(acc, p64.check_pitch_row(x[i], y[i], pos[i], s[i], g, where=(sr, st, T, k)))
        if k in ("silence", "dc"):  # every correlation ties: the nominal positions
            assert np.array_equal(pos[i, : g.J], p64.tied_positions(g)), (sr, st, T, k)
    return acc, x, y, pos


def check_stretch(eng, sr, factor, T, kinds, seed=0):
    x = np.stack([p64.signal(k, T, sr, seed + i) for i, k in enumerate(kinds)])
    if p64.stretch_out_len(T, factor) < 1:  # nothing to return: refused
        with pytest.raises(NotImplementedError):
            run_stretch(eng, x, sr, factor)
        return {}
    out, pos = run_stretch(eng, x, sr, factor)
    g = p64.stretch_geo(T, sr, factor)
    assert out.shape[1] == p64.stretch_out_len(T, factor)
    acc = {}
    for i, k in enumerate(kinds):
        _merge(acc, p64.check_stretch_row(x[i], out[i], pos[i], g, where=(sr, factor, T, k)))
    return acc


def edge_lengths(sr, st, main):
    """T = 1, 2, 3, Hs - 1, Hs, W - 1, W, W + 1, the first length at which frame 1 is searched and the one before,
    the first two lengths past W at which the last searched frame changes and the ones before, and main + 0 .. 3."""
    g0 = p64.Geo(1, sr, st)
    mk = lambda T: p64.Geo(T, sr, st)
    t1 = p64.first_searched_length(mk)
    flips = p64.last_search_flips(mk, g0.W + 1)
    Ts = {1, 2, 3, g0.Hs - 1, g0.Hs, g0.W - 1, g0.W, g0.W + 1, t1 - 1, t1}
    Ts |= {f - 1 for f in flips} | set(flips) | {main + i for i in range(4)}
    assert {T % 4 for T in Ts} == {0, 1, 2, 3}
    return sorted(T for T in Ts if T >= 1)


def main_length(sr):
    W = p64.Geo(1, sr, 0.0).W
    return 24 * W + 5


def factor_of(st):
    return 2.0 ** (-st / 12.0)


# --------------------------------------------------------------------------- geometry
def test_geometry_mirror_and_tiling(eng):
    """J against the library for every rate and shift; all six frame sizes and both loop shapes are reached."""
    seen = set()
    for sr in p64.RATES:
        for st in p64.SHIFTS + [0.0]:
            for T in (1, 1000, 48001, 10 ** 6 + 3):
                g = p64.Geo(T, sr, st)
                assert eng.lib.b2a_pitch_shift_num_frames(T, sr, st) == g.J, (sr, st, T)
                seen.add((g.W, g.KS, g.TS, g.steps))
    assert seen == {(64, 2, 8, 1), (128, 4, 8, 1), (256, 8, 8, 1), (512, 16, 8, 1), (1024, 16, 16, 2),
                    (2048, 8, 64, 8)}, seen


# --------------------------------------------------------------------------- per splice, per sample
@pytest.mark.parametrize("sr", p64.RATES)
@pytest.mark.parametrize("st", p64.SHIFTS)
def test_pitch_shift_per_splice_and_sample(eng, sr, st):
    main = main_length(sr)
    acc, x, y, pos = check_pitch(eng, sr, st, main, p64.KINDS, seed=int(sr + 100 * st))
    # the template never comes from global memory (tests/test_sim_pitch_accuracy.py proves it cannot)
    assert acc["searched"] > 0 and acc["fallback"] == 0, acc
    # a NaN or an inf changes its own row only
    xf = x.copy()
    for i, k in enumerate(p64.KINDS):
        if k in ("nan", "inf"):
            xf[i] = p64.signal("noise", main, sr, 12345 + i)
    yf = run_pitch(eng, xf, sr, [st])[0]
    keep = [i for i, k in enumerate(p64.KINDS) if k not in ("nan", "inf")]
    assert np.array_equal(y[keep], yf[keep])
    for T in edge_lengths(sr, st, main):
        assert check_pitch(eng, sr, st, T, ["noise", "tone+noise"], seed=T)[0]["fallback"] == 0


@pytest.mark.parametrize("sr", p64.RATES)
@pytest.mark.parametrize("st", p64.SHIFTS)
def test_time_stretch_per_splice_and_sample(eng, sr, st):
    fac = factor_of(st)
    main = main_length(sr)
    check_stretch(eng, sr, fac, main, ["noise", "tone+noise", "impulses", "noise_1e-6", "nan"], seed=int(sr - st))
    for T in edge_lengths(sr, st, main)[::2]:
        check_stretch(eng, sr, fac, T, ["noise"], seed=T)


def check_past_last_frame(eng, sr=1000, st=23.9, count=4):
    """At W = 64 and half > Hs the stretched row runs past frame J - 1's span: those samples come from frame J - 1
    alone (frame J is outside the row's frames and reads as 0).  Checked on the first ``count`` such lengths."""
    Ts = [T for T in range(300, 800) if (lambda g: g.J * g.Hs < g.SL - g.H)(p64.Geo(T, sr, st))][:count]
    assert len(Ts) == count
    for T in Ts:
        check_pitch(eng, sr, st, T, ["noise", "impulses"], seed=T)


def test_stretched_row_past_the_last_frame(eng):
    check_past_last_frame(eng)


MULTI = [-24.0, -7.0, -0.5, 0.0, 0.5, 7.0, 12.0, 24.0]


def check_multi(eng, sr, T, reps=2):
    """Eight geometries in one launch, rows interleaved: every row against float64 and bit for bit against its own
    single-shift launch; shift 0 copies."""
    n = len(MULTI)
    groups = np.tile(np.arange(n), reps)
    x = np.stack([p64.signal("noise" if i % 3 else "tone+noise", T, sr, 50 + i) for i in range(len(groups))])
    y, pos, s, geos = run_pitch(eng, x, sr, MULTI, groups)
    for i, gi in enumerate(groups):
        g = geos[gi]
        p64.check_pitch_row(x[i], y[i], pos[i], s[i], g, where=(sr, T, MULTI[gi], i))
        if MULTI[gi] == 0.0:
            assert np.array_equal(y[i], x[i])
        else:
            y1, pos1 = run_pitch(eng, x[i:i + 1], sr, [MULTI[gi]])[:2]
            assert np.array_equal(y[i], y1[0]) and np.array_equal(pos[i, : g.J], pos1[0, : g.J]), (sr, T, i)


@pytest.mark.parametrize("sr", [1000, 8000, 16000, 44100])
def test_multi_shift_launch(eng, sr):
    check_multi(eng, sr, main_length(sr) + 2)


# --------------------------------------------------------------------------- exact properties
def check_exact(eng, sr, st, T, rows_list=(1, 7, 300)):
    fac = factor_of(st)
    x = np.stack([p64.signal(k, T, sr, 7 + i) for i, k in enumerate(["noise", "tone+noise", "noise_1e-6"])])
    y, pos = run_pitch(eng, x, sr, [st])[:2]
    o, opos = run_stretch(eng, x, sr, fac)
    for k in (-20, -7, 1, 20):
        yk, posk = run_pitch(eng, x * np.float32(2.0 ** k), sr, [st])[:2]
        assert np.array_equal(yk, y * np.float32(2.0 ** k)) and np.array_equal(posk, pos), k
        ok, oposk = run_stretch(eng, x * np.float32(2.0 ** k), sr, fac)
        assert np.array_equal(ok, o * np.float32(2.0 ** k)) and np.array_equal(oposk, opos), k
    yn, posn = run_pitch(eng, -x, sr, [st])[:2]
    assert np.array_equal(yn, -y) and np.array_equal(posn, pos)
    on, oposn = run_stretch(eng, -x, sr, fac)
    assert np.array_equal(on, -o) and np.array_equal(oposn, opos)
    for rows in rows_list:
        xb = np.stack([p64.signal("noise", T, sr, 1000 + r) for r in range(rows)])
        yb, pb = run_pitch(eng, xb, sr, [st])[:2]
        ob, opb = run_stretch(eng, xb, sr, fac)
        for r in sorted({0, rows // 2, rows - 1}):
            y1, p1 = run_pitch(eng, xb[r:r + 1], sr, [st])[:2]
            o1, op1 = run_stretch(eng, xb[r:r + 1], sr, fac)
            assert np.array_equal(yb[r], y1[0]) and np.array_equal(pb[r], p1[0]), (rows, r)
            assert np.array_equal(ob[r], o1[0]) and np.array_equal(opb[r], op1[0]), (rows, r)


@pytest.mark.parametrize("sr,st", [(1000, 24.0), (8000, -7.0), (16000, 0.5), (44100, -24.0), (192000, 12.0)])
def test_exact_invariances(eng, sr, st):
    check_exact(eng, sr, st, main_length(sr) + 1)


# --------------------------------------------------------------------------- large
def test_flat_index_past_2_31(eng):
    """17 rows of 2^27 samples at -24 semitones (r = 1/4 keeps the workspace small): the last row's tail against
    float64 from the kernel's positions, and the last row equal to itself launched alone."""
    sr, st, rows, T = 44100, -24.0, 17, 1 << 27
    g = p64.Geo(T, sr, st)
    gen = torch.Generator(device=DEV).manual_seed(3)
    xd = 0.3 * torch.randn(rows, T, device=DEV, generator=gen)
    sem = np.asarray([st], dtype=np.float32)
    sem_p = sem.ctypes.data_as(ctypes.c_void_p)
    ws_bytes = eng.lib.b2a_pitch_shift_multi_workspace_bytes(rows, T, sr, sem_p, 1)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    out = torch.empty_like(xd)
    eng._call(eng.lib.b2a_pitch_shift_multi_f32, _dptr(xd), rows, T, sr, sem_p, 1, None, _dptr(out), _dptr(ws),
              ws_bytes, eng._stream(xd))
    pos = ws[: rows * g.J * 4].view(torch.int32).reshape(rows, g.J)[-1].cpu().numpy()
    last = out[-1].cpu().numpy()
    x_last = xd[-1:].clone()
    del out, ws
    y1 = eng.pitch_shift(x_last, sr, st)
    assert torch.equal(y1[0].cpu(), torch.from_numpy(last))
    x = x_last[0].cpu().numpy()
    assert p64.check_search(x, pos, g, where="2^31", j0=g.J - 64)["searched"] > 0
    n0 = T - 4096
    w, env, src = p64.rate_taps(g, np.arange(n0, T))
    u0, u1 = int(src.min()), int(src.max()) + 1
    s, a, b = p64.ola64(x, pos, g, u0, u1)
    y, m, _ = p64.rate64(w, env, src, s, u0)
    _, mab, _ = p64.rate64(w, env, src, np.abs(a) + np.abs(b), u0)
    p64._held(last[n0:], y, p64.U * (p64.C_R * 2 * g.half * m + p64.C_O * mab), 1.0, "tail past 2^31", "2^31")


def test_time_stretch_long_row_length(eng):
    """One row of 196 885 100 samples at factor 0.26875: T r with r from float32 semitones falls short of T / factor
    by more than the rate change's slack, which made the call fail its own length check.  The exact length comes
    back, and the last 4096 samples match float64 from the kernel's positions."""
    sr, T, fac = 44100, 196_885_100, 0.26875
    g = p64.stretch_geo(T, sr, fac)
    assert g.H + p64.stretch_out_len(T, fac) > (g.H + g.Ls + 3) // 4 * 4  # the case the old sizing missed
    gen = torch.Generator(device=DEV).manual_seed(5)
    xd = 0.3 * torch.randn(1, T, device=DEV, generator=gen)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out, pos = eng.time_stretch(xd, sr, fac, return_positions=True)
    torch.cuda.synchronize()
    print(f"time_stretch of {T} samples at {fac}: {time.perf_counter() - t0:.2f} s")
    n = p64.stretch_out_len(T, fac)
    assert out.shape == (1, n)
    tail = out[0, n - 4096:].cpu().numpy()
    pos = pos[0].cpu().numpy()
    x = xd[0].cpu().numpy()
    s, a, b = p64.ola64(x, pos, g, n - 4096, n)
    p64._held(tail, s, p64.U * (np.abs(a) + np.abs(b)), p64.C_O, "stretch tail", "long row")
    assert np.any(tail != 0)
