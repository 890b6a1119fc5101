"""The pitch accuracy checks of tests/test_gpu_pitch_accuracy.py at small shapes on the CPU-simulated build of the
kernels (tests/cusim), with the same module and budgets (tests/pitch64.py), plus the host-only checks: the geometry
mirror, the search's staged region, and the time stretch's workspace at lengths where T r falls short of T / factor.
The simulator's ``sincospif`` / ``cospif`` are evaluated in double and its ``rcp.approx`` is a division, so a check
that fails only on the H100 names one of those instructions."""
import os
import subprocess
import sys

import numpy as np
import pytest

import tests.test_gpu_pitch_accuracy as G
from tests import pitch64 as p64
from tests.cusim.sim_engine import sim_engine

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    return sim_engine()


def sim_length(sr):
    return 6 * p64.Geo(1, sr, 0.0).W + 3


def test_geometry_mirror_and_tiling(eng):
    G.test_geometry_mirror_and_tiling(eng)


def test_global_template_branch_is_unreachable():
    """Every continuation a searched frame can have lies in its staged region at every frame size and at shifts on a
    1/64-semitone grid over [-24, 24]: the search's global-memory template branch cannot be reached by a legal input
    (DESIGN.md "Pitch accuracy").  The kernel tests count the branch on the kernel's own positions and find it unused.
    The region also never reaches its capacity rcap: the clamp to rcap binds nowhere, with at least 48 samples to spare,
    so shortening it by 16 changes no output."""
    least = 1 << 30
    for sr in (1000, 2000, 4000, 8000, 16000, 44100):
        for st in np.arange(-24 * 64, 24 * 64 + 1) / 64.0:
            if st != 0.0:
                g = p64.Geo(10 ** 6, sr, float(st))
                ok, headroom = p64.template_always_staged(g, 64)
                assert ok, (sr, st)
                least = min(least, headroom)
    assert least >= 48, least


@pytest.mark.parametrize("sr", p64.RATES)
def test_pitch_shift_per_splice_and_sample(eng, sr):
    main = sim_length(sr)
    for st in p64.SHIFTS:
        acc = G.check_pitch(eng, sr, st, main, p64.KINDS, seed=int(sr + 100 * st))[0]
        assert acc["searched"] > 0 and acc["fallback"] == 0, (st, acc)
        for T in G.edge_lengths(sr, st, main):
            assert G.check_pitch(eng, sr, st, T, ["noise", "tone+noise"], seed=T)[0]["fallback"] == 0


@pytest.mark.parametrize("sr", [1000, 8000, 16000, 44100])
def test_time_stretch_per_splice_and_sample(eng, sr):
    main = sim_length(sr)
    for st in p64.SHIFTS:
        fac = G.factor_of(st)
        G.check_stretch(eng, sr, fac, main, ["noise", "tone+noise", "nan"], seed=int(sr - st))
        for T in G.edge_lengths(sr, st, main)[::3]:
            G.check_stretch(eng, sr, fac, T, ["noise"], seed=T)


def test_stretched_row_past_the_last_frame(eng):
    G.check_past_last_frame(eng)


@pytest.mark.parametrize("sr", [1000, 8000])
def test_multi_shift_launch(eng, sr):
    G.check_multi(eng, sr, sim_length(sr) + 2)


@pytest.mark.parametrize("sr,st,rows", [(1000, 24.0, (1, 7, 300)), (8000, -7.0, (1, 7)), (16000, 0.5, (7,))])
def test_exact_invariances(eng, sr, st, rows):
    G.check_exact(eng, sr, st, sim_length(sr) + 1, rows)


# T, factor: T r falls short of T / factor by more than the rate change's half + 2 samples of slack
SHORT_STRETCH = [(196_345_837, 0.277), (196_885_100, 0.26875), (268_435_455, 0.26875)]


def _stretch_sizes(lib, T, sr, fac):
    g = p64.stretch_geo(T, sr, fac)
    ws = lib.b2a_time_stretch_workspace_bytes(1, T, sr, fac)
    n = lib.b2a_time_stretch_out_len(T, fac)
    return g, ws, n


@pytest.mark.parametrize("T,fac", SHORT_STRETCH)
def test_time_stretch_workspace_covers_the_output(eng, T, fac):
    """The workspace the library asks for holds the whole output, round(T / factor) samples past the halo, where the
    rate change's own length ceil(T r) + half + 2 does not."""
    for sr in (16000, 44100):
        g, ws, n = _stretch_sizes(eng.lib, T, sr, fac)
        assert n == p64.stretch_out_len(T, fac)
        assert g.H + n > (g.H + g.Ls + 3) // 4 * 4, "not a case the rate change's length misses"
        assert ws == p64.workspace_bytes(1, [g]) and g.H + n <= g.SL, (T, fac, sr)


def test_time_stretch_workspace_on_a_factor_grid(eng):
    """Every factor on a 1/4000 grid over [0.25, 4] at the longest accepted row: the stretched row covers the output."""
    T, sr, short = (1 << 28) - 1, 44100, 0
    for i in range(1000, 16001):
        fac = i / 4000.0
        g, ws, n = _stretch_sizes(eng.lib, T, sr, fac)
        short += g.H + n > (g.H + g.Ls + 3) // 4 * 4
        assert ws == p64.workspace_bytes(1, [g]) and g.H + n <= g.SL, fac
    assert short > 0


_SHUFFLED = r"""
import sys
sys.path.insert(0, sys.argv[1])
import tests.test_gpu_pitch_accuracy as G
from tests import pitch64 as p64
from tests.cusim.sim_engine import sim_engine
G.DEV = "cpu"
eng = sim_engine()
for sr, st in ((1000, 24.0), (4000, -0.5), (16000, 7.0), (44100, -12.0)):
    T = 4 * p64.Geo(1, sr, 0.0).W + 1
    acc = G.check_pitch(eng, sr, st, T, ["noise", "tone+noise", "dc"], seed=3)[0]
    assert acc["searched"] > 0
    G.check_stretch(eng, sr, G.factor_of(st), T, ["noise"], seed=4)
G.check_multi(eng, 1000, 6 * 64 + 2, reps=1)
print("ok")
"""


def test_pitch_under_shuffled_fiber_order():
    """The simulator visits the CUDA threads of a block in a random order under CUSIM_SHUFFLE: a missing barrier that
    the fixed order happens to satisfy shows up as a wrong result (the search has four barriers per frame and a
    double-buffered previous position).  (Read once per process: run in a child.)"""
    env = dict(os.environ, CUSIM_SHUFFLE="1")
    r = subprocess.run([sys.executable, "-c", _SHUFFLED, REPO], env=env, cwd=REPO, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
