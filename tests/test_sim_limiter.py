"""The limiter checks of tests/test_gpu_limiter.py on the CPU-simulated build of the kernels (tests/cusim), at smaller
sizes, and the checks of the float64 oracle itself (tests/limiter64.py): its stages against brute-force restatements,
the bound it promises (no envelope value passes the ceiling), and the overshoot study whose figure DESIGN.md K18
states.  The argument checks of the C entry point and the CPU refusal run against the real library."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import __graft_entry__ as graft
import audiotools_b200.engine as engine_mod
import tests.test_gpu_limiter as G
from audiotools_b200 import _lib
from tests import limiter64 as lim
from tests import truepeak64 as tp
from tests.cusim.sim_engine import sim_engine

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK = lim.CHUNK


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    return sim_engine()


# --------------------------------------------------------------------------- the oracle
def test_oracle_stages_against_brute_force():
    rng = np.random.default_rng(0)
    q = np.maximum(rng.standard_normal((2, 300)), 0)
    for A in (0, 1, 5, 64, 400):
        h = lim.hold(q, A)
        d = lim.release(h, 0.97)
        r = lim.attack(d, A)
        for n in (0, 1, min(A, 299), 150, max(299 - A, 0), 298, 299):
            lo, hi = max(n - A, 0), min(n + A, 299)
            assert (h[:, n] == q[:, lo:hi + 1].max(axis=1)).all()
            assert np.allclose(r[:, n], d[:, lo:hi + 1].mean(axis=1), rtol=0, atol=1e-12)
        want = np.max([0.97 ** (200 - j) * h[:, j] for j in range(201)], axis=0)  # the scan form of the recursion
        assert np.allclose(d[:, 200], want, rtol=1e-12)


def test_oracle_envelope_is_the_true_peak_of_truepeak64():
    x = G.make_batch(48000, 2, 700, seed=1)
    taps = tp.design(4)
    e = lim.envelope(x, taps)
    assert np.allclose(e.max(axis=1), tp.row_peaks(x, taps).max(axis=1), rtol=0, atol=0)
    assert (e >= np.abs(x).max(axis=1)).all()
    assert np.array_equal(lim.envelope(x, np.zeros((0, 12))), np.abs(x.astype(np.float64)).max(axis=1))


def test_oracle_gain_keeps_the_envelope_under_the_ceiling():
    """1 - r[n] <= c / e[n] wherever e[n] > c: every d in the attack window is at least q[n]."""
    sr = 44100
    x = G.make_batch(sr, 2, 5000, seed=2)
    A, a = lim.params(sr)
    taps = tp.design(4)
    c = 10 ** (-1 / 20)
    _, r = lim.limit(x, taps, c, A, a)
    e = lim.envelope(x, taps)
    assert ((1 - r) * e <= c * (1 + 1e-12)).all()
    assert (r[0] == 0).all() and (r[6] == 0).all()


@pytest.mark.parametrize("lookahead,worst", [(0.0015, 0.005), (0.0005, 0.015), (0.003, 0.002)])
def test_oracle_output_overshoot_study(lookahead, worst):
    """True peak of the limited output over the ceiling (the interpolator sees x gain, not gain interp(x)): 44.1 kHz,
    -1 dBTP, release 50 ms, over the test signals.  DESIGN.md K18 states the figures; TP_TOL rests on the default's."""
    sr = 44100
    rows = [tp.faded_sine(sr, f, 0.4, 1.6, seconds=0.2) for f in (0.01, 0.05, 0.11, 0.23, 0.31, 0.45)]
    T = len(rows[0])
    rows += [lim.quarter_rate_sine(T), lim.clipped_sine(T), lim.clicks_on_noise(sr, T / sr, 8, 3) * 3,
             lim.am_noise(sr, T / sr, 4, rate_hz=20.0) * 1.5]
    x = np.stack(rows)[:, None].astype(np.float32)
    out, r = lim.limit_db(x, sr, -1.0, lookahead)
    over = tp.true_peak_db(out, sr) + 1.0
    assert (r.max(axis=1) > 0.05).all()
    assert over.max() <= worst, over
    assert lookahead != 0.0015 or over.max() <= G.TP_TOL / 2, over


# --------------------------------------------------------------------------- the kernels on the simulator
SIM_LENGTHS = (1, 66, 133, CHUNK - 1, CHUNK, CHUNK + 1)


@pytest.mark.parametrize("sr,C", [(16000, 2), (44100, 1), (44100, 5), (48000, 2), (96000, 2), (192000, 1)])
def test_against_float64(eng, sr, C):
    for T in SIM_LENGTHS:
        G.check_against_oracle(eng, sr, C, T, seed=T, inplace=T % 2 == 0)


@pytest.mark.parametrize("A,release", [(0, 0.05), (1, 0.001), (1024, 2.0), (1024, 0.001), (37, 2.0)])
def test_lookaheads_and_releases(eng, A, release):
    for T in sorted({1, max(A, 1), 2 * A + 1, CHUNK + 1, 3 * CHUNK + 17}):
        G.check_against_oracle(eng, 44100, 2, T, A=A, release=release, seed=T + A, per_item=T % 2 == 1,
                               gain=T % 3 == 0, inplace=T % 4 == 1)


def test_gain_ceilings_and_in_place(eng):
    G.check_against_oracle(eng, 48000, 2, CHUNK + 123, release=0.02, gain=True, per_item=True, inplace=True)
    G.check_against_oracle(eng, 96000, 1, CHUNK + 123, release=0.02, gain=True)


def test_a_row_of_70_chunks_at_a_2_s_release(eng):
    """Three batches of the carry kernel's 32-chunk warp scan; a^4096 = 0.95."""
    sr, T = 44100, 70 * CHUNK + 77
    rng = np.random.default_rng(5)
    x = (0.02 * rng.standard_normal((1, 1, T))).astype(np.float32)
    x[0, 0, 5000:5040] = 1.5
    x[0, 0, 40 * CHUNK - 2] = -1.1
    got, want = G.check_against_oracle(eng, sr, 1, T, release=2.0, x=x)
    assert want[0, 30 * CHUNK] > 1e-3 and want[0, -1] > 1e-3


def test_nonfinite_samples(eng):
    G.check_nonfinite(eng, 44100)
    G.check_nonfinite(eng, 192000)


def test_properties(eng):
    G.check_properties(eng)


def test_signal_at_full_level_from_the_first_sample(eng):
    G.check_full_level_start(eng)


def test_the_point_of_the_feature(eng):
    G.check_point_of_the_feature(eng, seconds=2.0)


def test_api(eng):
    G.check_api(eng, sr=16000)


def test_gradient_and_cpu_tensors_are_refused():
    from audiotools_b200 import AudioSignal
    from audiotools_b200.engine import Engine

    graft.build()
    eng = Engine(_lib.B2ALibrary(_lib.LIB_PATH))  # product configuration: require_cuda=True
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        eng.limit(torch.zeros(1, 1, 100), 48000, -1.0)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        AudioSignal(torch.zeros(1, 1, 16000), 16000).limit(-1.0)


def test_bad_arguments_launch_nothing_in_the_real_library():
    graft.build()
    lib = _lib.B2ALibrary(_lib.LIB_PATH)
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    k0 = lib.kernel_launches.value
    assert lib.b2a_limiter_f32(p, None, 1, 1, 16, 3, p, 4, 0.5, p, None, p, None) == -1
    assert lib.b2a_limiter_f32(p, None, 1, 1, 16, 4, p, 1025, 0.5, p, None, p, None) == -1
    assert lib.b2a_limiter_f32(p, None, 1, 1, 16, 4, p, 4, 1.0, p, None, p, None) == -1
    assert lib.b2a_limiter_f32(p, None, 1, 1, 16, 4, p, 4, 0.5, p, None, None, None) == -1
    assert lib.b2a_limiter_f32(p, None, 1, 1, 1 << 62, 4, p, 4, 0.5, p, None, p, None) == -1
    assert lib.kernel_launches.value == k0


_SHUFFLED = r"""
import sys
sys.path.insert(0, sys.argv[1])
import audiotools_b200.engine as em
import tests.test_gpu_limiter as G
from tests.cusim.sim_engine import sim_engine
G.DEV = "cpu"
em._ENGINE = sim_engine()
eng = em._ENGINE
for sr, C, A in ((44100, 2, None), (192000, 1, 1024), (96000, 2, 5)):
    for T in (133, G.CHUNK - 1, 2 * G.CHUNK + 17):
        G.check_against_oracle(eng, sr, C, T, A=A, release=0.02, seed=T, gain=True, inplace=True)
G.check_nonfinite(eng, 48000)
G.check_properties(eng)
print("ok")
"""


def test_limiter_under_shuffled_fiber_order():
    """The simulator visits the CUDA threads of a block in a random order under CUSIM_SHUFFLE: a missing barrier that
    the fixed order happens to satisfy shows up as a wrong result.  (Read once per process: run in a child.)"""
    env = dict(os.environ, CUSIM_SHUFFLE="1")
    r = subprocess.run([sys.executable, "-c", _SHUFFLED, REPO], env=env, cwd=REPO, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
