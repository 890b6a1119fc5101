"""The octave-band checks of tests/test_gpu_rir_bands.py on the CPU-simulated build of the kernels (tests/cusim), at
small sizes, also under a shuffled thread order; and the argument checks of the C entry points against the real
library."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import __graft_entry__ as graft
import audiotools_b200.engine as engine_mod
import tests.test_gpu_rir_bands as G
from audiotools_b200 import _lib
from tests import rir_bands64 as R64
from tests.cusim.sim_engine import sim_engine

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FS = 8000


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    return sim_engine()


# --------------------------------------------------------------------------- the oracle
def test_oracle_definitions():
    assert [R64.kept(8, fs) for fs in (300, 8000, 16000, 22050, 44100, 96000)] == [1, 6, 7, 7, 8, 8]
    assert R64.half0(48000) == int(8 / (125 * 2 ** 0.5 / 48000) / 2)
    lp = R64.lowpass64(16000, 6)
    assert np.allclose(lp.sum(1), 1.0, rtol=0, atol=1e-13) and np.allclose(lp, lp[:, ::-1], rtol=0, atol=1e-15)
    # equal bands: every difference is 0 and the combination is the last band
    r = np.tile(np.random.default_rng(0).standard_normal(300), (4, 1))
    assert np.array_equal(R64.combine(r, lp[:3]), r[-1])


def test_crossover_taps_against_float64(eng):
    for fs in (8000, 16000, 48000):
        kept = R64.kept(8, fs)
        err = float(np.abs(G.crossover_taps(eng, fs, kept) - R64.lowpass64(fs, kept - 1)).max())
        assert err <= 64 * R64.U * float(np.abs(R64.lowpass64(fs, kept - 1)).max()), (fs, err)


# --------------------------------------------------------------------------- the kernels on the simulator
def test_unchanged_path(eng):
    G.check_unchanged(eng, rates=(FS, 16000), L=700)


def test_against_float64(eng):
    h = R64.half0(FS)
    for L in (G.TILE - 1, G.TILE + 1, 2 * h + 5):
        G.check_bands(eng, FS, L, kinds=("per", "mixed", "zero", "one"), seed=L)
    G.check_bands(eng, FS, 700, K=3, C=1, kinds=("per", "one"), air_on=False, seed=1)
    G.check_bands(eng, FS, 900, K=8, C=2, kinds=("per", "mixed"), td=0.01, seed=2)
    for max_order in (0, 2):
        G.check_bands(eng, 16000, 600, K=4, C=2, kinds=("per",), max_order=max_order, seed=3)


def test_bands_above_nyquist(eng):
    G.check_nyquist(eng, L=700)


def test_air_absorption(eng):
    G.check_air(eng, fs=16000, L=2048)


def test_api(eng):
    G.check_api(eng)


def test_launch_counts(eng):
    G.check_launches(eng)


def test_bad_arguments_launch_nothing_in_the_real_library():
    graft.build()
    lib = _lib.B2ALibrary(_lib.LIB_PATH)
    buf = (ctypes.c_double * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    k0 = lib.kernel_launches.value
    assert lib.b2a_rir_bands_kept(8, 8000.0) == 6 and lib.b2a_rir_bands_kept(9, 8000.0) == 0
    assert lib.b2a_rir_f32(p, p, p, p, None, None, None, 1, 1, 9, 16, 8000.0, 343.0, -1, p, None) == -1
    assert lib.b2a_rir_f32(p, p, p, p, None, p, None, 1, 1, 3, 16, 8000.0, 343.0, -1, p, None) == -1
    assert lib.b2a_rir_f32(p, p, p, p, None, None, None, 21846, 1, 3, 16, 8000.0, 343.0, -1, p, None) == -1
    assert lib.b2a_rir_band_sum_f32(p, p, None, 1, 1, 16, 8000.0, 343.0, 5, p, p, 8, p, None) == -1
    assert lib.kernel_launches.value == k0


_SHUFFLED = r"""
import sys
sys.path.insert(0, sys.argv[1])
import audiotools_b200.engine as em
import tests.test_gpu_rir_bands as G
from tests.cusim.sim_engine import sim_engine
G.DEV = "cpu"
em._ENGINE = sim_engine()
eng = em._ENGINE
G.check_unchanged(eng, rates=(8000,), L=700)
G.check_bands(eng, 8000, 700, K=8, C=2, kinds=("per", "mixed"), td=0.01, seed=4)
print("ok")
"""


def test_rir_bands_under_shuffled_fiber_order():
    """The simulator visits the CUDA threads of a block in a random order under CUSIM_SHUFFLE: a missing barrier
    around the staged band gains or the per-band envelope nodes shows up as a wrong result.  (Read once per process:
    run in a child.)"""
    env = dict(os.environ, CUSIM_SHUFFLE="1")
    r = subprocess.run([sys.executable, "-c", _SHUFFLED, REPO], env=env, cwd=REPO, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr


def test_decay_follows_the_bands(eng):
    G.check_decay(eng, fs=8000, L=7200, M=2)
