"""The diffuse-tail checks of tests/test_gpu_rir_diffuse.py on the CPU-simulated build of the kernels (tests/cusim), at
8 kHz and small sizes, also under a shuffled thread order; the oracle of tests/rir_diffuse64.py against known answers
and against the images it stands for; and the argument checks of the C entry point against the real library."""
import ctypes
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import __graft_entry__ as graft
import audiotools_b200.engine as engine_mod
import tests.test_gpu_rir_diffuse as G
from audiotools_b200 import _lib
from tests import rir64
from tests import rir_diffuse64 as D
from tests.cusim.sim_engine import sim_engine

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FS = 8000


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    return sim_engine()


# --------------------------------------------------------------------------- the oracle
def test_envelope_is_converged_and_flat_without_absorption():
    room, fs = [6.0, 5.0, 3.0], 16000
    n = np.array([0, 1, 10, 100, 1000, 4000, 16000, 48000])
    for beta in ([0.95, 0.95, 0.9, 0.9, 0.6, 0.8], [0.3, 0.99, 0.5, 0.5, 0.01, 0.9], np.full(6, 0.7)):
        e, e2 = D.envelope(room, beta, fs, n), D.envelope(room, beta, fs, n, K=128)
        live = e2 >= 1e-9 * 343.0 / (4 * math.pi * 90.0 * fs)
        assert np.all(np.abs(e[live] / e2[live] - 1) < 1e-8), beta
    flat = 343.0 / (4 * math.pi * 90.0 * fs)
    assert np.allclose(D.envelope(room, np.ones(6), fs, n), flat, rtol=1e-12, atol=0)
    assert (D.envelope(room, [0.9, 0.9, 0.0, 0.9, 0.9, 0.9], fs, n) == 0).all()
    # equal absorption on every axis: (1/4pi) int exp(-a |u|_1) dOmega at n = 0 is 1
    assert abs(D.direction_mean(np.full(3, 0.01), [0.0])[0] - 1) < 1e-12


def test_envelope_matches_the_images():
    """The energy of the images (sum of g^2) in 10 ms windows from 20 ms on against the envelope: median within
    1 dB per room, equal and unequal walls."""
    fs, L, w = 16000, 4000, 160
    for room, src, mic, beta in (([5.0, 4.0, 3.0], [1.0, 1.0, 1.5], [3.0, 2.5, 1.2], np.full(6, 0.9)),
                                 ([6.0, 5.0, 3.0], [1.0, 1.0, 1.5], [4.0, 3.0, 1.2],
                                  [0.95, 0.95, 0.9, 0.9, 0.6, 0.8])):
        d, g, _ = rir64.images(room, src, mic, beta, fs, L)
        got = np.bincount((d // w).astype(np.int64), weights=g ** 2, minlength=L // w)[:L // w]
        want = np.array([D.envelope(room, beta, fs, np.arange(k * w, (k + 1) * w) + 0.5).sum()
                         for k in range(L // w)])
        diff = 10 * np.log10(got[2:] / want[2:])
        assert abs(float(np.median(diff))) < 1.0, (room, diff)


def test_generator_stream():
    """The numpy generator: 1e7 samples over 10 seeds x 10 microphones; keys differ per seed and microphone."""
    n = np.arange(100_000)
    x = np.stack([np.stack([D.xi(s, c, n)[0] for c in range(10)]) for s in range(10)])
    N = x.size
    m, v = x.mean(), x.var()
    assert abs(m) < 5 / math.sqrt(N) and abs(v - 1) < 5 * math.sqrt(2 / N)
    assert abs(((x - m) ** 4).mean() / v ** 2 - 3) < 5 * math.sqrt(24 / N)
    rho = lambda a, b: float(np.corrcoef(a.reshape(-1), b.reshape(-1))[0, 1])  # noqa: E731
    assert abs(rho(x[..., 1:], x[..., :-1])) < 5 / math.sqrt(N)
    assert abs(rho(x[:, 1:], x[:, :-1])) < 5 / math.sqrt(N)
    assert abs(rho(x[1:], x[:-1])) < 5 / math.sqrt(N)
    # the SplitMix64 finaliser's published first output for state 0 advanced once
    assert int(D._mix(np.uint64(D.GAMMA))) == 0xE220A8397B1DCDAF
    assert D.xi_bits(1, 0, 5) != D.xi_bits(1, 1, 5) != D.xi_bits(2, 0, 5)


def test_ramp_is_complementary():
    Tw, n_d = 64, 1000
    n = np.arange(n_d - Tw // 2, n_d + Tw // 2)
    w2 = D.ramp(n, n_d, Tw) ** 2
    assert np.allclose(w2 + w2[::-1], 1.0, rtol=0, atol=1e-15)
    assert D.ramp([n_d + Tw // 2], n_d, Tw)[0] == 1.0


# --------------------------------------------------------------------------- the kernels on the simulator
def test_unchanged_path(eng):
    G.check_unchanged(eng, fs=FS, L=1600)


def test_against_float64(eng):
    G.check_tail(eng, FS, 1600, seed=1)


def test_generator(eng):
    G.check_generator(eng, B=3, C=3, L=20_000)


def test_api(eng):
    G.check_api(eng)


def test_bad_arguments_launch_nothing_in_the_real_library():
    graft.build()
    lib = _lib.B2ALibrary(_lib.LIB_PATH)
    buf = (ctypes.c_double * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    k0 = lib.kernel_launches.value
    assert lib.b2a_rir_f32(p, p, p, p, None, None, p, 1, 1, 1, 16, 8000.0, 343.0, -1, p, None) == -1
    assert lib.b2a_rir_f32(p, p, p, p, None, p, None, 1, 1, 1, 16, 8000.0, 343.0, -1, p, None) == -1
    assert lib.b2a_rir_f32(p, p, p, p, None, p, p, 1, 1, 1, 16, 124.0, 343.0, -1, p, None) == -1
    assert lib.b2a_rir_f32(p, p, p, p, None, p, p, 65536, 1, 1, 16, 8000.0, 343.0, -1, p, None) == -1
    assert lib.kernel_launches.value == k0


_SHUFFLED = r"""
import sys
sys.path.insert(0, sys.argv[1])
import audiotools_b200.engine as em
import tests.test_gpu_rir_diffuse as G
from tests.cusim.sim_engine import sim_engine
G.DEV = "cpu"
em._ENGINE = sim_engine()
eng = em._ENGINE
G.check_unchanged(eng, fs=8000, L=1600)
G.check_tail(eng, 8000, 1300, seed=2)
print("ok")
"""


def test_rir_diffuse_under_shuffled_fiber_order():
    """The simulator visits the CUDA threads of a block in a random order under CUSIM_SHUFFLE: a missing barrier
    around the envelope's nodes shows up as a wrong result.  (Read once per process: run in a child.)"""
    env = dict(os.environ, CUSIM_SHUFFLE="1")
    r = subprocess.run([sys.executable, "-c", _SHUFFLED, REPO], env=env, cwd=REPO, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
