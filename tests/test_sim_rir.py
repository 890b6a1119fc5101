"""The image-source checks of tests/test_gpu_rir.py on the CPU-simulated build of the kernels (tests/cusim), at 8 kHz
and at most ~1500 samples, also under a shuffled thread order; the oracle of tests/rir64.py against known answers;
and the argument checks of the C entry point against the real library."""
import ctypes
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import __graft_entry__ as graft
import audiotools_b200.engine as engine_mod
import tests.test_gpu_rir as G
from audiotools_b200 import _lib
from tests import rir64
from tests.cusim.sim_engine import sim_engine

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FS = 8000


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    return sim_engine()


# --------------------------------------------------------------------------- the oracle
def test_oracle_direct_path_and_window():
    """One image: the taps peak at d, sum to about 1 (a windowed sinc), and Tw rounds halves up."""
    assert [rir64.window(f) for f in (124, 125, 8000, 44100, 96000)] == [0, 2, 64, 352, 768]
    d, g, o = rir64.images([5.0, 4.0, 3.0], [1.0, 1.0, 1.5], [3.0, 2.5, 1.2], np.zeros(6), FS, 1000)
    assert (g[o > 0] == 0).all()
    d, g, o = d[o == 0], g[o == 0], o[o == 0]
    assert len(d) == 1
    dist = math.sqrt(4 + 2.25 + 0.09)
    assert abs(d[0] - dist * FS / 343.0) < 1e-12 and abs(g[0] - 1 / (4 * math.pi * dist)) < 1e-15
    y = rir64.render(d, g, rir64.window(FS), 1000)
    assert abs(int(np.argmax(y)) - d[0]) <= 0.5 and abs(y.sum() / g[0] - 1) < 1e-2


def test_oracle_counts_the_issue_rooms():
    """The image counts of the probe's first room (max_order = 20 leaves 11,521)."""
    d, _, o = rir64.images([5.0, 4.0, 3.0], [1.0, 1.0, 1.5], [3.0, 2.5, 1.2], np.full(6, 0.9), 16000, 8000)
    assert len(d) == 352121
    assert int((o <= 20).sum()) == 11521


def test_highpass_matches_the_sequential_recursion():
    """Allen & Berkley's published recursion (w[n] = x[n] + 2 R cos(W) w[n-1] - R^2 w[n-2], y[n] = w[n] - (1 + R)
    w[n-1] + R w[n-2]) equals the one section of ``highpass_sos`` to 1e-11 of the peak in float64 (the poles
    near z = 1 amplify the two realisations' rounding differently)."""
    from scipy import signal as sps

    for fs in (8000, 16000, 48000, 96000):
        W = 2 * math.pi * 100 / fs
        R = math.exp(-W)
        x = np.random.default_rng(0).standard_normal(4000)
        y = np.zeros_like(x)
        w1 = w2 = 0.0
        for n in range(len(x)):
            w0 = x[n] + 2 * R * math.cos(W) * w1 - R * R * w2
            y[n] = w0 - (1 + R) * w1 + R * w2
            w2, w1 = w1, w0
        assert np.abs(sps.sosfilt(rir64.highpass_sos(fs), x) - y).max() < 1e-11 * np.abs(y).max()


# --------------------------------------------------------------------------- the kernel on the simulator
@pytest.mark.parametrize("L", [1, 40, 63, 511, 512, 513, 1500])
def test_against_float64(eng, L):
    G.check_accuracy(eng, FS, L, 2, list(G.ROOMS), ["corner", "near", "random", "random", "near"],
                     ["per", "one", "zero", "per", "per"], max_order=(-1, 10, 2)[L % 3], seed=L)


@pytest.mark.parametrize("max_order", [-1, 0, 1, 2, 10])
def test_orders_and_channels(eng, max_order):
    for C in (1, 2, 8):
        G.check_accuracy(eng, FS, 700, C, [G.ROOMS[1], G.ROOMS[4]], ["random", "near"], ["per", "one"], max_order,
                         seed=max_order + C)


def test_high_pass(eng):
    G.check_highpass(eng, fs=FS, L=1500)


def test_properties(eng):
    G.check_properties(eng)


def test_api(eng):
    G.check_api(eng)


def test_cpu_tensors_are_refused(monkeypatch):
    from audiotools_b200.core.room import image_source_ir
    from audiotools_b200.engine import Engine

    graft.build()
    monkeypatch.setattr(engine_mod, "_ENGINE", Engine(_lib.B2ALibrary(_lib.LIB_PATH)))  # require_cuda=True
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        image_source_ir([4.0, 3.0, 2.5], [1.0, 1.0, 1.0], [[2.0, 2.0, 1.5]], FS, 100, rt60=0.3, device="cpu")


def test_bad_arguments_launch_nothing_in_the_real_library():
    graft.build()
    lib = _lib.B2ALibrary(_lib.LIB_PATH)
    buf = (ctypes.c_double * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    k0 = lib.kernel_launches.value
    assert lib.b2a_rir_f32(p, p, p, None, None, None, None, 1, 1, 1, 16, 8000.0, 343.0, -1, p, None) == -1
    assert lib.b2a_rir_f32(p, p, p, p, None, None, None, 1, 1, 1, 16, 124.0, 343.0, -1, p, None) == -1
    assert lib.b2a_rir_f32(p, p, p, p, None, None, None, 1, 1, 1, 16, 8000.0, -1.0, -1, p, None) == -1
    assert lib.b2a_rir_f32(p, p, p, p, None, None, None, 65536, 1, 1, 16, 8000.0, 343.0, -1, p, None) == -1
    assert lib.kernel_launches.value == k0


_SHUFFLED = r"""
import sys
sys.path.insert(0, sys.argv[1])
import audiotools_b200.engine as em
import tests.test_gpu_rir as G
from tests.cusim.sim_engine import sim_engine
G.DEV = "cpu"
em._ENGINE = sim_engine()
eng = em._ENGINE
for L, mo in ((513, -1), (1500, 10)):
    G.check_accuracy(eng, 8000, L, 2, list(G.ROOMS), ["corner", "near", "random", "random", "near"],
                     ["per", "one", "zero", "per", "per"], max_order=mo, seed=L)
G.check_properties(eng)
print("ok")
"""


def test_rir_under_shuffled_fiber_order():
    """The simulator visits the CUDA threads of a block in a random order under CUSIM_SHUFFLE: a missing barrier
    around the staged images shows up as a wrong result.  (Read once per process: run in a child.)"""
    env = dict(os.environ, CUSIM_SHUFFLE="1")
    r = subprocess.run([sys.executable, "-c", _SHUFFLED, REPO], env=env, cwd=REPO, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
