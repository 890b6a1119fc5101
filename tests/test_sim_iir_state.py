"""The checks of tests/test_gpu_iir_state.py on the CPU-simulated build of the kernels (tests/cusim), at smaller
sizes, the float32 baseline of tests/iirfilt64.py against scipy, and the argument checks of the new C entry points
against the real library."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy import signal as sps

import __graft_entry__ as graft
import audiotools_b200.engine as engine_mod
import tests.test_gpu_iir as GI
import tests.test_gpu_iir_state as G
from audiotools_b200 import _lib
from tests import iir64, iirfilt64
from tests.cusim.sim_engine import sim_engine

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK = G.CHUNK


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(GI, "DEV", "cpu")
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    return sim_engine()


# --------------------------------------------------------------------------- the oracle
@pytest.mark.parametrize("padtype", G.PADTYPES)
def test_baseline_follows_scipy(padtype):
    """The float32 restatement of sosfiltfilt's steps is scipy's own call when run in float64."""
    rng = np.random.default_rng(0)
    x = rng.standard_normal((2, 2, 300)).astype(np.float32)
    sos = np.stack([sps.butter(3, 0.1, output="sos"), sps.cheby1(3, 1.0, 0.3, "highpass", output="sos")])
    s32 = iir64.coefficients(sos, 2)
    base = iirfilt64.baseline_filtfilt(x, s32, padtype=padtype)
    ref = iirfilt64.reference_filtfilt(x, s32, padtype=padtype)
    assert np.abs(base - ref).max() <= 1e-4 * np.abs(ref).max()
    assert (iirfilt64.default_padlen(s32) == 3 * (2 * 2 + 1 - 1)).all()
    for n in (0, 1, 7):
        got = iirfilt64._extend(x.astype(np.float64), padtype, n)
        if padtype is not None and n > 0:
            want = {"odd": sps._arraytools.odd_ext, "even": sps._arraytools.even_ext,
                    "constant": sps._arraytools.const_ext}[padtype](x.astype(np.float64), n, axis=-1)
            assert np.array_equal(got, want)


# --------------------------------------------------------------------------- the kernels on the simulator
@pytest.mark.parametrize("S", [1, 2, 3, 5, 8])
def test_zero_phase_against_float64(eng, S):
    edge = 3 * (2 * S + 1)
    for i, T in enumerate((edge + 1, CHUNK - 1, CHUNK + 1, 3 * CHUNK + 17)):
        G.check_filtfilt(eng, 48000, 2, T, S, per_item=i % 2 == 1, seed=10 * S + i, gain=i % 3 == 0,
                         padtype=G.PADTYPES[(i + S) % 4], padlen=None if i == 0 else (None, 0, 30)[(i + S) % 3])


def test_thirty_three_chunks(eng):
    """The carry kernel's 32-chunk warp scan, forwards and backwards, with a 20 Hz Q 8 +12 dB peak."""
    sr = 48000
    sos = np.concatenate([sps.butter(3, 30.0, "highpass", fs=sr, output="sos"),
                          iir64.cookbook("peaking", 20.0, 12.0, 8.0, sr)[None]])[None]
    rng = np.random.default_rng(9)
    x = np.stack([GI.make_signal(s, rng, sr, 1, 32 * CHUNK + 1) for s in ("noise", "low_tone")])
    G.check_filtfilt(eng, sr, 1, x.shape[-1], 3, x=x, sos=sos)


@pytest.mark.parametrize("S", [1, 4, 8])
def test_streaming(eng, S):
    G.check_streaming(eng, 48000, 2, 3 * CHUNK + 7, S, seed=S,
                      cuts=[1, 2, 3, 500, CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK + 40])


def test_zero_state_equals_sos_filter(eng):
    G.check_zero_state_equals_sos_filter(eng, T=CHUNK + 9)


def test_properties(eng):
    G.check_properties(eng, T=2 * CHUNK + 77)


def test_gradient(eng):
    G.check_gradient(eng, T=150)


def test_api(eng):
    G.check_api(eng)


def test_cpu_tensors_are_refused():
    from audiotools_b200 import AudioSignal
    from audiotools_b200.engine import Engine

    graft.build()
    eng = Engine(_lib.B2ALibrary(_lib.LIB_PATH))  # product configuration: require_cuda=True
    ident = np.array([[1.0, 0, 0, 1, 0, 0]])
    x = torch.zeros(1, 1, 100)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        eng.sos_filtfilt(x, ident)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        eng.sos_filtfilt_backward(x, ident)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        eng.sos_filter_zi(x, ident, np.zeros((1, 1, 1, 2)))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        AudioSignal(torch.zeros(1, 1, 16000), 16000).sos_filter(ident, zero_phase=True)


def test_bad_arguments_launch_nothing_in_the_real_library():
    graft.build()
    lib = _lib.B2ALibrary(_lib.LIB_PATH)
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    k0 = lib.kernel_launches.value
    assert lib.b2a_sos_filter_zi_f32(p, None, 1, 1, 16, p, 1, 9, p, p, None, p, None) == -1
    assert lib.b2a_sos_filter_zi_f32(p, None, 1, 1, 16, p, 1, 1, None, p, None, p, None) == -1
    assert lib.b2a_sos_filtfilt_f32(p, None, 1, 1, 16, p, 1, 1, 7, -1, p, p, None) == -1
    assert lib.b2a_sos_filtfilt_f32(p, None, 1, 1, 16, p, 1, 1, 1, 16, p, p, None) == -1
    assert lib.b2a_sos_filtfilt_backward_f32(p, None, 1, 1, 9, p, 1, 1, 1, -1, p, p, None) == -1
    assert lib.b2a_sos_filtfilt_workspace_bytes(1, 1, 9, 1, 1, -1) == 0
    assert lib.b2a_sos_filtfilt_workspace_bytes(1, 1, 10, 1, 1, -1) > 0
    assert lib.kernel_launches.value == k0


_SHUFFLED = r"""
import sys
sys.path.insert(0, sys.argv[1])
import audiotools_b200.engine as em
import tests.test_gpu_iir as GI
import tests.test_gpu_iir_state as G
from tests.cusim.sim_engine import sim_engine
G.DEV = GI.DEV = "cpu"
em._ENGINE = sim_engine()
eng = em._ENGINE
for S, T, pt in ((1, 700, "odd"), (3, G.CHUNK + 1, "even"), (8, 2 * G.CHUNK + 17, "constant")):
    G.check_filtfilt(eng, 48000, 2, T, S, per_item=True, seed=T, gain=True, padtype=pt)
G.check_streaming(eng, 48000, 1, 2 * G.CHUNK + 5, 4, seed=1, cuts=[1, 700, G.CHUNK + 1])
G.check_gradient(eng, T=120)
print("ok")
"""


def test_iir_state_under_shuffled_fiber_order():
    """The simulator visits the CUDA threads of a block in a random order under CUSIM_SHUFFLE: a missing warp barrier
    that the fixed order happens to satisfy shows up as a wrong result.  (Read once per process: run in a child.)"""
    env = dict(os.environ, CUSIM_SHUFFLE="1")
    r = subprocess.run([sys.executable, "-c", _SHUFFLED, REPO], env=env, cwd=REPO, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
