"""The true-peak checks of tests/test_gpu_true_peak.py on the CPU-simulated build of the kernels (tests/cusim), and
the checks of the float64 oracle itself (tests/truepeak64.py): the library's taps are the double design rounded to
float, phase 0 is the sample, and the interpolator's error on faded steady sines stays within the documented range.
The argument checks of the C entry points and the CPU refusal run against the real library."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import __graft_entry__ as graft
import audiotools_b200.engine as engine_mod
import tests.test_gpu_true_peak as G
from audiotools_b200 import _lib
from tests import truepeak64 as tp
from tests.cusim.sim_engine import sim_engine

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RATES = [16000, 22050, 44100, 48000, 96000, 192000]


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    return sim_engine()


# --------------------------------------------------------------------------- the oracle and the taps
@pytest.mark.parametrize("sr", RATES)
def test_factor(sr):
    lib = _lib.get_lib()
    assert lib.b2a_true_peak_factor(float(sr)) == tp.factor(sr)


def test_factor_edges_and_bad_rates():
    lib = _lib.get_lib()
    assert [lib.b2a_true_peak_factor(r) for r in (8000.0, 95999.0, 96000.0, 191999.0, 192000.0, 384000.0)] == \
        [4, 4, 2, 2, 1, 1]
    for r in (0.0, -44100.0, float("nan"), float("inf")):
        assert lib.b2a_true_peak_factor(r) == -1


@pytest.mark.parametrize("L", [2, 4])
def test_taps_are_the_float64_design_rounded(L):
    lib = _lib.get_lib()
    got = np.zeros((L - 1, 12), np.float32)
    assert lib.b2a_true_peak_taps(L, got.ctypes.data_as(ctypes.c_void_p)) == 0
    want = tp.design(L)
    ulp = np.spacing(np.abs(want).astype(np.float32))
    assert (np.abs(got.astype(np.float64) - want) <= ulp).all()
    # no renormalisation: the phase sums are those of the windowed sinc
    sums = want.sum(axis=1)
    if L == 4:
        assert np.allclose(sums, [1.00048, 1.00090, 1.00048], atol=1e-5)
        assert np.array_equal(got[0], got[2][::-1])  # phase 3 mirrors phase 1
    else:
        assert np.allclose(sums, [1.00090], atol=1e-5)
    assert lib.b2a_true_peak_taps(1, None) == 0
    assert lib.b2a_true_peak_taps(3, got.ctypes.data_as(ctypes.c_void_p)) == -1
    assert lib.b2a_true_peak_taps(4, None) == -1


def test_phase_zero_is_the_sample():
    """With every interpolated phase removed the oracle's peak is max |x|; with them it is never below."""
    x = np.random.default_rng(0).standard_normal((6, 500))
    assert np.array_equal(tp.row_peaks(x, np.zeros((0, 12))), np.abs(x).max(axis=1))
    assert (tp.row_peaks(x, tp.design(4)) >= np.abs(x).max(axis=1)).all()


@pytest.mark.parametrize("sr,lo,hi", [(44100, -0.45, 0.15), (48000, -0.45, 0.15), (96000, -0.75, 0.15)])
def test_sine_error_range(sr, lo, hi):
    """Steady sines with 50 ms raised-cosine fades, 0.005 .. 0.45 fs, 40 random phases each: dBTP - 20 log10(amp)."""
    rng = np.random.default_rng(1)
    errs = []
    for f in np.linspace(0.005, 0.45, 46):
        amp = 10 ** rng.uniform(-2, 0)
        x = np.stack([tp.faded_sine(sr, f, ph, amp, seconds=0.15) for ph in rng.uniform(0, 2 * np.pi, 40)])
        errs.append(tp.true_peak_db(x[:, None], sr) - 20 * np.log10(amp))
    errs = np.concatenate(errs)
    assert lo <= errs.min() and errs.max() <= hi, (errs.min(), errs.max())


def test_quarter_rate_sine_at_45_degrees():
    x = tp.faded_sine(48000, 0.25, np.pi / 4)
    mid = x[2400:-2400]
    assert abs(20 * np.log10(np.abs(mid).max()) + 3.0103) < 1e-3  # sample peak -3.01 dB
    assert abs(tp.true_peak_db(x[None, None], 48000)[0]) < 0.05


def test_clipped_sine_reads_above_plus_2():
    n = np.arange(12000)
    x = np.clip(1.5 * np.sin(2 * np.pi * 0.21 * n + 0.3), -1, 1)
    assert np.abs(x).max() == 1.0
    assert tp.true_peak_db(x[None, None], 48000)[0] > 2.0


# --------------------------------------------------------------------------- the kernel on the simulator
@pytest.mark.parametrize("C", [1, 2, 5])
@pytest.mark.parametrize("sr", RATES)
def test_against_float64(eng, sr, C):
    for T in G.LENGTHS:
        G.check_against_oracle(eng, sr, C, T, seed=T)


def test_long_rows_against_float64(eng):
    G.check_against_oracle(eng, 44100, 2, 3 * G.CHUNK + 123)


@pytest.mark.parametrize("sr", [16000, 44100, 96000, 192000])
def test_nonfinite_rows(eng, sr):
    G.check_nonfinite(eng, sr)


@pytest.mark.parametrize("sr", [44100, 96000, 192000])
def test_exactness(eng, sr):
    G.check_exact(eng, sr)


def test_launches_and_rejected_calls(eng):
    G.check_launches(eng)


def test_api(eng):
    G.check_api(eng)


def test_volume_norm_partial_mask(eng):
    G.check_volume_norm_mask()


def test_gradient_and_cpu_tensors_are_refused():
    from audiotools_b200 import AudioSignal
    from audiotools_b200.engine import Engine

    graft.build()
    eng = Engine(_lib.B2ALibrary(_lib.LIB_PATH))  # product configuration: require_cuda=True
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        eng.true_peak(torch.zeros(1, 1, 100), 48000)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        AudioSignal(torch.zeros(1, 1, 16000), 16000).true_peak()
    with pytest.raises(NotImplementedError, match="true_peak"):
        sim_engine().true_peak(torch.zeros(1, 1, 100, requires_grad=True), 48000)
    with pytest.raises(_lib.B2AError, match="bad sample rate"):
        sim_engine().true_peak(torch.zeros(1, 1, 100), 0)


def test_bad_arguments_launch_nothing_in_the_real_library():
    graft.build()
    lib = _lib.B2ALibrary(_lib.LIB_PATH)
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    k0 = lib.kernel_launches.value
    assert lib.b2a_true_peak_f32(p, 1, 1, 16, 3, p, None, None) == -1
    assert lib.b2a_true_peak_f32(p, 1, 0, 16, 4, p, None, None) == -1
    assert lib.b2a_true_peak_f32(p, 1, 1, 16, 4, None, None, None) == -1
    assert lib.kernel_launches.value == k0


_SHUFFLED = r"""
import sys
sys.path.insert(0, sys.argv[1])
import audiotools_b200.engine as em
import tests.test_gpu_true_peak as G
from tests.cusim.sim_engine import sim_engine
G.DEV = "cpu"
em._ENGINE = sim_engine()
eng = em._ENGINE
for sr in (44100, 96000, 192000):
    for T in G.LENGTHS:
        G.check_against_oracle(eng, sr, 2, T, seed=T)
G.check_nonfinite(eng, 48000)
G.check_exact(eng, 48000)
print("ok")
"""


def test_true_peak_under_shuffled_fiber_order():
    """The simulator visits the CUDA threads of a block in a random order under CUSIM_SHUFFLE: a missing barrier that
    the fixed order happens to satisfy shows up as a wrong result.  (Read once per process: run in a child.)"""
    env = dict(os.environ, CUSIM_SHUFFLE="1")
    r = subprocess.run([sys.executable, "-c", _SHUFFLED, REPO], env=env, cwd=REPO, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
