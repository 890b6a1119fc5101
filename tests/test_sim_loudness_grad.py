"""The checks of tests/test_gpu_loudness_grad.py on the CPU-simulated build of the kernels (tests/cusim), at smaller
sizes; the float64 oracle (tests/loudness_grad64.py) against central finite differences of its own loudness; and the
argument checks of b2a_lufs_backward_f32 against the real library."""
import ctypes

import numpy as np
import pytest

import __graft_entry__ as graft
import audiotools_b200.engine as engine_mod
import tests.test_gpu_loudness_grad as G
from audiotools_b200 import _lib
from tests import loudness_grad64 as lg
from tests.cusim.sim_engine import sim_engine


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    return sim_engine()


@pytest.mark.parametrize("rate", G.RATES)
@pytest.mark.parametrize("C", [1, 2, 5])
def test_gradient_against_float64(eng, rate, C):
    G.check_accuracy(rate, C, int(0.9 * rate) + 77)


@pytest.mark.parametrize("rate", G.RATES)
def test_short_rows_are_zero_extended(eng, rate):
    G.check_accuracy(rate, 2, int(0.3 * rate) + 5)


def test_tail_under_relative_gate(eng):
    G.check_tail_under_relative_gate(16000)


def test_silent_clamped_and_nan_items(eng):
    G.check_silent_clamped_and_nan(16000)


def test_deferred_normalize_gain(eng):
    G.check_deferred_gain(16000)


def test_batch_single_and_value(eng):
    G.check_batch_and_value(11025)


def test_launch_counts(eng):
    G.check_launches(16000)


def test_refusals(eng):
    G.check_refusals(16000)


@pytest.mark.parametrize("rate,T", [(16000, 12000), (11025, 3000), (44100, 30000)])
def test_oracle_gradient_is_the_finite_difference(rate, T):
    """Central differences of the float64 loudness along random directions, on items whose blocks all sit at least
    0.01 LU from both gates (so a step of 1e-6 relative changes no decision)."""
    x = G.signals(rate, 2, T, seed=5).astype(np.float64)
    Tp = lg.padded_length(T, rate)
    fw = lg.forward64(x, rate, Tp)
    assert (lg.gate_margin(fw) > 0.01).all()
    g = lg.grad64(x, rate, Tp, fw=fw)
    rng = np.random.default_rng(0)
    for _ in range(3):
        d = rng.standard_normal(x.shape)
        h = 1e-6 * np.abs(x).max()
        fd = (lg.loud_of(x + h * d, rate, Tp) - lg.loud_of(x - h * d, rate, Tp)) / (2 * h)
        an = (g * d).sum(axis=(1, 2))
        np.testing.assert_allclose(an, fd, rtol=1e-5, atol=1e-9)


def test_backward_argument_checks():
    graft.build()
    lib = _lib.B2ALibrary(_lib.LIB_PATH)
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    dbl = (ctypes.c_double * 12)()
    dp = ctypes.cast(dbl, ctypes.POINTER(ctypes.c_double))
    args = lambda **k: dict(dict(g=p, x=p, gain=None, B=1, C=1, T=16000, Tp=16000, rate=16000.0, sos=dp, sg=dp,  # noqa
                                 ns=2, blk=0.4, G=dp, z=p, lufs=p, gx=p, ws=p, wsb=1 << 30, st=None), **k)

    def call(**k):
        a = args(**k)
        return lib.b2a_lufs_backward_f32(a["g"], a["x"], a["gain"], a["B"], a["C"], a["T"], a["Tp"], a["rate"],
                                         a["sos"], a["sg"], a["ns"], a["blk"], a["G"], a["z"], a["lufs"], a["gx"],
                                         a["ws"], a["wsb"], a["st"])

    assert call(z=None) == -1 and b"lufs_backward: null pointer" in lib.b2a_last_error()
    assert call(C=6) == -1 and b"at most 5 channels" in lib.b2a_last_error()
    assert call(ns=3) == -2
    assert call(rate=100.0) == -2 and b"stride" in lib.b2a_last_error()
    need = lib.b2a_lufs_backward_workspace_bytes(1, 1, 16000, 16000.0, 0.4)
    assert need > 0 and lib.b2a_lufs_backward_workspace_bytes(1, 1, 16000, 100.0, 0.4) == 0
    assert call(wsb=need - 1) == -1 and b"workspace too small" in lib.b2a_last_error()
