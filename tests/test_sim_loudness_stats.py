"""The loudness-statistics checks of tests/test_gpu_loudness_stats.py on the CPU-simulated build of the kernels
(tests/cusim), at 8 and 16 kHz and shorter signals.  The simulator build keeps at most 64 short-term keys in shared
memory (8192 on the GPU), so rows over 9.3 s run the selection from the workspace here; the argument checks of the C
entry points and the CPU refusal run against the real library."""
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
import tests.test_gpu_loudness_stats as G
from audiotools_b200 import _lib
from tests import loudness_stats64 as ls
from tests.cusim.sim_engine import sim_engine

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    return sim_engine()


@pytest.mark.parametrize("sr,C,T", [(16000, 1, 16000 * 5 + 77), (16000, 5, 16000 * 4), (11025, 2, 11025 * 4 + 3),
                                    (8000, 2, 8000 * 11)])
def test_integrated_is_bit_identical(eng, sr, C, T):
    G.check_integrated_identity(eng, sr, C, T)


def test_integrated_is_bit_identical_padded(eng):
    G.check_integrated_identity(eng, 16000, 2, 10000, Tp=16000 * 4)


@pytest.mark.parametrize("C", [1, 2, 5])
@pytest.mark.parametrize("sr", [16000, 44100, 48000])
def test_series_against_float64(eng, sr, C):
    G.check_series(eng, sr, C, int(3.4 * sr), ["noise", "sin30+noise"])


def test_series_spilled_row(eng):
    G.check_series(eng, 8000, 2, 8000 * 12, ["noise", "sin20+noise"])


@pytest.mark.parametrize("sr", [8000, 16000])
def test_gating_and_ranks_exact(eng, sr):
    G.check_gating(eng, sr)


def test_short_items(eng):
    G.check_short_items(eng, 16000)


@pytest.mark.parametrize("case,seg_s", [(1, 10.0), (2, 10.0), (3, 10.0), (4, 20.0)])
def test_ebu3342_loudness_range(eng, case, seg_s):
    G.check_ebu3342(eng, case, 8000, seg_s)


def test_signal_method(eng):
    G.check_signal_method(16000)


def test_eleven_khz_window_is_30_strides():
    lib = _lib.get_lib()
    assert lib.b2a_loudness_stats_num_short_term(33060, 11025.0) == 1       # 30 * 1102 samples, not 33075
    assert lib.b2a_loudness_stats_num_short_term(33059, 11025.0) == 0
    assert lib.b2a_loudness_stats_num_short_term(441000, 44100.0) == 71     # the bench clip: 10 s
    assert lib.b2a_loudness_stats_num_short_term(48000 * 3600, 48000.0) == 35971
    assert lib.b2a_loudness_stats_num_short_term(1000, 100.0) == -1         # stride under 64 samples
    for rate in (8000, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 176400, 192000):
        assert lib.b2a_loudness_stats_num_short_term(3 * rate, float(rate)) == 1


def test_bad_arguments_return_codes():
    graft.build()
    lib = _lib.B2ALibrary(_lib.LIB_PATH)
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    d = (ctypes.c_double * 12)()
    dp = ctypes.cast(d, ctypes.POINTER(ctypes.c_double))
    assert lib.b2a_loudness_stats_workspace_bytes(2, 2, 441000, 44100.0) > lib.b2a_lufs_workspace_bytes(
        2, 2, 441000, 44100.0, 0.4)
    assert lib.b2a_loudness_stats_workspace_bytes(0, 2, 441000, 44100.0) == 0
    rc = lib.b2a_loudness_stats_f32(p, 1, 1, 16000, 16000, 16000.0, dp, dp, 2, dp, None, None, None, p, 1 << 20, None)
    assert rc == -1 and b"loudness_stats: null pointer" in lib.b2a_last_error()
    rc = lib.b2a_loudness_stats_f32(p, 1, 6, 16000, 16000, 16000.0, dp, dp, 2, dp, p, None, None, p, 1 << 20, None)
    assert rc == -1 and b"at most 5 channels" in lib.b2a_last_error()
    rc = lib.b2a_loudness_stats_f32(p, 1, 1, 16000, 15000, 16000.0, dp, dp, 2, dp, p, None, None, p, 1 << 20, None)
    assert rc == -1 and b"T_padded < T" in lib.b2a_last_error()
    rc = lib.b2a_loudness_stats_f32(p, 1, 1, 16000, 16000, 16000.0, dp, dp, 3, dp, p, None, None, p, 1 << 20, None)
    assert rc == -2 and b"biquad stages" in lib.b2a_last_error()
    rc = lib.b2a_loudness_stats_f32(p, 1, 1, 1000, 1000, 100.0, dp, dp, 2, dp, p, None, None, p, 1 << 20, None)
    assert rc == -2 and b"gating stride" in lib.b2a_last_error()
    rc = lib.b2a_loudness_stats_f32(p, 1, 1, 16000, 16000, 16000.0, dp, dp, 2, dp, p, None, None, p, 16, None)
    assert rc == -1 and b"loudness_stats: workspace too small" in lib.b2a_last_error()


def test_cpu_tensors_are_refused():
    from audiotools_b200 import AudioSignal
    from audiotools_b200.engine import Engine

    graft.build()
    eng = Engine(_lib.B2ALibrary(_lib.LIB_PATH))  # product configuration: require_cuda=True
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        eng.loudness_stats(torch.zeros(1, 1, 16000), 16000)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        AudioSignal(torch.zeros(1, 1, 16000), 16000).loudness_stats()


def test_lra64_nearest_rank():
    """The oracle's ranks: n = 1 .. 40 values 1 .. n (all kept) give Low = floor(0.1 (n - 1) + 0.5) + 1 etc."""
    for n in range(1, 41):
        S = -30.0 + np.arange(n, dtype=np.float32) * 0.01
        r = ls.lra64(S)
        assert r["n"] == n
        assert r["LRA Low"] == np.float32(S[math.floor(0.1 * (n - 1) + 0.5)])
        assert r["LRA High"] == np.float32(S[math.floor(0.95 * (n - 1) + 0.5)])
        assert math.floor(0.1 * (n - 1) + 0.5) == (n + 4) // 10 and math.floor(0.95 * (n - 1) + 0.5) == (19 * n - 9) // 20


_SHUFFLED = r"""
import sys
sys.path.insert(0, sys.argv[1])
import audiotools_b200.engine as em
import tests.test_gpu_loudness_stats as G
from tests.cusim.sim_engine import sim_engine
G.DEV = "cpu"
em._ENGINE = sim_engine()
eng = em._ENGINE
G.check_gating(eng, 8000)
G.check_series(eng, 16000, 5, int(3.4 * 16000), ["noise", "sin30+noise"])
G.check_ebu3342(eng, 1, 8000, 10.0)
G.check_integrated_identity(eng, 8000, 2, 8000 * 11)
print("ok")
"""


def test_loudness_stats_under_shuffled_fiber_order():
    """The simulator visits the CUDA threads of a block in a random order under CUSIM_SHUFFLE: a missing barrier that
    the fixed order happens to satisfy shows up as a wrong result.  (Read once per process: run in a child.)"""
    env = dict(os.environ, CUSIM_SHUFFLE="1")
    r = subprocess.run([sys.executable, "-c", _SHUFFLED, REPO], env=env, cwd=REPO, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
