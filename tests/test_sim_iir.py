"""The biquad-cascade checks of tests/test_gpu_iir.py on the CPU-simulated build of the kernels (tests/cusim), at
smaller sizes, the cookbook restatement of tests/iir64.py against its known answers, and the argument checks of the
C entry point against the real library."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import __graft_entry__ as graft
import audiotools_b200.engine as engine_mod
import tests.test_gpu_iir as G
from audiotools_b200 import _lib
from tests import iir64
from tests.cusim.sim_engine import sim_engine

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK = G.CHUNK


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    return sim_engine()


# --------------------------------------------------------------------------- the oracle's cookbook
@pytest.mark.parametrize("sr", [16000, 44100, 48000, 192000])
def test_cookbook_known_answers(sr):
    db = lambda h: 20 * np.log10(h)  # noqa: E731
    for f0 in (30.0, 1000.0, 0.4 * sr):
        for q in (0.3, 0.7071, 4.0):
            for g in (-12.0, 6.0, 24.0):
                assert abs(db(iir64.response([iir64.cookbook("peaking", f0, g, q, sr)], [f0], sr)[0]) - g) < 1e-6
                low = iir64.cookbook("low_shelf", f0, g, q, sr)
                high = iir64.cookbook("high_shelf", f0, g, q, sr)
                assert abs(db(iir64.response([low], [0.0], sr)[0]) - g) < 1e-6
                assert abs(db(iir64.response([low], [sr / 2], sr)[0])) < 1e-6
                assert abs(db(iir64.response([high], [sr / 2], sr)[0]) - g) < 1e-6
                assert abs(db(iir64.response([high], [0.0], sr)[0])) < 1e-6
            assert iir64.response([iir64.cookbook("notch", f0, 0, q, sr)], [f0], sr)[0] < 1e-9
            f = np.linspace(0, sr / 2, 97)
            assert np.allclose(iir64.response([iir64.cookbook("all_pass", f0, 0, q, sr)], f, sr), 1, atol=1e-12)
            assert abs(iir64.response([iir64.cookbook("band_pass", f0, 0, q, sr)], [f0], sr)[0] - 1) < 1e-9
        for kind in ("low_pass", "high_pass"):
            assert abs(db(iir64.response([iir64.cookbook(kind, f0, 0, 1 / np.sqrt(2), sr)], [f0], sr)[0]) + 3.0103) < 1e-3


def test_library_design_matches_the_cookbook():
    from audiotools_b200.core import biquad

    sr = 44100
    kinds = list(biquad.KINDS)
    rng = np.random.default_rng(0)
    f = rng.uniform(10, 0.45 * sr, (3, len(kinds)))
    g = rng.uniform(-24, 24, (3, len(kinds)))
    q = rng.uniform(0.1, 20, (3, len(kinds)))
    got = biquad.design(kinds, f, g, q, sr, 3, "cpu").numpy()
    for b in range(3):
        for i, k in enumerate(kinds):
            assert np.allclose(got[b, i], iir64.cookbook(k, f[b, i], g[b, i], q[b, i], sr), rtol=1e-12, atol=1e-12)


def test_block_error_floors_quiet_blocks():
    ref = np.concatenate([np.ones(1024), 1e-9 * np.ones(1024)])[None]
    got = ref.copy()
    got[0, 1500] += 1e-6
    assert np.isclose(iir64.block_error(got, ref)[0], 1e-6 / 1e-3 / iir64.U)


# --------------------------------------------------------------------------- the kernels on the simulator
SIM_LENGTHS = (1, 2, 700, CHUNK - 1, CHUNK, CHUNK + 1, 3 * CHUNK + 17)


@pytest.mark.parametrize("sr,C", [(16000, 2), (44100, 1), (44100, 5), (48000, 2), (192000, 1)])
def test_against_float64(eng, sr, C):
    for i, T in enumerate(SIM_LENGTHS):
        G.check_accuracy(eng, sr, C, T, S=1 + (i + C) % 8, per_item=i % 2 == 1, seed=100 * i + C, gain=i % 3 == 0,
                         inplace=i % 4 == 1, reverse=i % 3 == 2)


@pytest.mark.parametrize("S", [1, 2, 5, 8])
def test_sections(eng, S):
    for per_item, reverse in ((False, False), (True, True)):
        G.check_accuracy(eng, 48000, 2, 2 * CHUNK + 5, S, per_item=per_item, seed=S, reverse=reverse)


def test_every_kind_at_the_edges_of_its_parameters(eng):
    sr = 48000
    rows = [iir64.cookbook(k, f, g, q, sr) for k in G.KINDS for f, q, g in ((10.0, 20.0, 24.0), (0.45 * sr, 0.1, -24.0),
                                                                            (20.0, 0.7071, -24.0))]
    sos = np.stack(rows)[:, None]
    rng = np.random.default_rng(3)
    x = np.stack([G.make_signal(G.SIGNALS[i % len(G.SIGNALS)], rng, sr, 1, 3 * CHUNK + 11) for i in range(len(rows))])
    G.check_accuracy(eng, sr, 1, x.shape[-1], 1, x=x, sos=sos)


def test_a_row_of_70_chunks(eng):
    """Three batches of the carry kernel's 32-chunk warp scan, with a 20 Hz Q 8 +12 dB peak."""
    sr = 48000
    sos = np.stack([iir64.cookbook("peaking", 20.0, 12.0, 8.0, sr), iir64.cookbook("high_pass", 10.0, 0.0, 0.7071, sr)])
    rng = np.random.default_rng(9)
    x = np.stack([G.make_signal(s, rng, sr, 1, 70 * CHUNK + 9) for s in ("noise", "low_tone")])
    G.check_accuracy(eng, sr, 1, x.shape[-1], 2, x=x, sos=sos[None])


def test_properties(eng):
    G.check_properties(eng)


def test_peak_gain_at_its_centre(eng):
    G.check_peak_gain(eng)


def test_gradient(eng):
    G.check_gradient(eng)


def test_api(eng):
    G.check_api(eng)


def test_cpu_tensors_are_refused():
    from audiotools_b200 import AudioSignal
    from audiotools_b200.engine import Engine

    graft.build()
    eng = Engine(_lib.B2ALibrary(_lib.LIB_PATH))  # product configuration: require_cuda=True
    ident = np.array([[1.0, 0, 0, 1, 0, 0]])
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        eng.sos_filter(torch.zeros(1, 1, 100), ident)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        AudioSignal(torch.zeros(1, 1, 16000), 16000).parametric_eq("peaking", 1000.0, 3.0)


def test_bad_arguments_launch_nothing_in_the_real_library():
    graft.build()
    lib = _lib.B2ALibrary(_lib.LIB_PATH)
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    k0 = lib.kernel_launches.value
    assert lib.b2a_sos_filter_f32(p, None, 1, 1, 16, p, 1, 9, 0, p, p, None) == -1
    assert lib.b2a_sos_filter_f32(p, None, 1, 1, 16, p, 2, 1, 0, p, p, None) == -1
    assert lib.b2a_sos_filter_f32(p, None, 1, 1, 16, None, 1, 1, 0, p, p, None) == -1
    assert lib.b2a_sos_filter_f32(p, None, 1, 1, 1 << 62, p, 1, 1, 0, p, p, None) == -1
    assert lib.kernel_launches.value == k0


_SHUFFLED = r"""
import sys
sys.path.insert(0, sys.argv[1])
import audiotools_b200.engine as em
import tests.test_gpu_iir as G
from tests.cusim.sim_engine import sim_engine
G.DEV = "cpu"
em._ENGINE = sim_engine()
eng = em._ENGINE
for S, T in ((1, 700), (3, G.CHUNK + 1), (8, 2 * G.CHUNK + 17)):
    G.check_accuracy(eng, 48000, 2, T, S, per_item=True, seed=T, gain=True, inplace=True, reverse=S == 3)
G.check_properties(eng)
print("ok")
"""


def test_iir_under_shuffled_fiber_order():
    """The simulator visits the CUDA threads of a block in a random order under CUSIM_SHUFFLE: a missing warp barrier
    that the fixed order happens to satisfy shows up as a wrong result.  (Read once per process: run in a child.)"""
    env = dict(os.environ, CUSIM_SHUFFLE="1")
    r = subprocess.run([sys.executable, "-c", _SHUFFLED, REPO], env=env, cwd=REPO, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
