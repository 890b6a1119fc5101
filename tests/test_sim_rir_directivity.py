"""The directivity checks of tests/test_gpu_rir_directivity.py on the CPU-simulated build of the kernels (tests/cusim),
at 8 kHz and small sizes, also under a shuffled thread order; the oracle of tests/rir_dir64.py against known answers;
and the launch counts pinned."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import audiotools_b200.engine as engine_mod
import tests.test_gpu_rir_bands as GB
import tests.test_gpu_rir_directivity as G
from tests import rir64
from tests import rir_diffuse64 as D
from tests import rir_dir64 as R
from tests.cusim.sim_engine import sim_engine

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FS = 8000


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(GB, "DEV", "cpu")
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    return sim_engine()


# --------------------------------------------------------------------------- the oracle
def test_oracle_known_answers():
    room, fs = [6.0, 5.0, 3.0], 16000
    beta = [0.95, 0.95, 0.9, 0.9, 0.6, 0.8]
    lam = D.rates(room, beta, fs)
    n = np.array([0, 1, 10, 100, 1000, 4000])
    # omni: the one-octant envelope of tests/rir_diffuse64.py
    assert np.allclose(R.direction_mean(lam, n), D.direction_mean(lam, n), rtol=1e-12, atol=0)
    # no absorption: (1/4pi) int D_m^2 dOmega = p^2 + (1 - p)^2 / 3; a figure-eight source averages to 1/3 too
    flat = np.zeros(3)
    for p in (0.0, 0.25, 0.5, 1.0):
        v = np.array([0.6, 0.0, 0.8])
        want = p * p + (1 - p) ** 2 / 3
        assert abs(R.direction_mean(flat, [0.0], (p, v))[0] - want) < 1e-12
        assert abs(R.direction_mean(flat, [0.0], (1.0, v), (p, v))[0] - want) < 1e-12
    # the images: omni gains are tests/rir64.py's, with their parities
    d, g, off, par = R.images(room, [1.0, 1.2, 1.5], [4.0, 3.0, 1.2], beta, fs, 2000, 4)
    d2, g2, _ = rir64.images(room, [1.0, 1.2, 1.5], [4.0, 3.0, 1.2], beta, fs, 2000, 4)
    assert len(d) == len(d2) and np.allclose(np.sort(d), np.sort(d2)) and np.allclose(np.sort(g), np.sort(g2))
    assert np.array_equal(R.gains(d, g, off, par), g)
    assert np.allclose(np.linalg.norm(off, axis=1), d)


def test_envelope_matches_the_images():
    """The weighted envelope tracks sum (g D_m D_s)^2 of the images in 10 ms windows: median within 1 dB."""
    fs, L, w = 16000, 4000, 160
    rng = np.random.default_rng(0)
    room, src, mic, beta = [6.0, 5.0, 3.0], [1.0, 1.0, 1.5], [4.0, 3.0, 1.2], [0.95, 0.95, 0.9, 0.9, 0.6, 0.8]
    d, g, off, par = R.images(room, src, mic, beta, fs, L)
    for pm, ps in ((0.5, 1.0), (1.0, 0.25), (0.5, 0.25)):
        mpv, spv = (pm, G.unit(rng)), (ps, G.unit(rng))
        got = np.bincount((d // w).astype(np.int64), weights=R.gains(d, g, off, par, mpv, spv) ** 2,
                          minlength=L // w)[:L // w]
        want = np.array([R.envelope(room, beta, fs, np.arange(k * w, (k + 1) * w) + 0.5, mpv, spv).sum()
                         for k in range(L // w)])
        assert abs(float(np.median(10 * np.log10(got[2:] / want[2:])))) < 1.0, (pm, ps)


# --------------------------------------------------------------------------- the kernels on the simulator
def test_against_float64(eng):
    for mo in (-1, 0, 2):
        G.check_accuracy(eng, FS, 700, max_order=mo, seed=mo + 1)


def test_bands(eng):
    G.check_bands(eng, FS, 600, K=3, air_on=True)
    G.check_bands(eng, FS, 600, K=2, air_on=False, seed=1)


def test_hybrid(eng):
    G.check_hybrid(eng, FS, 1300, seed=1)


def test_bit_identity(eng):
    G.check_bit_identity(eng, FS, 900)


def test_reciprocity(eng):
    G.check_reciprocity(eng, FS, 900)


def test_free_field(eng):
    G.check_free_field(eng, FS, 400)


def test_launches_are_pinned(eng):
    counts = G.check_launches(eng)
    # images 1, high-pass 3, tail 1; three bands: the crossovers' fftconv and the sum on top of the images
    assert counts["flat"] == {1} and counts["hp"] == {4} and counts["tail"] == {2}
    n_bands = counts["bands"].pop()
    assert n_bands > 2


def test_errors(eng):
    G.check_errors(eng)


def test_transform(eng):
    G.check_transform(eng, T=2500, B=3)


_SHUFFLED = r"""
import sys
sys.path.insert(0, sys.argv[1])
import audiotools_b200.engine as em
import tests.test_gpu_rir_directivity as G
from tests.cusim.sim_engine import sim_engine
G.DEV = "cpu"
em._ENGINE = sim_engine()
eng = em._ENGINE
G.check_accuracy(eng, 8000, 600, seed=3)
G.check_hybrid(eng, 8000, 1100, seed=2)
print("ok")
"""


def test_rir_directivity_under_shuffled_fiber_order():
    """The simulator visits the CUDA threads of a block in a random order under CUSIM_SHUFFLE: a missing barrier
    around the staged patterns or the tail's weight tables shows up as a wrong result.  (Read once per process: run
    in a child.)"""
    env = dict(os.environ, CUSIM_SHUFFLE="1")
    r = subprocess.run([sys.executable, "-c", _SHUFFLED, REPO], env=env, cwd=REPO, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
