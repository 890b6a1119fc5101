"""The float64 restatement of pystoi (tests/stoi_oracle.py) that checks metrics.quality.stoi: it reproduces the golden
of the real reference's wrapper, gives 1 for identical signals, and follows the reference's test_stoi ladder
(ref:tests/metrics/test_quality.py:12-33) rebuilt on synthetic speech-like signals."""
import os
import warnings

import numpy as np
import pytest

from tests import stoi_oracle as so
from tests.golden import make_golden_quality as mg

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_golden_quality.npz")
SNRS = [50, 25, 10, 5, 0, -10, -20]


def ladder_signals(sr=44100, seconds=1.0):
    """A clean clip, a different clip and uniform [0, 1) noise, as the reference's test_stoi builds them from a WAV."""
    T = int(sr * seconds)
    x = mg.speech(sr, T, 5)
    other = mg.speech(sr, T, 0)
    nz = np.random.default_rng(1).random(T).astype(np.float32)
    return x, other, nz


def mix(x, nz, snr_db):
    """x + noise scaled to ``snr_db`` (power ratio over the clip), float32."""
    g = np.sqrt((x.astype(np.float64) ** 2).sum() / (nz.astype(np.float64) ** 2).sum() / 10 ** (snr_db / 10))
    return (x + np.float32(g) * nz).astype(np.float32)


@pytest.mark.parametrize("key", sorted(mg.CASES))
def test_oracle_reproduces_golden(key):
    g = np.load(GOLDEN)
    est, ref, sr = mg.case_signals(key)
    np.testing.assert_allclose([np.abs(est).astype(np.float64).sum(), np.abs(ref).astype(np.float64).sum()],
                               g[key + "_sum"], rtol=1e-9)
    for mode, ext in (("std", False), ("ext", True)):
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            score, kept, M = so.batch_stoi(est, ref, sr, ext)
        assert (len(w) > 0) == key.startswith("short"), [str(x.message) for x in w]
        np.testing.assert_allclose(score, g[f"{key}_{mode}"], rtol=0, atol=1e-12)
        np.testing.assert_array_equal(kept, g[key + "_kept"])
        np.testing.assert_array_equal(M, g[key + "_M"])
        assert (M == kept - 1).all()


@pytest.mark.parametrize("sr", [10000, 16000, 44100])
def test_identity_is_one(sr):
    x, _, _ = ladder_signals(sr)
    assert abs(so.stoi(x, x, sr) - 1.0) < 1e-12
    assert abs(so.stoi(x, 0.3 * x, sr) - 1.0) < 1e-12


@pytest.mark.parametrize("extended", [False, True])
def test_reference_ladder(extended):
    x, other, nz = ladder_signals()
    identity = so.stoi(x, x, 44100, extended)
    assert np.isclose(identity, 1.0)
    assert so.stoi(x, other, 44100, extended) < identity
    old = 1.0
    for snr in SNRS:
        new = so.stoi(x, mix(x, nz, snr), 44100, extended)
        assert new < old, (snr, new, old)
        old = new


def test_errors():
    x = np.zeros(1000, dtype=np.float32)
    with pytest.raises(ValueError, match="same length"):
        so.stoi(x, x[:-1], 10000)
    with pytest.raises(ValueError, match="no full 256-sample frame"):
        so.stoi(x[:256], x[:256], 10000)


def test_band_edges_are_pystoi_thirdoct():
    edges = so.band_edges()
    assert edges == [7, 9, 11, 14, 17, 22, 27, 34, 43, 55, 69, 87, 109, 138, 174, 219]  # csrc/stoi.cu band_edge
    for k in range(15):
        assert (so.OBM[k, edges[k]:edges[k + 1]] == 1).all() and so.OBM[k].sum() == edges[k + 1] - edges[k]
