"""metrics.quality.stoi on the H100 (csrc/stoi.cu): the real reference's golden for every case, the silence-removal
frame counts, a full-size 64 x 2ch x 10 s batch at 44.1 kHz against the float64 restatement of pystoi, bit-identical
reruns, a detached float64 CPU result, deferred gains and the reference's SNR ladder."""
import numpy as np
import pytest
import torch

from audiotools_b200 import AudioSignal, metrics
from tests import quality_cases as qc
from tests import stoi_oracle as so
from tests.golden import make_golden_quality as mg

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("key", sorted(mg.CASES))
def test_stoi_matches_reference_golden(key):
    qc.check_golden(key, DEV)


@pytest.mark.parametrize("extended", [False, True])
def test_reference_ladder(extended):
    qc.check_ladder(DEV, extended)


def test_full_size_batch_matches_float64_and_reruns_bit_identical():
    B, C, sr = 64, 2, 44100
    T = 10 * sr
    clips = np.stack([np.stack([mg.speech(sr, T, 8 * i + c, ((2.0 + 0.3 * i, 3.0 + 0.3 * i),)) for c in range(C)])
                      for i in range(8)])
    ref = np.tile(clips, (B // 8, 1, 1))
    g = np.random.default_rng(0)
    gains = np.float32(10.0) ** (g.uniform(-2, 0.5, size=(B, 1, 1)).astype(np.float32))
    est = (ref + gains * np.float32(0.02) * g.standard_normal(ref.shape, dtype=np.float32)).astype(np.float32)
    e, r = qc.signals(est, ref, sr, DEV)
    for ext in (False, True):
        a = metrics.quality.stoi(e, r, ext)
        b = metrics.quality.stoi(e, r, ext)
        assert torch.equal(a, b)
        want = so.batch_stoi(est, ref, sr, ext)[0]
        assert np.abs(a.numpy() - want).max() < 1e-5, np.abs(a.numpy() - want).max()


def test_result_is_detached_float64_cpu():
    est, ref, sr = mg.case_signals("sr16000")
    x = torch.from_numpy(est).to(DEV).requires_grad_()
    v = metrics.quality.stoi(AudioSignal(x, sr), AudioSignal(torch.from_numpy(ref), sr).to(DEV))
    assert v.dtype == torch.float64 and v.device.type == "cpu" and v.shape == (est.shape[0],)
    assert not v.requires_grad and v.grad_fn is None


def test_deferred_gain_is_applied():
    """volume_change on a CUDA signal defers its gain; stoi reads the materialised samples (STOI is scale invariant,
    so the score equals the one of the eagerly scaled signal)."""
    est, ref, sr = mg.case_signals("gaps16000")
    e, r = qc.signals(est, ref, sr, DEV)
    e.volume_change(-12.0)
    r.volume_change(6.0)
    eager = metrics.quality.stoi(*qc.signals(est * np.float32(10 ** (-12 / 20)), ref * np.float32(10 ** (6 / 20)), sr,
                                            DEV))
    assert (metrics.quality.stoi(e, r) - eager).abs().max() < 1e-6
