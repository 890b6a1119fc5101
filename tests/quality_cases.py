"""Checks of metrics.quality.stoi shared by the simulator tests (tests/test_sim_quality.py, CPU tensors on the
CPU-simulated kernels) and the GPU tests (tests/test_gpu_quality.py): the golden of the real reference's wrapper, the
silence-removal frame counts, the short-item rule and the reference's SNR ladder."""
import os
import warnings

import numpy as np
import torch

from audiotools_b200 import AudioSignal, metrics
from audiotools_b200.engine import get_engine
from tests.golden import make_golden_quality as mg
from tests.test_oracle_quality import SNRS, ladder_signals, mix

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_golden_quality.npz")


def signals(est, ref, sr, device):
    return (AudioSignal(torch.from_numpy(np.ascontiguousarray(est)), sr).to(device),
            AudioSignal(torch.from_numpy(np.ascontiguousarray(ref)), sr).to(device))


def stoi_warned(est_sig, ref_sig, extended):
    """metrics.quality.stoi -> (scores, number of warnings it raised)."""
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        v = metrics.quality.stoi(est_sig, ref_sig, extended)
    return v, len([x for x in w if "Returning 1e-5" in str(x.message)])


def check_golden(key, device):
    """Scores within 1e-5 of the golden in both modes (exactly 1e-5 with one warning for the short item), kept-frame
    counts and STFT frame counts equal to the oracle's."""
    g = np.load(GOLDEN)
    est, ref, sr = mg.case_signals(key)
    np.testing.assert_allclose([np.abs(est).astype(np.float64).sum(), np.abs(ref).astype(np.float64).sum()],
                               g[key + "_sum"], rtol=1e-9)
    for mode, ext in (("std", False), ("ext", True)):
        v, n_warn = stoi_warned(*signals(est, ref, sr, device), ext)
        assert v.dtype == torch.float64 and v.device.type == "cpu" and v.shape == (est.shape[0],)
        want = g[f"{key}_{mode}"]
        assert np.abs(v.numpy() - want).max() < 1e-5, (key, mode, v.numpy(), want)
        short = g[key + "_M"] < 30
        assert n_warn == int(short.any())
        assert (v.numpy()[short] == 1e-5).all()
    e, r = signals(est, ref, sr, device)
    _, kept, short_flag = get_engine().stoi(e.audio_data, r.audio_data, sr)
    np.testing.assert_array_equal(kept.cpu().numpy(), g[key + "_kept"])
    np.testing.assert_array_equal(kept.cpu().numpy() - 1, g[key + "_M"])
    np.testing.assert_array_equal(short_flag.cpu().numpy(), g[key + "_M"] < 30)


def check_ladder(device, extended):
    """The reference's test_stoi: identity gives 1, a different clip scores lower, the score falls strictly as the SNR
    falls from 50 to -20 dB."""
    x, other, nz = ladder_signals()

    def score(est):
        e, r = signals(est[None, None], x[None, None], 44100, device)
        return float(metrics.quality.stoi(e, r, extended)[0])

    identity = score(x)
    assert abs(identity - 1.0) < 1e-6
    assert score(other) < identity
    old = 1.0
    for snr in SNRS:
        new = score(mix(x, nz, snr))
        assert new < old, (snr, new, old)
        old = new
