"""metrics.quality.stoi on the CPU-simulated build of csrc/stoi.cu (tests/cusim): the real reference's golden for every
case (sample rates 10 / 16 / 22.05 / 44.1 / 48 kHz, stereo, identity and scaled estimates, an SNR sweep, silent gaps, a
short item), the frame counts of the silence removal, scale invariance, bit-identical reruns and the ABI's argument
checks."""
import ctypes

import numpy as np
import pytest
import torch

import audiotools_b200.engine as engine_mod
from audiotools_b200 import AudioSignal, metrics
from tests import quality_cases as qc
from tests import stoi_oracle as so
from tests.cusim.sim_engine import sim_engine
from tests.golden import make_golden_quality as mg


@pytest.fixture
def sim(monkeypatch):
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    yield sim_engine()


@pytest.mark.parametrize("key", sorted(mg.CASES))
def test_stoi_matches_reference_golden(sim, key):
    qc.check_golden(key, "cpu")


@pytest.mark.parametrize("extended", [False, True])
def test_reference_ladder(sim, extended):
    qc.check_ladder("cpu", extended)


def test_scaled_estimate_and_reference(sim):
    est, ref, sr = mg.case_signals("sr16000")
    base = metrics.quality.stoi(*qc.signals(est, ref, sr, "cpu"))
    for ge, gr in ((0.37, 1.0), (1.0, 4.0), (2.5, 0.2)):
        v = metrics.quality.stoi(*qc.signals(est * np.float32(ge), ref * np.float32(gr), sr, "cpu"))
        assert (v - base).abs().max() < 1e-6


def test_reruns_are_bit_identical_and_match_float64(sim):
    est, ref, sr = mg.case_signals("gaps16000")
    for ext in (False, True):
        a = sim.stoi(torch.from_numpy(est), torch.from_numpy(ref), sr, ext)[0]
        b = sim.stoi(torch.from_numpy(est), torch.from_numpy(ref), sr, ext)[0]
        assert torch.equal(a, b)
        want = so.batch_stoi(est, ref, sr, ext)[0]
        assert np.abs(a.numpy() - want).max() < 1e-5


def test_gradient_input_gives_detached_result(sim):
    est, ref, sr = mg.case_signals("sr10000")
    e = AudioSignal(torch.from_numpy(est).requires_grad_(), sr)
    v = metrics.quality.stoi(e, AudioSignal(torch.from_numpy(ref), sr))
    assert not v.requires_grad and v.dtype == torch.float64


def test_errors(sim):
    x = torch.zeros(1, 1, 4000)
    with pytest.raises(ValueError, match="same"):
        metrics.quality.stoi(AudioSignal(x, 16000), AudioSignal(x[..., :-1], 16000))
    with pytest.raises(ValueError, match="no full 256-sample frame"):
        metrics.quality.stoi(AudioSignal(x[..., :400], 16000), AudioSignal(x[..., :400], 16000))
    with pytest.raises(NotImplementedError, match="P.862"):
        metrics.quality.pesq(AudioSignal(x, 16000), AudioSignal(x, 16000))
    with pytest.raises(NotImplementedError, match="ViSQOL"):
        metrics.quality.visqol(AudioSignal(x, 16000), AudioSignal(x, 16000))


def test_cpu_signal_raises_on_the_product_engine():
    """Like every DSP method, stoi of CPU signals on the CUDA build raises instead of falling back to the CPU."""
    import __graft_entry__ as graft
    from audiotools_b200 import _lib
    from audiotools_b200.engine import Engine

    graft.build()
    eng = Engine(_lib.get_lib())  # the product configuration: require_cuda=True
    x = torch.zeros(1, 1, 16000)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        eng.stoi(x, x, 16000)


def test_taps_are_pystoi_resample_window():
    from audiotools_b200.engine import Engine

    for sr in (8000, 16000, 22050, 44100, 48000):
        up, down = Engine.stoi_ratio(sr)
        h = so.resample_window_oct(so.FS, sr)
        np.testing.assert_allclose(Engine.stoi_taps(sr), h / h.sum() * up, rtol=1e-13, atol=0)
    assert Engine.stoi_ratio(10000) == (1, 1) and Engine.stoi_taps(10000).tolist() == [1.0]


def test_abi_argument_checks(sim):
    lib = sim.lib
    buf = (ctypes.c_double * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    ok = int(lib.b2a_stoi_workspace_bytes(1, 1000, 1, 1))
    assert ok > 0 and lib.b2a_stoi_workspace_bytes(0, 1000, 1, 1) == 0

    def call(est=p, T=1000, n_taps=1, up=1, down=1, ws_bytes=ok, channels=1):
        return lib.b2a_stoi_f32(est, p, 1, channels, T, 0, p, n_taps, up, down, p, p, p, p, ws_bytes, None)

    assert call(est=None) == -1 and b"null" in lib.b2a_last_error()
    assert call(channels=0) == -1 and b"bad argument" in lib.b2a_last_error()
    assert call(n_taps=2) == -1 and b"odd number of taps" in lib.b2a_last_error()
    assert call(T=256) == -1 and b"no full 256-sample frame" in lib.b2a_last_error()
    assert call(ws_bytes=ok - 1) == -1 and b"workspace" in lib.b2a_last_error()
    assert call(T=100000, up=1, down=60, n_taps=3, ws_bytes=1 << 40) == -2 and b"shared memory" in lib.b2a_last_error()
