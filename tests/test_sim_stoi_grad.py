"""metrics.quality.STOILoss on the CPU-simulated build of csrc/stoi.cu (tests/cusim): the loss equals -stoi() for every
golden case, its gradient matches autograd through the float64 restatement (tests/stoi_grad_cases.py), the
restatement matches the numpy oracle and scipy, the gradient's properties, the plumbing and the backward ABI's
argument checks."""
import ctypes

import numpy as np
import pytest
import torch

import audiotools_b200.engine as engine_mod
from tests import stoi_grad_cases as sg
from tests import stoi_oracle as so
from tests.cusim.sim_engine import sim_engine
from tests.golden import make_golden_quality as mg


@pytest.fixture
def sim(monkeypatch):
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    yield sim_engine()


@pytest.mark.parametrize("key", sorted(mg.CASES))
def test_loss_is_minus_stoi(sim, key):
    sg.check_value(key, "cpu")


@pytest.mark.parametrize("extended", [False, True])
@pytest.mark.parametrize("key", sorted(mg.CASES))
def test_gradient_matches_float64(sim, key, extended):
    sg.check_gradient(key, extended, "cpu")


@pytest.mark.parametrize("extended", [False, True])
def test_restatement_matches_oracle_and_its_directional_derivative(extended):
    for key in ("sr16000", "stereo44100", "gaps16000", "short16000"):
        est, ref, sr = mg.case_signals(key)
        got = sg.batch_stoi(torch.from_numpy(est).double(), torch.from_numpy(ref).double(), sr, extended).numpy()
        want = np.array([so.stoi_detail(ref[b].astype(np.float64).mean(0), est[b].astype(np.float64).mean(0), sr,
                                        extended)[0] for b in range(est.shape[0])])
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)
    sg.check_directional(extended)


def test_restatement_resampler_is_resample_poly():
    x = np.random.default_rng(0).standard_normal(20000)
    for sr in (8000, 16000, 22050, 44100, 48000):
        got = sg.resample(torch.from_numpy(x), sr).numpy()
        np.testing.assert_allclose(got, so.resample_oct(x, so.FS, sr), rtol=0, atol=1e-12)


def test_golden_cases_keep_clear_of_clip_decisions():
    """Every standard-mode cell of the golden cases is at least 5e-5 relative away from its clip threshold: fifty
    times the float32 envelopes' relative error, so the kernel and the float64 restatement clip the same cells."""
    for key in sorted(mg.CASES):
        assert sg.clip_margin(*mg.case_signals(key)) > 5e-5, key


@pytest.mark.parametrize("extended", [False, True])
def test_gradient_properties(sim, extended):
    sg.check_properties("cpu", extended)


def test_reruns_are_bit_identical(sim):
    est, ref, sr = mg.case_signals("stereo44100")
    for ext in (False, True):
        a = sg.kernel_grad(est, ref, sr, ext, "cpu")[1]
        b = sg.kernel_grad(est, ref, sr, ext, "cpu")[1]
        assert torch.equal(a, b)


def test_plumbing(sim):
    sg.check_plumbing("cpu")


def test_backward_launches(sim):
    est, ref, sr = mg.case_signals("sr16000")
    x, e, r = sg.signals(est, ref, sr, "cpu", grad=True)
    from audiotools_b200 import metrics

    loss = metrics.STOILoss()(e, r)
    n0 = sim.launches
    loss.backward()
    assert sim.launches - n0 == 4 and x.grad.shape == x.shape


def test_backward_abi_argument_checks(sim):
    lib = sim.lib
    buf = (ctypes.c_double * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    fwd = int(lib.b2a_stoi_workspace_bytes(1, 1000, 1, 1))
    ok = int(lib.b2a_stoi_backward_workspace_bytes(1, 1000, 1, 1))
    assert ok > 0 and lib.b2a_stoi_backward_workspace_bytes(1, 1000, 0, 1) == 0

    def call(g=p, fwd_ws=p, fwd_bytes=fwd, T=1000, n_taps=1, up=1, down=1, ws_bytes=ok, channels=1):
        return lib.b2a_stoi_backward_f32(g, fwd_ws, fwd_bytes, 1, channels, T, 0, p, n_taps, up, down, p, p, ws_bytes,
                                         None)

    assert call(g=None) == -1 and b"null" in lib.b2a_last_error()
    assert call(fwd_ws=None) == -1 and b"null" in lib.b2a_last_error()
    assert call(channels=0) == -1 and b"bad argument" in lib.b2a_last_error()
    assert call(up=0) == -1 and b"bad argument" in lib.b2a_last_error()
    assert call(n_taps=2) == -1 and b"odd number of taps" in lib.b2a_last_error()
    assert call(T=256) == -1 and b"no full 256-sample frame" in lib.b2a_last_error()
    assert call(fwd_bytes=fwd - 1) == -1 and b"forward workspace" in lib.b2a_last_error()
    assert call(ws_bytes=ok - 1) == -1 and lib.b2a_last_error().startswith(b"stoi_backward: workspace")
    assert call(T=100000, up=60, down=1, n_taps=3, fwd_bytes=1 << 40, ws_bytes=1 << 40) == -2 and \
        b"shared memory" in lib.b2a_last_error()
