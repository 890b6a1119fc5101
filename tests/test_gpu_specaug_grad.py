"""Gradients through the spectral masks and the spectral gate on the H100 (``-m gpu``): the REAL reference's golden
gradients (tests/golden/make_golden_specaug_grad.py), bit-identical reruns, the three mask rows of the reference's
test_audio_grad, and SpectralGate inside an nn.Module."""
import pytest
import torch

from tests import specaug_grad_cases as sc

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(scope="module")
def at():
    import __graft_entry__ as graft

    graft.build()
    import audiotools_b200

    return audiotools_b200


@pytest.fixture(scope="module")
def golden():
    return sc.load_golden()


@pytest.mark.parametrize("key", sc.spec_keys())
def test_spectral_domain_grads_match_reference_golden(at, golden, key):
    sc.check_spec_case(golden, key, DEV)


@pytest.mark.parametrize("key", sc.wave_keys())
def test_end_to_end_grads_match_reference_golden(at, golden, key):
    sc.check_wave_case(golden, key, DEV)


def test_bit_identical_reruns(at):
    from tests.golden import make_golden_specaug_grad as mg

    for key in ["freq_val025", "time_val0", "low_val05", "gate_items_items", "e2e_compose", "e2e_gate"]:
        a = mg.run_case(at, key, DEV)[1]
        b = mg.run_case(at, key, DEV)[1]
        assert torch.equal(a, b), key


def test_reference_audio_grad_mask_rows(at):
    """ref:tests/core/test_grad.py::test_audio_grad's mask_low_magnitudes / mask_frequencies / mask_timesteps rows:
    the method on a clone of a signal that requires a gradient, istft, sum, backward -> a finite x.grad."""
    sr = 44100
    base = 0.1 * torch.randn(1, 1, sr, generator=torch.Generator().manual_seed(7))
    for name, kw in [("mask_low_magnitudes", {"db_cutoff": 0}), ("mask_frequencies", {"fmin_hz": 100, "fmax_hz": 1000}),
                     ("mask_timesteps", {"tmin_s": 0.1, "tmax_s": 0.5})]:
        x = base.clone().to(DEV).requires_grad_()
        sig = at.AudioSignal(x, sr)
        result = getattr(sig.clone(), name)(**kw)
        result.istft()
        result.audio_data.sum().backward()
        assert x.grad is not None and torch.isfinite(x.grad).all() and x.grad.abs().sum() > 0, name


def test_spectral_gate_in_a_module(at):
    """SpectralGate as a layer of an nn.Module: forward and backward on 16 x 1 ch x 1 s @ 44.1 kHz; the gradient
    reaches the module's parameter through the gate and equals the no-gate path where the gate passes everything."""
    from audiotools_b200.ml.layers import SpectralGate

    class Denoiser(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.gain = torch.nn.Parameter(torch.ones(1))
            self.gate = SpectralGate()

        def forward(self, x, nz, amount):
            return self.gate(at.AudioSignal(x * self.gain, 44100), at.AudioSignal(nz, 44100), amount).audio_data

    g = torch.Generator().manual_seed(3)
    x = (0.1 * torch.randn(16, 1, 44100, generator=g)).to(DEV)
    nz = (0.01 * torch.randn(16, 1, 22050, generator=g)).to(DEV)
    m = Denoiser().to(DEV)
    y = m(x, nz, 0.9)
    y.pow(2).mean().backward()
    assert y.shape == x.shape and torch.isfinite(m.gain.grad).all() and m.gain.grad.abs() > 0
    m.zero_grad()
    y0 = m(x, nz, 0.0)  # amount 0: the gate is the identity, the gradient that of stft -> istft
    y0.pow(2).mean().backward()
    want = 2 * (y0.detach() * x).mean()  # d/dgain mean(y^2) with y = istft(stft(gain x)) = gain x
    assert abs(m.gain.grad.item() - want.item()) <= 1e-4 * abs(want.item())
