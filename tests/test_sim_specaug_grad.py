"""Gradients through mask_frequencies / mask_timesteps / mask_low_magnitudes and ml.layers.SpectralGate on the
CPU-simulated build of the kernels (tests/cusim): against the REAL reference's gradients
(tests/golden/make_golden_specaug_grad.py), the adjoint identity of the band masks, the no-gradient path's launches,
the noise signal and denoise_amount, and shuffled thread order."""
import os
import subprocess
import sys

import pytest
import torch

import audiotools_b200.engine as engine_mod
from audiotools_b200 import AudioSignal
from tests import specaug_grad_cases as sc
from tests.cusim.sim_engine import sim_engine

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def sim_signals(monkeypatch):
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    yield sim_engine()


@pytest.fixture(scope="module")
def golden():
    return sc.load_golden()


@pytest.mark.parametrize("key", sc.spec_keys())
def test_spectral_domain_grads_match_reference_golden(sim_signals, golden, key):
    """Band masks on each axis (val 0 / 0.25, per-item bands), mask_low_magnitudes (val 0 / 0.5), the gate (shared /
    per-item noise, scalar / per-item amount), on an input with a silent item and zero edge frames.  mask_low with
    val = 0.5: its masked cells scale as 1 / |X|; against float64 they are 3.7e-8 away (of the largest such gradient),
    the reference's own FP32 gradient 7.2e-8 (held to 2x the reference's)."""
    sc.check_spec_case(golden, key, "cpu")


@pytest.mark.parametrize("key", sc.wave_keys())
def test_end_to_end_grads_match_reference_golden(sim_signals, golden, key):
    """stft -> masks -> istft, Compose([FrequencyMask, TimeMask, MaskLowMagnitudes]), TimeNoise, SpectralGate and
    SpectralDenoising on a waveform that requires a gradient."""
    sc.check_wave_case(golden, key, "cpu")


def _cplx(shape, seed):
    return torch.randn(shape, dtype=torch.complex64, generator=torch.Generator().manual_seed(seed))


def _inner(a, b):
    return (torch.view_as_real(a).double() * torch.view_as_real(b).double()).sum().item()


@pytest.mark.parametrize("axis", [0, 1])
def test_band_mask_adjoint_identity(sim_signals, axis):
    """<mask(X), G> = <X, mask^T(G)> (val = 0: the mask is linear; X has no zero cell)."""
    eng = sim_signals
    X, G = _cplx((3, 2, 33, 70), 1), _cplx((3, 2, 33, 70), 2)
    vals = torch.linspace(0, 8000.0 if axis == 0 else 0.5, 33 if axis == 0 else 70)
    lo = torch.tensor([1000.0, 0.0, 5000.0]) if axis == 0 else torch.tensor([0.1, 0.0, 0.3])
    hi = torch.tensor([3000.0, 600.0, 8000.0]) if axis == 0 else torch.tensor([0.2, 0.05, 0.5])
    Y = eng.spec_band_mask_out(X, vals, lo, hi, axis)
    GX = eng.spec_band_mask_backward(G, X, vals, lo, hi, axis)
    lhs, rhs = _inner(Y, G), _inner(X, GX)
    assert abs(lhs - rhs) <= 1e-6 * abs(lhs), (lhs, rhs)
    assert torch.equal(Y, eng.spec_band_mask(X.clone(), vals, lo, hi, axis))  # the in-place forward's result


def test_in_place_change_of_the_saved_spectrogram_is_caught(sim_signals):
    X = _cplx((2, 1, 33, 20), 3).requires_grad_()
    s = AudioSignal(torch.zeros(2, 1, 4000), 16000)
    s.stft_data = X * 1
    saved = s.stft_data
    out = s.mask_low_magnitudes(-10.0).stft_data
    saved.mul_(2)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        torch.view_as_real(out).sum().backward()


def test_no_grad_path_is_unchanged(sim_signals, monkeypatch):
    """Without a gradient the masks and the gate never enter the new Functions and make the same launches, with the
    same outputs, in grad mode as under torch.no_grad()."""
    from audiotools_b200.core import grad as _grad
    from audiotools_b200.ml.layers import SpectralGate

    def refuse(*a, **k):
        raise AssertionError("autograd Function used without a gradient")

    for f in (_grad.SpecBandMask, _grad.SpecMaskLow, _grad.SpecGate):
        monkeypatch.setattr(f, "apply", refuse)
    eng = sim_signals
    x = 0.3 * torch.randn(2, 1, 8000, generator=torch.Generator().manual_seed(4))
    nz = 0.01 * torch.randn(2, 1, 8000, generator=torch.Generator().manual_seed(5))

    def run():
        n0 = eng.launches
        s = AudioSignal(x.clone(), 16000)
        s.stft()
        outs = [s.mask_frequencies(1000.0, 3000.0).stft_data.clone(), s.mask_timesteps(0.1, 0.2, val=0.25).stft_data.clone(),
                s.mask_low_magnitudes(torch.tensor([-10.0, 0.0]), val=0.5).stft_data.clone(),
                SpectralGate()(AudioSignal(x.clone(), 16000), AudioSignal(nz.clone(), 16000), 0.8,
                               win_length=512, hop_length=128).audio_data]
        return eng.launches - n0, outs

    n_grad_mode, a = run()
    with torch.no_grad():
        n_no_grad, b = run()
    assert n_grad_mode == n_no_grad
    for u, v in zip(a, b):
        assert u.grad_fn is None and torch.equal(u, v)


def test_gradient_path_forward_equals_the_in_place_forward(sim_signals):
    """The out-of-place forwards of the gradient path give the no-gradient path's outputs bit for bit."""
    x = 0.3 * torch.randn(2, 1, 8000, generator=torch.Generator().manual_seed(6))

    def masks(v):
        s = AudioSignal(v, 16000)
        s.stft()
        s.mask_frequencies(1000.0, 3000.0, val=0.25).mask_timesteps(0.1, 0.2).mask_low_magnitudes(-5.0, val=0.5)
        return s.stft_data

    with torch.no_grad():
        want = masks(x.clone())
    got = masks(x.clone().requires_grad_())
    assert got.grad_fn is not None and torch.equal(got.detach(), want)


def test_noise_signal_gets_no_gradient_and_amount_refuses_one(sim_signals):
    from audiotools_b200.ml.layers import SpectralGate

    x = (0.3 * torch.randn(2, 1, 8000, generator=torch.Generator().manual_seed(7))).requires_grad_()
    nz = (0.01 * torch.randn(2, 1, 8000, generator=torch.Generator().manual_seed(8))).requires_grad_()
    out = SpectralGate()(AudioSignal(x, 16000), AudioSignal(nz, 16000), 0.9, win_length=512, hop_length=128)
    gx, gn = torch.autograd.grad(out.audio_data.sum(), (x, nz), allow_unused=True)
    assert gn is None and torch.isfinite(gx).all() and gx.abs().sum() > 0
    with pytest.raises(NotImplementedError, match="denoise_amount requires a gradient"):
        SpectralGate()(AudioSignal(x, 16000), AudioSignal(nz.detach(), 16000), torch.tensor(0.9, requires_grad=True),
                       win_length=512, hop_length=128)


_SHUFFLED = r"""
import sys
sys.path.insert(0, sys.argv[1])
import audiotools_b200.engine as em
from tests import specaug_grad_cases as sc
from tests.cusim.sim_engine import sim_engine
em._ENGINE = sim_engine()
golden = sc.load_golden()
for key in ["freq_val025", "time_val0", "low_val05", "gate_items_items"]:
    sc.check_spec_case(golden, key, "cpu")
print("ok")
"""


@pytest.mark.parametrize("seed", ["1", "2"])
def test_specaug_grad_kernels_under_shuffled_fiber_order(seed):
    """The simulator visits the CUDA threads of a block in a random order under CUSIM_SHUFFLE: a missing barrier that
    the fixed order happens to satisfy shows up as a wrong result.  (Read once per process: run in a child.)"""
    env = dict(os.environ, CUSIM_SHUFFLE=seed)
    r = subprocess.run([sys.executable, "-c", _SHUFFLED, REPO], env=env, cwd=REPO, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
