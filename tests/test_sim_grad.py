"""Gradients through stft / istft / mel_spectrogram / mfcc / normalize (csrc/grad.cu and the adjoint modes of the
inverse kernels) on the CPU-simulated build of the kernels (tests/cusim): against torch.autograd through torch.stft /
torch.istft in float64 (the reference's arithmetic, ref:audiotools/core/audio_signal.py:1123-1426), the adjoint
identity of every route, the reference's two spectral losses restated over AudioSignal, the no-gradient path's
launches, and the error raised by methods without a backward."""
import os
import subprocess
import sys

import pytest
import torch

import audiotools_b200.engine as engine_mod
from audiotools_b200 import AudioSignal, _lib
from tests import grad_cases as gc
from tests.conftest import elementwise_ok, rel_err
from tests.cusim.sim_engine import sim_engine

TOL = 1e-4
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def sim_signals(monkeypatch):
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    yield sim_engine()


def _x(shape, seed):
    return 0.5 * torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("wl,hop,ms,pt,T", gc.STFT_GEOMETRIES)
def test_stft_and_istft_grads_match_autograd(sim_signals, wl, hop, ms, pt, T):
    """dL/dx of stft() and dL/dstft_data of istft() against torch.autograd through torch.stft / torch.istft (float64),
    for every backward route (warp FFT, large FFT, dense DFT) and padding mode, with and without match_stride."""
    x = _x((2, 2, T), wl + T)
    xg = x.clone().requires_grad_()
    X = AudioSignal(xg, 44100).stft(window_length=wl, hop_length=hop, match_stride=ms, padding_type=pt)
    G = torch.randn(X.shape, dtype=torch.complex64, generator=torch.Generator().manual_seed(1))
    (gx,) = torch.autograd.grad(gc.real_inner(X, G), xg)
    xd = x.double().requires_grad_()
    (want,) = torch.autograd.grad(gc.real_inner(gc.stft64(xd, wl, hop, ms=ms, pt=pt), G), xd)
    assert rel_err(gx, want) < TOL and elementwise_ok(gx, want, frame_dim=-1)

    S = X.detach().clone().requires_grad_()
    sig = AudioSignal(torch.zeros(2, 2, T), 44100)
    sig.stft_data = S
    y = sig.istft(window_length=wl, hop_length=hop, match_stride=ms).audio_data
    gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(2))
    (gS,) = torch.autograd.grad((y * gy).sum(), S)
    Sd = S.detach().to(torch.complex128).requires_grad_()
    (wantS,) = torch.autograd.grad((gc.istft64(Sd, T, wl, hop, ms=ms) * gy.double()).sum(), Sd)
    assert rel_err(torch.view_as_real(gS), torch.view_as_real(wantS)) < TOL
    assert elementwise_ok(gS.abs(), wantS.abs())


@pytest.mark.parametrize("wl,hop,ms,pt,T", gc.STFT_GEOMETRIES)
def test_adjoint_identity(sim_signals, wl, hop, ms, pt, T):
    """<A x, G> = <x, A^T G> in float64 sums, for the STFT (A = stft) and the inverse (A = istft) of every route."""
    eng = sim_signals
    x = _x((1, 2, T), 7)
    w = AudioSignal.get_window("hann", wl, "cpu")
    right_pad, pad = gc.padding(T, wl, hop, ms)
    drop = 2 if ms else 0
    X = eng.spectral(x, wl, hop, w, pad=pad, right_pad=right_pad, pad_mode=pt, drop_edge=drop)["stft"]
    G = torch.randn(X.shape, dtype=torch.complex64, generator=torch.Generator().manual_seed(3))
    gx = eng.stft_backward(G, T, wl, hop, w, pad, right_pad, pt, drop)
    lhs, rhs = gc.real_inner(X, G).item(), (x.double() * gx.double()).sum().item()
    assert abs(lhs - rhs) <= 1e-5 * (abs(lhs) + (x.double().abs() * gx.double().abs()).sum().item())

    y = eng.istft(X, wl, hop, w, length=T, pad_frames=drop, trim=pad)
    gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(4))
    gS = eng.istft_backward(gy, X.shape[-1], wl, hop, w, pad_frames=drop, trim=pad)
    lhs, rhs = (y.double() * gy.double()).sum().item(), gc.real_inner(X, gS).item()
    assert abs(lhs - rhs) <= 1e-5 * (abs(lhs) + (y.double().abs() * gy.double().abs()).sum().item())


def test_conjugate_views_reach_the_kernels_resolved(sim_signals):
    """``X.conj()`` is a lazy view on X's buffer.  The engine hands the kernels its values: istft, stft_backward,
    mel_backward and a band mask give what they give for the resolved tensor, and a loss through stft_data.conj()
    (autograd passes STFT.backward a conjugate view) gets autograd's gradient."""
    eng = sim_signals
    wl, hop, T = 512, 128, 4096
    x = _x((1, 2, T), 11)
    w = AudioSignal.get_window("hann", wl, "cpu")
    X = eng.spectral(x, wl, hop, w)["stft"]
    Xc, Xr = X.conj(), X.conj().resolve_conj()
    assert Xc.is_conj() and Xc.data_ptr() == X.data_ptr()
    assert torch.equal(eng.istft(Xc, wl, hop, w, T), eng.istft(Xr, wl, hop, w, T))
    assert torch.equal(eng.stft_backward(Xc, T, wl, hop, w), eng.stft_backward(Xr, T, wl, hop, w))
    fb, lo, hi = AudioSignal._mel_tables(44100, wl, 40, 0.0, None, "cpu")
    gm = torch.randn(1, 2, 40, X.shape[-1], generator=torch.Generator().manual_seed(6))
    assert torch.equal(eng.mel_backward(Xc, gm, fb, lo, hi), eng.mel_backward(Xr, gm, fb, lo, hi))
    vals, band = torch.linspace(0, 22050, X.shape[2]), (torch.tensor([1000.0]), torch.tensor([5000.0]))
    assert torch.equal(eng.spec_band_mask_out(Xc, vals, *band, 0), eng.spec_band_mask_out(Xr, vals, *band, 0))

    xg = x.clone().requires_grad_()
    Xg = AudioSignal(xg, 44100).stft(window_length=wl, hop_length=hop)
    G = torch.randn(Xg.shape, dtype=torch.complex64, generator=torch.Generator().manual_seed(7))
    (gx,) = torch.autograd.grad((Xg.conj() * G).real.sum(), xg)
    xd = x.double().requires_grad_()
    (want,) = torch.autograd.grad((gc.stft64(xd, wl, hop).conj() * G.to(torch.complex128)).real.sum(), xd)
    assert rel_err(gx, want) < TOL


@pytest.mark.parametrize("wl,n_mels,log", [(2048, 150, False), (512, 80, False), (512, 80, True), (400, 40, False),
                                           (8192, 128, False)])
def test_mel_spectrogram_grad_matches_autograd(sim_signals, wl, n_mels, log):
    """mel_spectrogram's backward (fb^T projection, X/|X|, the fused log10 post-op) and the reference's
    clamp(1e-5).pow(2).log10() on top, against torch.autograd through torch.stft (float64)."""
    sr, T = 44100, 4 * wl
    x = _x((2, 2, T), wl)
    xg = x.clone().requires_grad_()
    mel = AudioSignal(xg, sr).mel_spectrogram(n_mels, window_length=wl, hop_length=wl // 4, log=log)
    xd = x.double().requires_grad_()
    ref = gc.mel64(xd, sr, n_mels, wl, wl // 4)
    ref = ref.clamp(1e-5).pow(2).log10() if log else ref
    gm = torch.randn(mel.shape, generator=torch.Generator().manual_seed(5))
    (gx,) = torch.autograd.grad((mel * gm).sum(), xg)
    (want,) = torch.autograd.grad((ref * gm.double()).sum(), xd, retain_graph=True)
    assert rel_err(gx, want) < TOL
    if not log:
        mel2 = AudioSignal(xg, sr).mel_spectrogram(n_mels, window_length=wl, hop_length=wl // 4)
        (gx2,) = torch.autograd.grad((mel2.clamp(1e-5).pow(2).log10() * gm).sum(), xg)
        (want2,) = torch.autograd.grad((ref.clamp(1e-5).pow(2).log10() * gm.double()).sum(), xd)
        assert rel_err(gx2, want2) < TOL


def test_golden_inputs_are_the_generators():
    import numpy as np

    from tests.golden import make_golden_grad as mg

    d = np.load(os.path.join(REPO, "tests", "golden", "reference_golden_grad.npz"))
    for key, t in (("input_sum_abs", mg.make_input()), ("target_sum_abs", mg.make_input(1))):
        got = t.double().abs().sum().item()
        assert abs(got - float(d[key])) <= 1e-9 * got, key


def test_grads_match_reference_golden(sim_signals):
    """stft / istft / mel / log-mel / mfcc VJPs and the reference's MelSpectrogramLoss (default, 7 scales) and
    MultiScaleSTFTLoss: values and dL/dx against the REAL reference's (tests/golden/make_golden_grad.py)."""
    import numpy as np

    gc.check_golden(np.load(os.path.join(REPO, "tests", "golden", "reference_golden_grad.npz")), "cpu")


def test_mfcc_grad_matches_autograd(sim_signals):
    sr, wl, T = 16000, 512, 4000
    x = _x((2, 1, T), 11)
    xg = x.clone().requires_grad_()
    out = AudioSignal(xg, sr).mfcc(n_mfcc=20, n_mels=40, window_length=wl, hop_length=128)
    xd = x.double().requires_grad_()
    dct = AudioSignal.get_dct(20, 40, "ortho", "cpu").double()
    ref = (torch.log(gc.mel64(xd, sr, 40, wl, 128) + 1e-6).transpose(-1, -2) @ dct).transpose(-1, -2)
    gm = torch.randn(out.shape, generator=torch.Generator().manual_seed(6))
    (gx,) = torch.autograd.grad((out * gm).sum(), xg)
    (want,) = torch.autograd.grad((ref * gm.double()).sum(), xd)
    assert rel_err(gx, want) < TOL


def test_reference_losses_backpropagate(sim_signals):
    """MelSpectrogramLoss (default and 7 scales) and MultiScaleSTFTLoss, as the reference writes them, over this
    package's AudioSignal: loss values and dL/dx against the same code on torch.stft in float64."""
    sr, T = 16000, 6000
    x, y = _x((2, 1, T), 21), _x((2, 1, T), 22)
    for k in range(3):
        xg = x.clone().requires_grad_()
        loss = gc.signal_losses(xg, y, sr)[k]
        (gx,) = torch.autograd.grad(loss, xg)
        xd = x.double().requires_grad_()
        want_loss = gc.oracle_losses(xd, y.double(), sr)[k]
        (want,) = torch.autograd.grad(want_loss, xd)
        assert abs(loss.item() - want_loss.item()) < TOL * abs(want_loss.item()), k
        assert rel_err(gx, want) < TOL, k


def test_no_grad_path_is_unchanged(sim_signals, monkeypatch):
    """A signal that needs no gradient never enters the differentiable path (the autograd Functions are made to
    raise), runs the launches of the no-gradient path -- one fused launch for a mel spectrogram -- and gives the same
    outputs as under torch.no_grad()."""
    from audiotools_b200.core import grad as _grad

    def refuse(*a, **k):
        raise AssertionError("autograd Function used without a gradient")

    for f in (_grad.Spectral, _grad.ISTFT, _grad.MelDCT, _grad.Gain):
        monkeypatch.setattr(f, "apply", refuse)
    eng = sim_signals
    x = _x((2, 1, 3000), 31)
    n0 = eng.launches
    AudioSignal(x.clone(), 16000).mel_spectrogram(40, window_length=512, hop_length=128)
    assert eng.launches - n0 == 1

    def run():
        n0 = eng.launches
        s = AudioSignal(x.clone(), 16000)
        mel = s.clone().mel_spectrogram(40, window_length=512, hop_length=128)
        X = s.stft(window_length=400, hop_length=100)
        y = s.istft(window_length=400, hop_length=100).audio_data
        m = AudioSignal(x.clone(), 16000).normalize(-20).mfcc(n_mfcc=13, n_mels=40, window_length=512, hop_length=128)
        return eng.launches - n0, [mel, X, y, m]

    n_grad_mode, a = run()
    with torch.no_grad():
        n_no_grad, b = run()
    assert n_grad_mode == n_no_grad
    for u, v in zip(a, b):
        assert u.grad_fn is None and torch.equal(u, v)


def test_methods_without_backward_raise(sim_signals):
    xg = _x((1, 1, 3000), 41).requires_grad_()
    with pytest.raises(NotImplementedError, match="sinc_filter.*requires a gradient.*mel_spectrogram"):
        AudioSignal(xg, 16000).low_pass(2000)
    with pytest.raises(NotImplementedError, match="spec_rotate"):
        s = AudioSignal(xg, 16000)
        s.stft(window_length=256, hop_length=64)
        s.shift_phase(0.5)
    with pytest.raises(NotImplementedError, match="hop <= window_length"):
        AudioSignal(xg, 16000).stft(window_length=256, hop_length=512)  # at forward time, not in backward()
    with torch.no_grad():
        AudioSignal(xg, 16000).low_pass(2000)
    AudioSignal(xg.detach(), 16000).low_pass(2000)


def test_normalize_then_mel_spectrogram(sim_signals):
    """normalize() on a signal that requires grad applies its gain at once (the gain is a constant, as the reference's
    loudness is not differentiable): d mel / dx = gain * (d mel / dx at the scaled signal)."""
    x = _x((2, 1, 8000), 51)
    xg = x.clone().requires_grad_()
    s = AudioSignal(xg, 16000).normalize(-20)
    assert s._pending_gain is None and s.audio_data.grad_fn is not None
    gain = (s.audio_data.detach()[:, 0, 100] / x[:, 0, 100])
    mel = s.mel_spectrogram(40, window_length=512, hop_length=128)
    gm = torch.randn(mel.shape, generator=torch.Generator().manual_seed(8))
    (gx,) = torch.autograd.grad((mel * gm).sum(), xg)
    xd = (x.double() * gain.double()[:, None, None]).requires_grad_()
    (want,) = torch.autograd.grad((gc.mel64(xd, 16000, 40, 512, 128) * gm.double()).sum(), xd)
    assert rel_err(gx, want * gain.double()[:, None, None]) < TOL


def test_deferred_gain_reaches_the_gradient_path(sim_signals):
    """A gain deferred while grad mode was off (normalize / volume_change under torch.no_grad() on a CUDA signal: the
    state is set directly here, as CPU signals never defer) is applied before the differentiable STFT, and a later
    volume_change keeps it."""
    x = _x((2, 1, 4000), 61)
    g1 = torch.tensor([0.5, 2.0])
    xg = x.clone().requires_grad_()
    s = AudioSignal(xg, 16000)
    s._pending_gain = g1.clone()
    mel = s.mel_spectrogram(40, window_length=512, hop_length=128)
    assert s._pending_gain is None
    gm = torch.randn(mel.shape, generator=torch.Generator().manual_seed(9))
    (gx,) = torch.autograd.grad((mel * gm).sum(), xg)
    xd = x.double().requires_grad_()
    want_mel = gc.mel64(xd * g1.double()[:, None, None], 16000, 40, 512, 128)
    (want,) = torch.autograd.grad((want_mel * gm.double()).sum(), xd)
    assert rel_err(mel, want_mel.detach()) < TOL and rel_err(gx, want) < TOL

    s = AudioSignal(xg, 16000)
    s._pending_gain = g1.clone()
    s.volume_change(6.0)
    g2 = 10 ** (6.0 / 20)
    assert s._pending_gain is None and rel_err(s.audio_data.detach(), x * g1[:, None, None] * g2) < 1e-6
    (gx,) = torch.autograd.grad(s.audio_data.sum(), xg)
    assert rel_err(gx, (g1 * g2)[:, None, None].expand_as(x)) < 1e-6
    with pytest.raises(NotImplementedError, match="db requires a gradient"):
        AudioSignal(xg, 16000).volume_change(torch.tensor([1.0, 2.0], requires_grad=True))


_SHUFFLED = r"""
import sys, torch
import numpy as np
sys.path.insert(0, sys.argv[1])
import audiotools_b200.engine as em
from audiotools_b200 import AudioSignal
from tests import grad_cases as gc
from tests.conftest import rel_err
from tests.cusim.sim_engine import sim_engine
em._ENGINE = sim_engine()
for wl, hop, ms, pt, T in [(256, 64, True, "reflect", 1500), (4096, 1024, False, "constant", 6000), (400, 100, False, "replicate", 1500)]:
    x = torch.randn(1, 2, T, generator=torch.Generator().manual_seed(wl))
    xg = x.clone().requires_grad_()
    mel = AudioSignal(xg, 16000).mel_spectrogram(40, window_length=wl, hop_length=hop, match_stride=ms, padding_type=pt)
    (gx,) = torch.autograd.grad(mel.sum(), xg)
    xd = x.double().requires_grad_()
    fb = torch.from_numpy(np.asarray(AudioSignal.get_mel_filters(16000, wl, 40), dtype=np.float64))
    ref = (gc.stft64(xd, wl, hop, ms=ms, pt=pt).abs().transpose(2, -1) @ fb.T).sum()
    (want,) = torch.autograd.grad(ref, xd)
    assert rel_err(gx, want) < 1e-4, (wl, rel_err(gx, want))
    S = torch.randn(1, 2, wl // 2 + 1, 12, dtype=torch.complex64, generator=torch.Generator().manual_seed(1)).requires_grad_()
    sig = AudioSignal(torch.zeros(1, 2, 11 * hop), 16000)
    sig.stft_data = S
    (gS,) = torch.autograd.grad(sig.istft(window_length=wl, hop_length=hop).audio_data.sum(), S)
    Sd = S.detach().to(torch.complex128).requires_grad_()
    (wS,) = torch.autograd.grad(gc.istft64(Sd, 11 * hop, wl, hop).sum(), Sd)
    assert rel_err(torch.view_as_real(gS), torch.view_as_real(wS)) < 1e-4, wl
print("ok")
"""


def test_grad_kernels_under_shuffled_fiber_order():
    """The simulator visits the CUDA threads of a block in a random order under CUSIM_SHUFFLE: a missing barrier that
    the fixed order happens to satisfy shows up as a wrong result.  (Read once per process: run in a child.)"""
    env = dict(os.environ, CUSIM_SHUFFLE="1")
    r = subprocess.run([sys.executable, "-c", _SHUFFLED, REPO], env=env, cwd=REPO, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
