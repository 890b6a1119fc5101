"""Gradients through the spectral front end on the H100 (``-m gpu``): stft / istft / mel_spectrogram / mfcc backward
(csrc/grad.cu and the adjoint modes of the inverse kernels) against torch.autograd through torch.stft / torch.istft in
float64 on the same GPU, the reference's spectral losses in a training-shaped step, a cfg2-size mel backward,
determinism, and no torch.stft / torch.istft / torch.fft call on either pass."""
import pytest
import torch

from tests.conftest import elementwise_ok, rel_err

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TOL = 1e-4


@pytest.fixture(scope="module")
def at():
    import __graft_entry__ as graft

    graft.build()
    import audiotools_b200

    return audiotools_b200


def _x(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return (0.5 * torch.randn(*shape, generator=g)).to(DEV)


class _NoTorchSpectral:
    """torch.stft / torch.istft / torch.fft.* raise inside the block: neither pass may delegate to them."""

    NAMES = ("rfft", "irfft", "fft", "ifft")

    def __enter__(self):
        self.saved = (torch.stft, torch.istft, {n: getattr(torch.fft, n) for n in self.NAMES})

        def forbidden(*a, **k):
            raise AssertionError("torch.stft / torch.istft / torch.fft called")

        torch.stft = torch.istft = forbidden
        for n in self.NAMES:
            setattr(torch.fft, n, forbidden)

    def __exit__(self, *exc):
        torch.stft, torch.istft, fft = self.saved
        for n, f in fft.items():
            setattr(torch.fft, n, f)


def test_stft_istft_grads_match_autograd(at):
    from tests import grad_cases as gc

    for wl, hop, ms, pt, T in gc.STFT_GEOMETRIES:
        x = _x((2, 2, T), wl + T)
        xg = x.clone().requires_grad_()
        G = torch.randn(2, 2, wl // 2 + 1, gc.stft64(x[:1, :1].double(), wl, hop, ms=ms, pt=pt).shape[-1],
                        dtype=torch.complex64, generator=torch.Generator().manual_seed(1)).to(DEV)
        with _NoTorchSpectral():
            X = at.AudioSignal(xg, 44100).stft(window_length=wl, hop_length=hop, match_stride=ms, padding_type=pt)
            (gx,) = torch.autograd.grad(gc.real_inner(X, G), xg)
        xd = x.double().requires_grad_()
        (want,) = torch.autograd.grad(gc.real_inner(gc.stft64(xd, wl, hop, ms=ms, pt=pt), G), xd)
        assert rel_err(gx.cpu(), want.cpu()) < TOL and elementwise_ok(gx.cpu(), want.cpu(), frame_dim=-1), (wl, hop)

        S = X.detach().clone().requires_grad_()
        sig = at.AudioSignal(torch.zeros(2, 2, T, device=DEV), 44100)
        sig.stft_data = S
        gy = torch.randn(2, 2, T, generator=torch.Generator().manual_seed(2)).to(DEV)
        with _NoTorchSpectral():
            y = sig.istft(window_length=wl, hop_length=hop, match_stride=ms).audio_data
            (gS,) = torch.autograd.grad((y * gy).sum(), S)
        Sd = S.detach().to(torch.complex128).requires_grad_()
        (wantS,) = torch.autograd.grad((gc.istft64(Sd, T, wl, hop, ms=ms) * gy.double()).sum(), Sd)
        assert rel_err(torch.view_as_real(gS).cpu(), torch.view_as_real(wantS).cpu()) < TOL, (wl, hop)


def test_mel_and_mfcc_grads_match_autograd(at):
    from tests import grad_cases as gc

    for wl, n_mels, log in [(2048, 150, False), (512, 80, True), (400, 40, False), (8192, 128, False)]:
        x = _x((2, 2, 6 * wl), wl)
        xg = x.clone().requires_grad_()
        with _NoTorchSpectral():
            mel = at.AudioSignal(xg, 44100).mel_spectrogram(n_mels, window_length=wl, hop_length=wl // 4, log=log)
            gm = torch.randn(mel.shape, generator=torch.Generator().manual_seed(5)).to(DEV)
            (gx,) = torch.autograd.grad((mel * gm).sum(), xg)
        xd = x.double().requires_grad_()
        ref = gc.mel64(xd, 44100, n_mels, wl, wl // 4)
        ref = ref.clamp(1e-5).pow(2).log10() if log else ref
        (want,) = torch.autograd.grad((ref * gm.double()).sum(), xd)
        assert rel_err(gx.cpu(), want.cpu()) < TOL, (wl, n_mels, log)
    x = _x((2, 1, 8000), 11)
    xg = x.clone().requires_grad_()
    with _NoTorchSpectral():
        out = at.AudioSignal(xg, 16000).mfcc(n_mfcc=20, n_mels=40, window_length=512, hop_length=128)
        gm = torch.randn(out.shape, generator=torch.Generator().manual_seed(6)).to(DEV)
        (gx,) = torch.autograd.grad((out * gm).sum(), xg)
    xd = x.double().requires_grad_()
    dct = at.AudioSignal.get_dct(20, 40, "ortho", DEV).double()
    ref = (torch.log(gc.mel64(xd, 16000, 40, 512, 128) + 1e-6).transpose(-1, -2) @ dct).transpose(-1, -2)
    (want,) = torch.autograd.grad((ref * gm.double()).sum(), xd)
    assert rel_err(gx.cpu(), want.cpu()) < TOL


def test_training_step_reference_losses(at):
    """16 x 1 ch x 1 s at 44.1 kHz through MelSpectrogramLoss (default, 7 scales) and MultiScaleSTFTLoss as the
    reference writes them: bit-identical gradients on a rerun, loss values to 1e-4 of float64, and dL/dx as close to
    the float64 gradient as the reference's own FP32 arithmetic (torch.stft + abs + matmul on this GPU) gets, or 1e-4.

    The two mel losses are compared on the cells FP32 can resolve (``grad_cases.fp32_resolution_keep``), the same mask
    for ours, torch's FP32 path and float64.  Measured on this input without the mask: the 7-scale gradient was 9.7e-4
    from float64, 8.1e-5 for torch's FP32 path.  All of it came from ONE cell of the 5-mel / 32-sample term where the
    two mels are 3.3e-7 apart (1.4e-7 in log10 units, below one FP32 spacing of log10 values near -3): torch's FP32
    log10 returns the same value for both, the L1 sign is 0 and the cell's gradient vanishes.  Every kernel launch on
    the way is within 3e-6 of float64 given its inputs (tests/probes/mel7_hook_probe.py).  With the mask: 6.3e-6 (ours)
    and 1.2e-5 (torch FP32) for the 7-scale loss, 6.5e-6 and 8.1e-6 for the default one."""
    from tests import grad_cases as gc

    x, y = _x((16, 1, 44100), 21), _x((16, 1, 44100), 22)
    keep, dropped = [], {}
    for params in (gc.MEL_LOSS_DEFAULT, gc.MEL_LOSS_7SCALE):
        k, d = gc.fp32_resolution_keep(x, y, 44100, **params)
        keep.append(k)
        dropped = {n: dropped.get(n, 0) + v for n, v in d.items()}
    # measured: 105 of 3.7 million cells (sign 16, clamp 0, zero 89: mostly first / last frames, whose reflect-padded
    # frame is symmetric and its spectrum real)
    assert dropped["sign"] + dropped["clamp"] + dropped["zero"] <= 1e-4 * dropped["cells"], dropped
    for k in range(3):
        grads = []
        for _ in range(2):
            xg = x.clone().requires_grad_()
            with _NoTorchSpectral():
                loss = gc.signal_losses(xg, y, 44100, keep)[k]
                (gx,) = torch.autograd.grad(loss, xg)
            grads.append(gx)
        assert torch.equal(grads[0], grads[1]), k  # deterministic: no atomics, fixed summation order
        xd = x.double().requires_grad_()
        want_loss = gc.oracle_losses(xd, y.double(), 44100, keep)[k]
        (want,) = torch.autograd.grad(want_loss, xd)
        xr = x.clone().requires_grad_()
        (ref32,) = torch.autograd.grad(gc.oracle_losses(xr, y, 44100, keep)[k], xr)
        assert abs(loss.item() - want_loss.item()) < TOL * abs(want_loss.item()), k
        ours, theirs = rel_err(grads[0].cpu(), want.cpu()), rel_err(ref32.cpu(), want.cpu())
        assert ours <= max(TOL, 1.25 * theirs), (k, ours, theirs, dropped)


def test_cfg2_size_mel_backward(at):
    """64 x 2 ch x 10 s at 44.1 kHz, 2048 / 512, 128 mels: the backward of the whole batch, compared on a strided
    subset of items with torch.autograd through torch.stft (float64) on the same GPU."""
    from tests import grad_cases as gc

    x = _x((64, 2, 441000), 31)
    xg = x.clone().requires_grad_()
    with _NoTorchSpectral():
        mel = at.AudioSignal(xg, 44100).mel_spectrogram(128, window_length=2048, hop_length=512)
        gm = torch.randn(mel.shape, generator=torch.Generator().manual_seed(7)).to(DEV)
        (gx,) = torch.autograd.grad((mel * gm).sum(), xg)
    for b in (0, 21, 63):
        xd = x[b:b + 1].double().requires_grad_()
        (want,) = torch.autograd.grad((gc.mel64(xd, 44100, 128, 2048, 512) * gm[b:b + 1].double()).sum(), xd)
        assert rel_err(gx[b:b + 1].cpu(), want.cpu()) < TOL, b


def test_grads_match_reference_golden(at):
    """The golden cases of tests/golden/make_golden_grad.py (the REAL reference's gradients) on the H100."""
    import os

    import numpy as np

    from tests import grad_cases as gc

    d = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_golden_grad.npz"))
    with _NoTorchSpectral():
        errs = gc.golden_errors(d, DEV)
    assert all(v[0] < TOL for k, v in errs.items() if k != "loss_stft_grad"), errs
    gc.check_golden(d, DEV)


def test_gain_deferred_under_no_grad_is_kept(at):
    """normalize() under torch.no_grad() defers its gain on a CUDA signal; a mel spectrogram taken later with grad
    mode on applies it, differentiably (the value and the gradient are those of the normalised signal)."""
    from tests import grad_cases as gc

    x = _x((2, 1, 16000), 61)
    xg = x.clone().requires_grad_()
    s = at.AudioSignal(xg, 16000)
    with torch.no_grad():
        s.normalize(-20)
    gain = s._pending_gain.clone()
    mel = s.mel_spectrogram(40, window_length=512, hop_length=128)
    assert s._pending_gain is None
    gm = torch.randn(mel.shape, generator=torch.Generator().manual_seed(9)).to(DEV)
    (gx,) = torch.autograd.grad((mel * gm).sum(), xg)
    xd = x.double().requires_grad_()
    want_mel = gc.mel64(xd * gain.double()[:, None, None], 16000, 40, 512, 128)
    (want,) = torch.autograd.grad((want_mel * gm.double()).sum(), xd)
    assert rel_err(mel.detach().cpu(), want_mel.detach().cpu()) < TOL and rel_err(gx.cpu(), want.cpu()) < TOL


def test_grad_guard_and_no_grad_bypass(at):
    xg = _x((1, 1, 8000), 41).requires_grad_()
    with pytest.raises(NotImplementedError, match="requires a gradient"):
        at.AudioSignal(xg, 16000).low_pass(2000)
    with torch.no_grad():
        at.AudioSignal(xg, 16000).low_pass(2000)
