"""Large power-of-two windows (``-m gpu``): the FFT kernels of csrc/fft_large.cu behind AudioSignal.stft / istft /
mel_spectrogram / mfcc (forward 8192 .. 32768, inverse 4096 .. 32768) -- the default window at 88.2 / 96 kHz (4096)
and 176.4 / 192 kHz (8192).  Against the REAL reference's outputs (tests/golden/make_golden_largewindow.py) and the
oracle (oracle/signal_path.py); frame counts exactly, values to 1e-4 (global) + the element-wise criterion."""
import os

import numpy as np
import pytest
import torch

from tests.conftest import elementwise_ok, rel_err

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TOL = 1e-4
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def at():
    import __graft_entry__ as graft

    graft.build()
    import audiotools_b200

    return audiotools_b200


@pytest.fixture(scope="module")
def sp():
    from oracle import signal_path

    return signal_path


@pytest.fixture(scope="module")
def golden_large():
    return np.load(os.path.join(REPO, "tests", "golden", "reference_golden_largewindow.npz"))


def _x(B, C, T, seed):
    g = torch.Generator().manual_seed(seed)
    return 0.1 * torch.randn(B, C, T, generator=g) * (0.2 + torch.rand(B, 1, 1, generator=g))


class _NoTorchSpectral:
    """Make torch.stft / torch.istft raise inside the block: the engine must not delegate to them."""

    def __enter__(self):
        self.saved = torch.stft, torch.istft

        def forbidden(*a, **k):
            raise AssertionError("torch.stft / torch.istft called")

        torch.stft = torch.istft = forbidden

    def __exit__(self, *exc):
        torch.stft, torch.istft = self.saved


def test_large_windows_match_reference_golden(at, golden_large):
    from tests.golden import make_golden_largewindow as mg

    x = mg.make_input()
    assert abs(x.double().abs().sum().item() - float(golden_large["input_sum_abs"])) <= 1e-9 * float(golden_large["input_sum_abs"])
    for key, wl, hop, wt, ms, pt in mg.STFT_CASES:  # (the fixture keeps strided bins / samples)
        sig = at.AudioSignal(x.clone(), mg.SR).to(DEV)
        X = sig.stft(window_length=wl, hop_length=hop, window_type=wt, match_stride=ms, padding_type=pt)
        assert tuple(X.shape) == tuple(golden_large[key + "_stft_shape"]) and X.dtype == torch.complex64, key
        ref = torch.from_numpy(golden_large[key + "_stft"])
        Xs = X[..., ::mg.BIN_STRIDE, :].cpu()
        assert rel_err(torch.view_as_real(Xs), torch.view_as_real(ref)) < TOL, key
        assert elementwise_ok(Xs.abs(), ref.abs()), key
        y = sig.istft(window_length=wl, hop_length=hop, window_type=wt, match_stride=ms).audio_data.cpu()
        assert y.shape[-1] == int(golden_large[key + "_istft_len"]), key
        assert rel_err(y[..., ::mg.SAMPLE_STRIDE], torch.from_numpy(golden_large[key + "_istft"])) < TOL, key
    mel = at.AudioSignal(x.clone(), mg.SR).to(DEV).mel_spectrogram(n_mels=128, window_length=8192, hop_length=2048)
    ref = torch.from_numpy(golden_large["w8192_mel128"])
    assert mel.shape == ref.shape and rel_err(mel.cpu(), ref) < TOL and elementwise_ok(mel.cpu(), ref)
    mf = at.AudioSignal(x.clone(), mg.SR).to(DEV).mfcc(n_mfcc=20, n_mels=64, window_length=8192, hop_length=2048)
    assert rel_err(mf.cpu(), torch.from_numpy(golden_large["w8192_mfcc"])) < TOL


@pytest.mark.parametrize("sr,n_fft,hop,wtype,padding_type,T", [
    (192000, 8192, 2048, "hann", "reflect", 192000), (192000, 8192, 1000, "sqrt_hann", "constant", 60001),
    (96000, 16384, 4096, "hamming", "replicate", 96000), (192000, 32768, 8192, "hann", "reflect", 200000),
    (44100, 32768, 32768, "hann", "constant", 150000)])
def test_large_stft_istft_vs_oracle(at, sp, sr, n_fft, hop, wtype, padding_type, T):
    x = _x(3, 2, T, n_fft + hop)
    sig = at.AudioSignal(x.clone(), sr).to(DEV)
    s = sig.stft(window_length=n_fft, hop_length=hop, window_type=wtype, padding_type=padding_type)
    ref = sp.stft(x, sr, n_fft, hop, wtype, False, padding_type)
    assert s.shape == ref.shape  # frame indexing bit-exact
    assert rel_err(torch.view_as_real(s.cpu()), torch.view_as_real(ref)) < TOL
    assert elementwise_ok(s.cpu().abs(), ref.abs())
    if hop > n_fft // 2:
        return  # the window envelope vanishes between frames: torch.istft refuses, so does the engine
    y = sig.istft(window_length=n_fft, hop_length=hop, window_type=wtype).audio_data.cpu()
    y_ref = sp.istft(ref, sr, T, n_fft, hop, wtype)
    assert y.shape == y_ref.shape and rel_err(y, y_ref) < TOL
    if wtype in ("hann", "sqrt_hann", "hamming") and hop <= n_fft // 4:  # COLA: the round trip returns the signal
        assert rel_err(y[..., n_fft:-n_fft], x[..., n_fft:-n_fft]) < TOL


def test_large_match_stride_all_padding_modes(at, sp):
    x = _x(2, 1, 100000, 5)
    for pt in ("reflect", "constant", "replicate"):
        sig = at.AudioSignal(x.clone(), 192000).to(DEV)
        s = sig.stft(window_length=8192, hop_length=2048, match_stride=True, padding_type=pt)
        ref = sp.stft(x, 192000, 8192, 2048, "hann", match_stride=True, padding_type=pt)
        assert s.shape == ref.shape and rel_err(torch.view_as_real(s.cpu()), torch.view_as_real(ref)) < TOL, pt
        y = sig.istft(window_length=8192, hop_length=2048, match_stride=True).audio_data.cpu()
        y_ref = sp.istft(ref, 192000, 100000, 8192, 2048, "hann", match_stride=True)
        assert y.shape == y_ref.shape and rel_err(y, y_ref) < TOL, pt


def test_default_window_at_high_rates_builds_no_matrix_and_calls_no_torch_fft(at, sp):
    """AudioSignal(x, 192000).stft() uses the default 8192 window; 96 kHz's 4096 inverse, 16384 and 32768 too: no DFT
    matrix in the engine cache, no torch.stft / torch.istft."""
    from audiotools_b200.engine import get_engine

    eng = get_engine()
    before = {k for k in eng._packed_cache if k[0] == "dft"}  # (earlier tests of the dense path leave theirs)
    for sr, wl in ((192000, None), (96000, None), (192000, 16384), (192000, 32768)):
        x = _x(2, 1, 100000, sr)
        sig = at.AudioSignal(x.clone(), sr).to(DEV)
        with _NoTorchSpectral():
            s = sig.stft(window_length=wl, hop_length=None if wl is None else wl // 4)
            y = sig.istft(window_length=wl, hop_length=None if wl is None else wl // 4).audio_data.cpu()
        n_fft = sig.stft_params.window_length if wl is None else wl
        if wl is None:
            assert n_fft == {192000: 8192, 96000: 4096}[sr]
        ref = sp.stft(x, sr, n_fft, n_fft // 4, "hann")
        assert s.shape == ref.shape and rel_err(torch.view_as_real(s.cpu()), torch.view_as_real(ref)) < TOL
        assert rel_err(y, sp.istft(ref, sr, 100000, n_fft, n_fft // 4, "hann")) < TOL
    assert {k for k in eng._packed_cache if k[0] == "dft"} == before, "a DFT matrix was built"
    with pytest.raises(NotImplementedError, match="32768"):
        at.AudioSignal(torch.zeros(1, 1, 200000), 192000).to(DEV).stft(window_length=65536, hop_length=16384)


@pytest.mark.parametrize("sr", [96000, 192000])
def test_spectral_masks_with_default_params_vs_oracle(at, sp, sr):
    """Compose[FrequencyMask, TimeMask] with the default stft_params (4096 at 96 kHz: FFT forward + the new inverse;
    8192 at 192 kHz: both new) against the oracle's stft -> masks -> istft."""
    from audiotools_b200.data import transforms as tfm

    B, T = 4, sr
    x = _x(B, 1, T, sr + 1)
    t = tfm.Compose([tfm.FrequencyMask(), tfm.TimeMask()])
    sig = at.AudioSignal(x.clone(), sr)
    kw = t.batch_instantiate(list(range(B)), sig)
    out = t(sig.clone().to(DEV), **at.util.prepare_batch(kw, DEV)).audio_data.cpu()
    flat = at.util.flatten(kw)
    fmin, fmax, tmin, tmax = (torch.as_tensor(flat[k]).cpu() for k in (
        ("Compose", "0.FrequencyMask", "fmin_hz"), ("Compose", "0.FrequencyMask", "fmax_hz"),
        ("Compose", "1.TimeMask", "tmin_s"), ("Compose", "1.TimeMask", "tmax_s")))
    wl = int(2 ** np.ceil(np.log2(0.032 * sr)))
    # every SpectralTransform is its own stft -> op -> istft round trip
    X = sp.mask_frequencies(sp.stft(x, sr, wl, wl // 4, "hann"), sr, fmin.reshape(-1, 1, 1, 1), fmax.reshape(-1, 1, 1, 1))
    y1 = sp.istft(X, sr, T, wl, wl // 4, "hann")
    X = sp.mask_timesteps(sp.stft(y1, sr, wl, wl // 4, "hann"), T / sr, tmin.reshape(-1, 1, 1, 1), tmax.reshape(-1, 1, 1, 1))
    ref = sp.istft(X, sr, T, wl, wl // 4, "hann")
    assert out.shape == ref.shape and rel_err(out, ref) < TOL


@pytest.mark.parametrize("sr", [96000, 192000])
def test_spectral_denoising_at_high_rates(at, sr):
    """SpectralDenoising gates with its own 2048 / 512 STFT whatever the rate; at 96 / 192 kHz it must run without any
    dense DFT matrix and equal the same transform applied item by item."""
    from audiotools_b200.data import transforms as tfm
    from audiotools_b200.engine import get_engine

    before = {k for k in get_engine()._packed_cache if k[0] == "dft"}  # (earlier tests of the dense path leave theirs)
    x = _x(2, 1, sr // 2, sr + 2)
    sd = tfm.SpectralDenoising()
    sig = at.AudioSignal(x.clone(), sr)
    kw = sd.batch_instantiate([3, 4], sig)
    res = sd(sig.clone().to(DEV), **at.util.prepare_batch(kw, DEV)).audio_data.cpu()
    assert res.shape == x.shape and torch.isfinite(res).all()
    assert {k for k in get_engine()._packed_cache if k[0] == "dft"} == before, "a DFT matrix was built"


def test_at_size_192k_default_window_strided_oracle(at, sp):
    """64 x 2 ch x 10 s at 192 kHz, default window (8192 / 2048): stft, log-mel and istft on the whole batch, the oracle
    on a strided subset of items."""
    B, C, T, sr = 64, 2, 1_920_000, 192000
    g = torch.Generator().manual_seed(192)
    x = torch.empty(B, C, T)
    for i in range(0, B, 8):
        x[i:i + 8] = 0.1 * torch.randn(8, C, T, generator=g)
    x *= 0.05 + 0.95 * torch.rand(B, 1, 1, generator=g)
    sig = at.AudioSignal(x, sr).to(DEV)
    s = sig.stft()
    assert s.shape == (B, C, 4097, 938)
    sub = [0, 29, 63]
    ref = sp.stft(x[sub], sr, 8192, 2048, "hann")
    a = s[sub].cpu()
    assert rel_err(torch.view_as_real(a), torch.view_as_real(ref)) < TOL and elementwise_ok(a.abs(), ref.abs())
    y = sig.istft().audio_data
    assert y.shape == (B, C, T)
    assert rel_err(y[sub].cpu(), sp.istft(ref, sr, T, 8192, 2048, "hann")) < TOL
    del s, y
    sig.stft_data = None
    lm = at.AudioSignal(x, sr).to(DEV).mel_spectrogram(n_mels=128, log=True)
    lm_ref = sp.log_mel(sp.mel_spectrogram(x[sub], sr, 128, window_length=8192, hop_length=2048, window_type="hann"))
    assert lm.shape == (B, C, 128, 938) and (lm[sub].cpu() - lm_ref).abs().max().item() < 2e-4
