"""Large power-of-two windows (csrc/fft_large.cu: forward 8192 .. 32768, inverse 4096 .. 32768) on the CPU-simulated
build of the kernels (tests/cusim): against the REAL reference's outputs (tests/golden/make_golden_largewindow.py) and
against torch.stft / torch.istft semantics (oracle/signal_path.py), frame counts exactly."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import audiotools_b200.engine as engine_mod
from audiotools_b200 import AudioSignal, _lib
from oracle import signal_path as sp
from tests.conftest import elementwise_ok, rel_err
from tests.cusim.sim_engine import sim_engine
from tests.golden import make_golden_largewindow as mg

TOL = 1e-4
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def eng():
    return sim_engine()


@pytest.fixture(scope="module")
def golden_large():
    return np.load(os.path.join(REPO, "tests", "golden", "reference_golden_largewindow.npz"))


@pytest.fixture
def sim_signals(monkeypatch):
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    yield sim_engine()


def _window(n_fft, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.hann_window(n_fft) + 0.05 + 0.1 * torch.rand(n_fft, generator=g)


def test_golden_input_is_the_generators(golden_large):
    got = mg.make_input().double().abs().sum().item()
    assert abs(got - float(golden_large["input_sum_abs"])) <= 1e-9 * got  # the seeded input the goldens were made from


def test_large_windows_match_reference_golden(sim_signals, golden_large):
    """stft / istft through AudioSignal for every case of the generator (the fixture keeps strided bins / samples),
    then mel_spectrogram and mfcc at 8192."""
    x = mg.make_input()
    for key, wl, hop, wt, ms, pt in mg.STFT_CASES:
        sig = AudioSignal(x.clone(), mg.SR)
        X = sig.stft(window_length=wl, hop_length=hop, window_type=wt, match_stride=ms, padding_type=pt)
        assert tuple(X.shape) == tuple(golden_large[key + "_stft_shape"]), key  # frame indexing bit-exact
        ref = torch.from_numpy(golden_large[key + "_stft"])
        Xs = X[..., ::mg.BIN_STRIDE, :]
        assert rel_err(torch.view_as_real(Xs), torch.view_as_real(ref)) < TOL, key
        assert elementwise_ok(Xs.abs(), ref.abs()), key
        y = sig.istft(window_length=wl, hop_length=hop, window_type=wt, match_stride=ms).audio_data
        assert y.shape[-1] == int(golden_large[key + "_istft_len"]), key
        y_ref = torch.from_numpy(golden_large[key + "_istft"])
        assert rel_err(y[..., ::mg.SAMPLE_STRIDE], y_ref) < TOL, key
    mel = AudioSignal(x.clone(), mg.SR).mel_spectrogram(n_mels=128, window_length=8192, hop_length=2048)
    ref = torch.from_numpy(golden_large["w8192_mel128"])
    assert mel.shape == ref.shape and rel_err(mel, ref) < TOL and elementwise_ok(mel, ref)
    mf = AudioSignal(x.clone(), mg.SR).mfcc(n_mfcc=20, n_mels=64, window_length=8192, hop_length=2048)
    ref = torch.from_numpy(golden_large["w8192_mfcc"])
    assert mf.shape == ref.shape and rel_err(mf, ref) < TOL


@pytest.mark.parametrize("n_fft,hop,T,pad_mode", [(8192, 2048, 30000, "reflect"), (8192, 1000, 9000, "constant"),
                                                  (16384, 4096, 40000, "replicate"), (16384, 16384, 50000, "reflect"),
                                                  (32768, 8192, 70000, "constant"), (32768, 5000, 40000, "replicate")])
def test_large_stft_all_padding_modes_vs_oracle(eng, n_fft, hop, T, pad_mode):
    """Centre framing with each padding mode, then a match_stride-style call (explicit F.pad + dropped edge frames)."""
    g = torch.Generator().manual_seed(n_fft + hop)
    x = torch.randn(2, 1, T, generator=g)
    w = _window(n_fft, hop)
    out = eng.spectral(x, n_fft, hop, w, pad_mode=pad_mode)["stft"]
    ref = torch.stft(x.reshape(2, T), n_fft, hop, window=w, center=True, return_complex=True)
    assert out.shape[2:] == ref.shape[1:]
    assert rel_err(torch.view_as_real(out[:, 0]), torch.view_as_real(ref)) < 2e-6
    pad, right_pad = (n_fft - hop) // 2, (-T) % hop
    if pad_mode == "reflect" and pad + right_pad >= T:
        return
    xp = torch.nn.functional.pad(x, (pad, pad + right_pad), pad_mode)
    ref2 = torch.stft(xp.reshape(2, -1), n_fft, hop, window=w, center=True, return_complex=True)[..., 2:-2]
    out2 = eng.spectral(x, n_fft, hop, w, pad=pad, right_pad=right_pad, pad_mode=pad_mode, drop_edge=2)["stft"]
    assert out2.shape[2:] == ref2.shape[1:]
    assert rel_err(torch.view_as_real(out2[:, 0]), torch.view_as_real(ref2)) < 2e-6


@pytest.mark.parametrize("n_fft,wtype,match_stride", [(8192, "hann", False), (8192, "sqrt_hann", True),
                                                      (16384, "hamming", False), (32768, "hann", False)])
def test_large_stft_vs_signal_path_oracle(eng, n_fft, wtype, match_stride):
    T = 50000
    x = 0.1 * torch.randn(1, 2, T, generator=torch.Generator().manual_seed(n_fft))
    hop = n_fft // 4
    right_pad, pad = sp.compute_stft_padding(T, n_fft, hop, match_stride)
    out = eng.spectral(x, n_fft, hop, sp.get_window(wtype, n_fft), pad=pad, right_pad=right_pad,
                       drop_edge=2 if match_stride else 0)["stft"]
    ref = sp.stft(x, 192000, n_fft, hop, wtype, match_stride, "reflect")
    assert out.shape == ref.shape
    assert rel_err(torch.view_as_real(out), torch.view_as_real(ref)) < 2e-6
    assert elementwise_ok(out.abs(), ref.abs())


@pytest.mark.parametrize("n_fft", [4096, 8192, 16384, 32768])
def test_large_istft_vs_torch_istft(eng, n_fft):
    """Per-frame inverse FFT + the fold of dft.cu, at several hops (hop = n_fft included), with perturbed spectra (not
    the STFT of any signal) and lengths that end inside and past the overlap-add's support."""
    rng = np.random.RandomState(n_fft)
    for hop in (n_fft // 4, n_fft // 2 + 7, n_fft):
        g = torch.Generator().manual_seed(hop)
        w = _window(n_fft, hop)
        X = torch.stft(torch.randn(2, 3 * n_fft, generator=g), n_fft, hop, window=w, center=True, return_complex=True)
        X = X * (1 + 0.2 * torch.randn(X.shape, generator=g))
        X[:, 0] += 0.5j  # imaginary DC / Nyquist parts do not enter (C2R semantics)
        X[:, -1] -= 0.25j
        for length in (int(rng.randint(n_fft // 2, (X.shape[-1] - 1) * hop)), (X.shape[-1] - 1) * hop + 100):
            ref = torch.istft(X, n_fft, hop, window=w, center=True, length=length)
            out = eng.istft(X[:, None].contiguous(), n_fft, hop, w, length)[:, 0]
            keep = max(1, min(length, (X.shape[-1] - 1) * hop) - 2 * hop)  # the envelope -> 0 at the very end
            assert out.shape == ref.shape
            assert rel_err(out[..., :keep], ref[..., :keep]) < 5e-5, (n_fft, hop, length)


def test_deferred_gain_before_8192_mel(sim_signals):
    """normalize() defers its gain; an 8192 log-mel must consume it (scaled waveform + spectrum of the scaled signal).
    48 kHz with an explicit 8192 window: the loudness gain itself agrees with the oracle to ~3e-6 there."""
    sr, T = 48000, 96000
    x = 0.1 * torch.randn(2, 1, T, generator=torch.Generator().manual_seed(3))
    sig = AudioSignal(x.clone(), sr).normalize(-20.0)
    lm = sig.mel_spectrogram(n_mels=64, window_length=8192, hop_length=2048, log=True)
    y_ref, _ = sp.normalize(x, sr, -20.0)
    lm_ref = sp.log_mel(sp.mel_spectrogram(y_ref, sr, 64, window_length=8192, hop_length=2048, window_type="hann"))
    assert lm.shape == lm_ref.shape
    assert (lm - lm_ref).abs().max().item() < 2e-4
    assert rel_err(sig.audio_data, y_ref) < TOL


def test_large_windows_build_no_dft_matrix(eng):
    x = torch.randn(1, 1, 40000, generator=torch.Generator().manual_seed(1))
    for n_fft in (8192, 16384, 32768):
        w = torch.hann_window(n_fft)
        X = eng.spectral(x, n_fft, n_fft // 4, w)["stft"]
        eng.istft(X, n_fft, n_fft // 4, w, 40000)
    X = eng.spectral(x, 4096, 1024, torch.hann_window(4096))["stft"]
    eng.istft(X, 4096, 1024, torch.hann_window(4096), 40000)
    assert not [k for k in eng._packed_cache if k[0] == "dft" and k[3] >= 4096]


def test_window_routes_and_kernel_names(eng):
    lib = eng.lib
    FFT, LARGE, NONE = _lib.ROUTE_FFT, _lib.ROUTE_LARGE, _lib.ROUTE_NONE
    assert [lib.b2a_stft_route(n, n // 4, 0) for n in (4096, 8192, 16384, 32768, 65536, 12288)] == \
        [FFT, LARGE, LARGE, LARGE, NONE, NONE]
    assert [lib.b2a_stft_route(n, n // 4, 1) for n in (2048, 4096, 8192, 32768, 65536)] == \
        [FFT, LARGE, LARGE, LARGE, NONE]
    assert lib.b2a_stft_route(8192, 8193, 1) == NONE and lib.b2a_stft_route(8192, 8193, 0) == LARGE
    assert eng.spectral_kernel_name(8192, 2048, want_mel=False, want_stft=True) == "stft_large_kernel<13>"
    assert eng.spectral_kernel_name(32768, 8192) == "stft_large_kernel<15> + mel_from_stft_kernel"
    assert eng.spectral_kernel_name(400, 100) == "dft_forward_kernel + mel_from_stft_kernel"
    x = torch.zeros(1, 1, 140000)
    with pytest.raises(NotImplementedError, match="up to 32768"):
        eng.spectral(x, 65536, 16384, torch.ones(65536))
    with pytest.raises(NotImplementedError, match="up to 32768"):
        eng.istft(torch.zeros(1, 1, 32769, 4, dtype=torch.complex64), 65536, 16384, torch.ones(65536), 40000)
    with pytest.raises(NotImplementedError, match="dense DFT path"):  # not a power of two: the dense path's limit
        eng.spectral(torch.zeros(1, 1, 40000), 10000, 2500, torch.ones(10000))
    buf = (ctypes.c_float * 2)()  # stft_out, never written: x is null
    out = ctypes.cast(buf, ctypes.c_void_p)
    with pytest.raises(_lib.B2AError, match="stft_large: null pointer"):  # the C ABI checks its arguments itself
        lib.check(lib.b2a_spectral_f32(None, 1, 40000, 8192, 2048, None, None, 0, 0, 0, 0, None, 1, None, None, None,
                                       None, 0, 0, 0, 0.0, 1.0, None, out, None, 0, None))


_SHUFFLED = r"""
import sys, torch
sys.path.insert(0, sys.argv[1])
from tests.cusim.sim_engine import sim_engine
from tests.conftest import rel_err
eng = sim_engine()
for n_fft, hop, mode in ((8192, 2048, "reflect"), (32768, 8192, "constant")):
    x = torch.randn(1, 2, 45000, generator=torch.Generator().manual_seed(n_fft))
    w = torch.hann_window(n_fft)
    out = eng.spectral(x, n_fft, hop, w, pad_mode=mode)["stft"]
    ref = torch.stft(x.reshape(2, -1), n_fft, hop, window=w, center=True, return_complex=True)
    assert rel_err(torch.view_as_real(out[0]), torch.view_as_real(ref)) < 2e-6, n_fft
for n_fft in (4096, 16384):
    w = torch.hann_window(n_fft)
    X = torch.stft(torch.randn(2, 3 * n_fft), n_fft, n_fft // 4, window=w, center=True, return_complex=True)
    y = eng.istft(X[:, None].contiguous(), n_fft, n_fft // 4, w, 2 * n_fft)[:, 0]
    assert rel_err(y, torch.istft(X, n_fft, n_fft // 4, window=w, center=True, length=2 * n_fft)) < 5e-5, n_fft
print("ok")
"""


def test_large_kernels_under_shuffled_fiber_order():
    """The simulator visits the CUDA threads of a block in a random order under CUSIM_SHUFFLE: a missing barrier that
    the fixed order happens to satisfy shows up as a wrong result.  (Read once per process: run in a child.)"""
    env = dict(os.environ, CUSIM_SHUFFLE="1")
    r = subprocess.run([sys.executable, "-c", _SHUFFLED, REPO], env=env, cwd=REPO, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
