"""Golden vectors of the REAL reference for the large power-of-two windows (the FFT kernels of csrc/fft_large.cu:
8192 .. 32768, the default window of AudioSignal at 176.4 / 192 kHz and above), produced exactly like
``make_golden.py`` (same shims; run here only):
``python tests/golden/make_golden_largewindow.py`` -> ``reference_golden_largewindow.npz``
(ref:audiotools/core/audio_signal.py:1123-1212 stft, :1214-1296 istft, :1333-1369 mel_spectrogram, :1398-1426 mfcc).
One seeded mono item at 192 kHz, long enough for the 16384-sample centre reflect pad of the 32768 window.  To keep the
fixture small, the spectra keep every BIN_STRIDE-th bin (all frames) and the waveforms every SAMPLE_STRIDE-th sample;
the strides are odd and co-prime with the transform sizes, so the kept cells sample every part of the computation."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)

SR = 192000
T = 24000
BIN_STRIDE = 11
SAMPLE_STRIDE = 7

# (key, window_length, hop_length, window_type, match_stride, padding_type)
STFT_CASES = [
    ("w8192", 8192, 2048, "hann", False, "reflect"),              # the default window at 192 kHz
    ("w8192_ms", 8192, 2048, "hann", True, "reflect"),            # match_stride: explicit pad + dropped edge frames
    ("w16384", 16384, 4096, "sqrt_hann", False, "constant"),
    ("w32768", 32768, 8192, "hann", False, "replicate"),
]


def make_input() -> torch.Tensor:
    """[1, 1, T] float32: a chirp plus seeded noise (broadband content in every bin)."""
    g = torch.Generator().manual_seed(192)
    t = torch.arange(T, dtype=torch.float64) / SR
    chirp = 0.3 * torch.sin(2 * np.pi * (200.0 * t + 0.5 * 200000.0 * t * t))
    return (chirp + 0.05 * torch.randn(T, generator=g, dtype=torch.float64)).float().reshape(1, 1, T)


def main():
    from tests.golden.make_golden import import_reference

    at = import_reference()
    AudioSignal = at.AudioSignal
    x = make_input()
    out = {"input_sum_abs": np.float64(x.double().abs().sum())}
    for key, wl, hop, wt, ms, pt in STFT_CASES:
        s = AudioSignal(x.clone(), SR)
        X = s.stft(window_length=wl, hop_length=hop, window_type=wt, match_stride=ms, padding_type=pt)
        out[key + "_stft_shape"] = np.array(X.shape)
        out[key + "_stft"] = X[..., ::BIN_STRIDE, :].numpy()
        y = s.istft(window_length=wl, hop_length=hop, window_type=wt, match_stride=ms)
        out[key + "_istft_len"] = np.int64(y.audio_data.shape[-1])
        out[key + "_istft"] = y.audio_data[..., ::SAMPLE_STRIDE].numpy()
    s = AudioSignal(x.clone(), SR)
    out["w8192_mel128"] = s.mel_spectrogram(n_mels=128, window_length=8192, hop_length=2048, window_type="hann").numpy()
    s = AudioSignal(x.clone(), SR)
    out["w8192_mfcc"] = s.mfcc(n_mfcc=20, n_mels=64, window_length=8192, hop_length=2048, window_type="hann").numpy()
    path = os.path.join(HERE, "reference_golden_largewindow.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, {k: v.shape for k, v in out.items()}, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
