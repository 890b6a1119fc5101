"""Golden gradients of the REAL reference (its AudioSignal and its spectral losses differentiate through torch),
produced like ``make_golden.py`` (same shims; run here only):
``python tests/golden/make_golden_grad.py`` -> ``reference_golden_grad.npz``
(ref:audiotools/core/audio_signal.py:1123-1212 stft, :1214-1296 istft, :1333-1369 mel_spectrogram, :1398-1426 mfcc;
ref:audiotools/metrics/spectral.py:70-95 MultiScaleSTFTLoss, :159-192 MelSpectrogramLoss).
Seeded inputs of two items x two channels at 44.1 kHz and seeded cotangents (``cotangent``).  An input gradient keeps
its first and last ``n_fft + pad`` samples in full (the padding adjoint lives there) and every SAMPLE_STRIDE-th sample
in between (``keep_index``); spectra keep every BIN_STRIDE-th bin and all frames.  Gradients keep two of the four
rows (``ROWS``: both items, both channels)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)

SR = 44100
T = 20000
SAMPLE_STRIDE = 17
BIN_STRIDE = 13
ROWS = ([0, 1], [0, 1])  # (item, channel) pairs kept: item 0 channel 0, item 1 channel 1

# (key, window_length, hop_length, window_type, match_stride, padding_type)
STFT_CASES = [
    ("w2048", 2048, 512, "hann", False, "reflect"),
    ("w512_ms", 512, 128, "hann", True, "reflect"),
    ("w32", 32, 8, "hann", False, "reflect"),
    ("w4096_sqrt", 4096, 1024, "sqrt_hann", False, "replicate"),
    ("w400_const", 400, 160, "hann", False, "constant"),
    ("w8192", 8192, 2048, "hann", False, "reflect"),
]
ISTFT_CASES = ["w2048", "w512_ms", "w400_const", "w8192"]
MEL_CASES = [("mel2048", 2048, 150), ("mel512", 512, 80)]
MFCC = dict(n_mfcc=20, n_mels=40, window_length=512, hop_length=128)
LOSS_7SCALE = dict(n_mels=[5, 10, 20, 40, 80, 160, 320], window_lengths=[32, 64, 128, 256, 512, 1024, 2048],
                   mag_weight=0.0, pow=1.0, mel_fmin=[0.0] * 7, mel_fmax=[None] * 7)


def make_input(seed=0) -> torch.Tensor:
    """[2, 2, T] float32: a chirp plus seeded noise, a different level per item."""
    g = torch.Generator().manual_seed(4400 + seed)
    t = torch.arange(T, dtype=torch.float64) / SR
    chirp = 0.3 * torch.sin(2 * np.pi * (100.0 * t + 0.5 * 40000.0 * t * t))
    x = chirp + 0.1 * torch.randn(2, 2, T, generator=g, dtype=torch.float64)
    return (x * torch.tensor([1.0, 0.25], dtype=torch.float64)[:, None, None]).float()


def cotangent(shape, seed, complex_=False) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    if complex_:
        return torch.randn(*shape, dtype=torch.complex64, generator=g)
    return torch.randn(*shape, generator=g)


def keep_index(length: int, edge: int) -> np.ndarray:
    """The samples an input gradient keeps: [0, edge), [length - edge, length) and a stride in between."""
    edge = min(edge, length)
    mid = np.arange(edge, max(edge, length - edge), SAMPLE_STRIDE)
    return np.unique(np.concatenate([np.arange(edge), mid, np.arange(length - edge, length)]))


def edge_of(wl, hop, ms):
    return wl + ((wl - hop) // 2 if ms else 0)


def main():
    from tests.golden.make_golden import import_reference

    at = import_reference()
    AudioSignal = at.AudioSignal
    from audiotools.metrics.spectral import MelSpectrogramLoss, MultiScaleSTFTLoss

    x = make_input()
    y = make_input(1)
    out = {"input_sum_abs": np.float64(x.double().abs().sum()), "target_sum_abs": np.float64(y.double().abs().sum())}
    for i, (key, wl, hop, wt, ms, pt) in enumerate(STFT_CASES):
        xg = x.clone().requires_grad_()
        s = AudioSignal(xg, SR)
        X = s.stft(window_length=wl, hop_length=hop, window_type=wt, match_stride=ms, padding_type=pt)
        G = cotangent(X.shape, 100 + i, complex_=True)
        (gx,) = torch.autograd.grad((X.real * G.real + X.imag * G.imag).sum(), xg)
        out[key + "_stft_vjp"] = gx[ROWS].numpy()[..., keep_index(T, edge_of(wl, hop, ms))]
        if key in ISTFT_CASES:
            S = X.detach().clone().requires_grad_()
            s2 = AudioSignal(x.clone(), SR)
            s2.stft_data = S
            yy = s2.istft(window_length=wl, hop_length=hop, window_type=wt, match_stride=ms).audio_data
            gy = cotangent(yy.shape, 200 + i)
            (gS,) = torch.autograd.grad((yy * gy).sum(), S)
            out[key + "_istft_len"] = np.int64(yy.shape[-1])
            out[key + "_istft_vjp"] = gS[ROWS][..., ::BIN_STRIDE, :].numpy()
    for i, (key, wl, nm) in enumerate(MEL_CASES):
        xg = x.clone().requires_grad_()
        mel = AudioSignal(xg, SR).mel_spectrogram(nm, window_length=wl, hop_length=wl // 4)
        gm = cotangent(mel.shape, 300 + i)
        (gx,) = torch.autograd.grad((mel * gm).sum(), xg, retain_graph=True)
        out[key + "_vjp"] = gx[ROWS].numpy()[..., keep_index(T, wl)]
        (gx,) = torch.autograd.grad((mel.clamp(1e-5).pow(2).log10() * gm).sum(), xg)
        out[key + "_log_vjp"] = gx[ROWS].numpy()[..., keep_index(T, wl)]
    xg = x.clone().requires_grad_()
    mf = AudioSignal(xg, SR).mfcc(**MFCC)
    (gx,) = torch.autograd.grad((mf * cotangent(mf.shape, 400)).sum(), xg)
    out["mfcc_vjp"] = gx[ROWS].numpy()[..., keep_index(T, MFCC["window_length"])]
    for key, loss_fn in [("loss_mel", MelSpectrogramLoss()), ("loss_stft", MultiScaleSTFTLoss()),
                         ("loss_mel7", MelSpectrogramLoss(**LOSS_7SCALE))]:
        xg = x.clone().requires_grad_()
        loss = loss_fn(AudioSignal(xg, SR), AudioSignal(y.clone(), SR))
        (gx,) = torch.autograd.grad(loss, xg)
        out[key] = np.float64(loss.item())
        out[key + "_grad"] = gx[ROWS].numpy()[..., keep_index(T, 2048)]
    path = os.path.join(HERE, "reference_golden_grad.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
