"""Small driver for compute-sanitizer runs (memcheck / racecheck / synccheck) over the backward kernels of
csrc/grad.cu and the adjoint modes of the inverse kernels, on small shapes through the public API: stft backward on the
warp (512, match_stride reflect), large (4096 replicate, 8192) and dense (400 constant) routes, istft backward on the
same routes, and the mel / log-mel / mfcc backward.  `compute-sanitizer --tool racecheck python tests/sanitize_grad.py`"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as graft  # noqa: E402

graft.build()
from audiotools_b200 import AudioSignal  # noqa: E402

dev = "cuda:0"
x = (0.1 * torch.randn(2, 1, 20000, generator=torch.Generator().manual_seed(0))).to(dev)
out = []
for wl, hop, ms, pt in [(512, 128, True, "reflect"), (4096, 1024, False, "replicate"), (8192, 2048, False, "reflect"),
                        (400, 100, False, "constant")]:
    xg = x.clone().requires_grad_()
    s = AudioSignal(xg, 44100)
    X = s.stft(window_length=wl, hop_length=hop, match_stride=ms, padding_type=pt)
    S = X.detach().clone().requires_grad_()
    s.stft_data = S
    y = s.istft(window_length=wl, hop_length=hop, match_stride=ms).audio_data
    (gx, gS) = torch.autograd.grad(X.abs().sum() + y.sum(), (xg, S))
    out += [float(gx.abs().mean()), float(gS.abs().mean())]
xg = x.clone().requires_grad_()
loss = (AudioSignal(xg, 44100).mel_spectrogram(80, window_length=1024, hop_length=256, log=True).sum()
        + AudioSignal(xg, 44100).mfcc(n_mfcc=13, n_mels=40, window_length=512, hop_length=128).sum())
(gx,) = torch.autograd.grad(loss, xg)
torch.cuda.synchronize()
print("ok", out, float(gx.abs().mean()))
