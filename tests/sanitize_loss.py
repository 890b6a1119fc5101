"""Small driver for compute-sanitizer runs (memcheck / racecheck / synccheck) over csrc/loss.cu on small shapes through
the public API: the mel and the STFT loss (both kernel modes), a target that requires a gradient, match_stride with
constant padding, an odd hop (engine level), and a no_grad forward.
`compute-sanitizer --tool racecheck python tests/sanitize_loss.py`"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as graft  # noqa: E402

graft.build()
from audiotools_b200 import AudioSignal, STFTParams, metrics  # noqa: E402
from audiotools_b200.engine import get_engine  # noqa: E402

dev = "cuda:0"
g = torch.Generator().manual_seed(0)
x = (0.1 * torch.randn(2, 2, 12000, generator=g)).to(dev)
y = (0.1 * torch.randn(2, 2, 12000, generator=g)).to(dev)
sp = STFTParams(512, 128, "hann", True, "constant")
out = []
for mod in (metrics.MelSpectrogramLoss([40, 20], [1024, 128]), metrics.MultiScaleSTFTLoss([2048, 256, 64])):
    xg, yg = x.clone().requires_grad_(), y.clone().requires_grad_()
    loss = mod(AudioSignal(xg, 44100), AudioSignal(yg, 44100))
    gx, gy = torch.autograd.grad(loss, (xg, yg))
    with torch.no_grad():
        out.append(float(mod(AudioSignal(x, 44100, stft_params=sp), AudioSignal(y, 44100, stft_params=sp))))
    out += [float(loss), float(gx.abs().mean()), float(gy.abs().mean())]
w = AudioSignal.get_window("hann", 256, dev)
loss, gX, gY = get_engine().spectral_loss(x, y, 256, 37, w, want_grad_x=True, want_grad_y=True)
torch.cuda.synchronize()
print("ok", out, float(loss), float(gX.abs().mean()), float(gY.abs().mean()))
