"""Small driver for compute-sanitizer runs (memcheck / racecheck / synccheck) over the large-window FFT kernels of
csrc/fft_large.cu on small shapes through the public API: stft at 8192 and 32768, stft + istft at 4096 and 16384
(the inverse includes the overlap-add fold).  The rest of the library: tests/sanitize_subset.py.
`compute-sanitizer --tool racecheck python tests/sanitize_large_window.py`"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as graft  # noqa: E402

graft.build()
from audiotools_b200 import AudioSignal  # noqa: E402

dev = "cuda:0"
x = 0.1 * torch.randn(2, 1, 40000, generator=torch.Generator().manual_seed(0))
a = AudioSignal(x.clone(), 192000).to(dev).stft(window_length=8192, hop_length=2048)
b = AudioSignal(x.clone(), 192000).to(dev).stft(window_length=32768, hop_length=8192, padding_type="constant")
ys = []
for wl in (4096, 16384):
    s = AudioSignal(x.clone(), 192000).to(dev)
    s.stft(window_length=wl, hop_length=wl // 4)
    ys.append(s.istft(window_length=wl, hop_length=wl // 4).audio_data)
torch.cuda.synchronize()
print("ok", float(a.abs().mean()), float(b.abs().mean()), [float(y.abs().mean()) for y in ys])
