"""Small driver for compute-sanitizer runs (memcheck / racecheck / synccheck) of csrc/truepeak.cu: every factor, rows
shorter than, equal to and longer than a chunk, a silent item, and the public methods on top.
`compute-sanitizer --tool racecheck python tests/sanitize_true_peak.py`"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as graft  # noqa: E402

graft.build()
from audiotools_b200 import AudioSignal  # noqa: E402
from audiotools_b200.engine import get_engine  # noqa: E402

dev = "cuda:0"
eng = get_engine()
g = torch.Generator().manual_seed(0)
for sr in (44100, 96000, 192000):
    for T in (1, 13, 4095, 4096, 4097, 9000):
        x = torch.randn(3, 2, T, generator=g).to(dev)
        x[2] = 0
        eng.true_peak(x, sr)
sig = AudioSignal(0.1 * torch.randn(3, 2, 30000, generator=g), 48000).to(dev)
tp = sig.loudness_stats(true_peak=True)["True Peak"]
sig.normalize(-14.0, true_peak_limit=-1.0)
y = sig.audio_data
torch.cuda.synchronize()
print("ok", tp.tolist(), float(y.abs().max()))
