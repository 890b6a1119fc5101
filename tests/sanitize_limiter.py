"""Small driver for compute-sanitizer runs (memcheck / racecheck / synccheck) of csrc/limiter.cu: every factor, rows
shorter than, equal to and longer than a chunk, look-aheads of 0, 1, the default and 1024 samples, in place and out of
place, with a gain, a silent item, and the public methods on top.
`compute-sanitizer --tool racecheck python tests/sanitize_limiter.py`"""
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
        for A in (0, 1, None, 1024):
            x = torch.randn(3, 2, T, generator=g).to(dev)
            x[2] = 0
            gain = torch.tensor([1.0, 0.5, 2.0], device=dev)
            lookahead = 0.0015 if A is None else A / sr
            eng.limit(x, sr, -1.0, lookahead, 0.05, gain=gain, want_reduction=True)
            eng.limit(x, sr, torch.tensor([-1.0, -3.0, -6.0], device=dev), lookahead, 2.0, out=x)
sig = AudioSignal(0.1 * torch.randn(3, 2, 30000, generator=g), 48000).to(dev)
sig.normalize(-14.0).limit(-1.0)
y = sig.audio_data
torch.cuda.synchronize()
print("ok", sig.true_peak().tolist(), float(y.abs().max()))
