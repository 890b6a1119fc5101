"""Small driver for compute-sanitizer runs (memcheck / racecheck / synccheck) of csrc/iir.cu: every section count,
rows shorter than, equal to and longer than a chunk and than one warp's 32 chunks, shared and per-item sections,
forward and reverse, in place and out of place, with a gain, an unstable item, and the public methods on top.
`compute-sanitizer --tool racecheck python tests/sanitize_iir.py`"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as graft  # noqa: E402

graft.build()
from audiotools_b200 import AudioSignal  # noqa: E402
from audiotools_b200.engine import get_engine  # noqa: E402
from tests import test_gpu_iir as G  # noqa: E402

dev = "cuda:0"
eng = get_engine()
rng = np.random.default_rng(0)
g = torch.Generator().manual_seed(0)
for S in range(1, 9):
    for T in (1, 13, 1023, 1024, 1025, 33 * 1024 + 7):
        x = torch.randn(3, 2, T, generator=g).to(dev)
        sos = G.random_sos(rng, 48000, S, 3)
        sos[2, 0] = [1.0, 0.0, 0.0, 1.0, 0.0, 1.5]  # unstable: item 2 is NaN
        gain = torch.tensor([1.0, 0.5, 2.0], device=dev)
        eng.sos_filter(x, sos, gain=gain)
        eng.sos_filter(x, sos[0], reverse=True, out=x)
sig = AudioSignal(0.1 * torch.randn(3, 2, 30000, generator=g), 48000).to(dev)
sig.normalize(-14.0).parametric_eq(["low_shelf", "peaking", "high_shelf"], [100.0, 1000.0, 8000.0], [3.0, -6.0, 2.0],
                                   [0.7, 2.0, 0.7])
y = sig.audio_data
torch.cuda.synchronize()
print("ok", float(y.abs().max()))
