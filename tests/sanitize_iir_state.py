"""Small driver for compute-sanitizer runs (memcheck / racecheck / synccheck) of the stateful and zero-phase passes of
csrc/iir.cu: every section count, rows just longer than the padding, around a chunk and longer than one warp's 32
chunks, every padtype, default and explicit padlen, shared and per-item sections, a gain, an unstable item, the zi /
zf pass, the backward, and the public methods on top.
`compute-sanitizer --tool racecheck python tests/sanitize_iir_state.py`"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as graft  # noqa: E402

graft.build()
from audiotools_b200 import AudioSignal  # noqa: E402
from audiotools_b200.core import iir  # noqa: E402
from audiotools_b200.engine import get_engine  # noqa: E402
from tests import test_gpu_iir as G  # noqa: E402

dev = "cuda:0"
eng = get_engine()
rng = np.random.default_rng(0)
g = torch.Generator().manual_seed(0)
for S in range(1, 9):
    for T, padtype, padlen in ((3 * (2 * S + 1) + 1, "odd", None), (1023, "even", 40), (1025, "constant", None),
                               (33 * 1024 + 7, None, None), (2000, "odd", 0)):
        x = torch.randn(3, 2, T, generator=g).to(dev)
        sos = G.random_sos(rng, 48000, S, 3)
        sos[2, 0] = [1.0, 0.0, 0.0, 1.0, 0.0, 1.5]  # unstable: item 2 is NaN
        gain = torch.tensor([1.0, 0.5, 2.0], device=dev)
        eng.sos_filtfilt(x, sos, padtype, padlen, gain=gain)
        eng.sos_filtfilt(x, sos[0], padtype, padlen, out=x)
        eng.sos_filtfilt_backward(x, sos, padtype, padlen, gain=gain)
        eng.sos_filter_zi(x, sos, torch.randn(S, 3, 2, 2, generator=g, dtype=torch.float64).to(dev), gain=gain)
sig = AudioSignal(0.1 * torch.randn(3, 2, 30000, generator=g), 48000).to(dev)
sig.audio_data.requires_grad_(True)
sig.normalize(-14.0).sos_filter(G.random_sos(rng, 48000, 3, 3), zero_phase=True)
sig.audio_data.sum().backward()
y, zf = iir.sosfilt(G.random_sos(rng, 48000, 2, 1)[0], sig.audio_data.detach(), zi=torch.zeros(2, 3, 2, 2))
torch.cuda.synchronize()
print("ok", float(y.abs().max()), float(zf.abs().max()))
