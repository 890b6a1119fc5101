"""Small driver for compute-sanitizer runs (memcheck / racecheck / synccheck) over the STOI backward of csrc/stoi.cu on
small shapes through the public API: both modes, stereo at 44.1 kHz, a 10 kHz item with a silent gap, a short item
beside a long one, and a no_grad forward.
`compute-sanitizer --tool racecheck python tests/sanitize_stoi_grad.py`"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as graft  # noqa: E402

graft.build()
from audiotools_b200 import AudioSignal, metrics  # noqa: E402
from tests.golden import make_golden_quality as mg  # noqa: E402

dev = "cuda:0"
out = []
cases = [mg.case_signals("stereo44100"), mg.case_signals("short16000")]
ref10 = mg.speech(10000, 24000, 51, ((0.6, 1.3),))[None, None]
cases.append((mg.with_snr(ref10, 5.0, 52), ref10, 10000))
for est, ref, sr in cases:
    for ext in (False, True):
        x = torch.from_numpy(est).to(dev).requires_grad_()
        r = AudioSignal(torch.from_numpy(ref).to(dev), sr)
        loss = metrics.STOILoss(ext)(AudioSignal(x, sr), r)
        (g,) = torch.autograd.grad(loss, x)
        with torch.no_grad():
            out.append(float(metrics.STOILoss(ext)(AudioSignal(x, sr), r)))
        out += [float(loss), float(g.abs().mean())]
torch.cuda.synchronize()
print("ok", np.round(out, 6).tolist())
