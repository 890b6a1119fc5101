"""Small driver for compute-sanitizer runs (memcheck / racecheck / synccheck) of the moving impulse response
(csrc/fftconv.cu ``path_fir_kernel`` + ``path_ifft_kernel``): waypoints on, beside and between block edges, one
waypoint, L = 1, L > T and many partitions, 1 / 2 / 5 channels with per-channel and shared IRs, bypassed items, and the
transform on top.
`compute-sanitizer --tool racecheck python tests/sanitize_moving_ir.py`"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as graft  # noqa: E402

graft.build()
from audiotools_b200 import AudioSignal  # noqa: E402
from audiotools_b200.data import transforms as tfm  # noqa: E402
from audiotools_b200.engine import get_engine  # noqa: E402
from tests.test_gpu_moving_ir import SHAPES, case  # noqa: E402

eng = get_engine()
for B, C, n_ch, T, L, hop in SHAPES:
    x, irs = case(B, C, n_ch, T, L, hop)
    eng.circular_convolve_moving(x, irs, hop)
    eng.circular_convolve_moving(x, irs, hop, bypass=torch.arange(B, device=x.device) % 2 == 0)
x = 0.1 * torch.randn(3, 2, 16000, generator=torch.Generator().manual_seed(0))
t = tfm.SyntheticRoomImpulseResponse(prob=0.7, duration=0.1, diffuse_after=0.02, source_speed=("uniform", 0.5, 3.0),
                                     waypoint_hop=0.07)
sig = AudioSignal(x, 16000).to("cuda:0")
y = t(sig, **t.batch_instantiate(list(range(3)), sig)).audio_data
torch.cuda.synchronize()
print("ok", float(y.abs().max()))
