"""Small driver for compute-sanitizer runs (memcheck / racecheck) over the shared-memory kernels of csrc/effects.cu and
csrc/dft.cu through the engine, at their stride edges: order_stat_kernel (1024 threads, a 256-bucket histogram per
pass) at T = 1023 / 1024 / 1025, alter_drr_kernel (512 threads, warp partials) at T = 511 / 512 / 513 with 1 and 2
channels, peak_scale_bwd_kernel (256-slot tree reductions) at T = 255 / 256 / 257 in both modes, and mel_dct_kernel
(the basis staged in dynamic shared memory) at 127 / 128 / 129 frames and 31 / 32 / 33 coefficients.
`compute-sanitizer --tool racecheck python tests/sanitize_effects.py`"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as graft  # noqa: E402

graft.build()
from audiotools_b200.engine import get_engine  # noqa: E402

dev = "cuda:0"
eng = get_engine()
gen = torch.Generator().manual_seed(0)


def randn(*shape):
    return torch.randn(shape, generator=gen).to(dev)


out = []
for T in (1023, 1024, 1025):
    out += eng.order_stats(randn(T), torch.tensor([0, T // 2, T - 1])).tolist()
for T in (511, 512, 513):
    for C in (1, 2):
        out.append(float(eng.alter_drr(randn(2, C, T), 44100, torch.tensor([3.0, -3.0])).abs().sum()))
for T in (255, 256, 257):
    g, y, x = randn(3, T), randn(3, T), randn(3, T)
    out.append(float(eng.peak_scale_backward(g, y, max_abs=0.5)[0].abs().sum()))
    gy, gx = eng.peak_scale_backward(g, y, x)
    out += [float(gy.abs().sum()), float(gx.abs().sum())]
for N in (127, 128, 129):
    for n_mfcc in (31, 32, 33):
        out.append(float(eng.mel_dct(randn(2, 1, 40, N), randn(40, n_mfcc)).abs().sum()))
torch.cuda.synchronize()
print("ok", [round(v, 3) for v in out])
