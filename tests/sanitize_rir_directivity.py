"""Small driver for compute-sanitizer runs (memcheck / racecheck / synccheck) of csrc/rir.cu's directional kernels:
lengths below, at and past a tile, 1 / 2 / 8 microphones with per-microphone patterns, images only, every max_order
kind, bands with air and the hybrid, and the transform on top.
`compute-sanitizer --tool racecheck python tests/sanitize_rir_directivity.py`"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as graft  # noqa: E402

graft.build()
from audiotools_b200 import AudioSignal  # noqa: E402
from audiotools_b200.core.room import image_source_ir  # noqa: E402
from audiotools_b200.data import transforms as tfm  # noqa: E402

dev = "cuda:0"
rng = np.random.default_rng(0)
rooms = np.array([[2.0, 2.0, 2.0], [5.0, 4.0, 3.0], [30.0, 1.5, 3.0]])
for fs in (8000, 48000):
    for L in (30, 511, 513, 2000):
        for C, mo in ((1, -1), (2, 0), (8, 10)):
            src = np.stack([rng.uniform(0.05, r - 0.05) for r in rooms])
            mics = np.stack([rng.uniform(0.05, r - 0.05, (C, 3)) for r in rooms])
            d = dict(mic_pattern=rng.uniform(0, 1, (3, C)), mic_orientation=rng.standard_normal((3, C, 3)),
                     source_pattern="cardioid", source_orientation=rng.standard_normal((3, 3)))
            image_source_ir(rooms, src, mics, fs, L, beta=rng.uniform(0, 1, (3, 6)), max_order=mo, device=dev, **d)
            image_source_ir(rooms, src, mics, fs, L, beta=rng.uniform(0.2, 1, (3, 6, 4)), bands=4,
                            air_absorption=rng.uniform(0, 0.2, 4), device=dev, **d)
            image_source_ir(rooms, src, mics, fs, L, beta=rng.uniform(0.2, 1, (3, 6)), diffuse_after=0.01,
                            seed=[1, 2, 3], device=dev, **d)
x = 0.1 * torch.randn(3, 2, 16000, generator=torch.Generator().manual_seed(0))
t = tfm.SyntheticRoomImpulseResponse(prob=0.7, diffuse_after=0.05, mic_pattern="cardioid", source_pattern=0.25)
sig = AudioSignal(x, 16000).to(dev)
y = t(sig, **t.batch_instantiate(list(range(3)), sig)).audio_data
torch.cuda.synchronize()
print("ok", float(y.abs().max()))
