"""Accuracy table of the pitch shifter and the time stretch against float64 (DESIGN.md "Pitch accuracy"): per frame
size W and shift, the worst search slack (the kernel's choice below the float64 best, in units of the rigorous bound
gamma (S_chosen + S_best)), the worst overlap-add error C_o (units of u (|a| + |b|)) and the worst rate-change error
C_r (units of u sum env |s| / |sum w| per tap), with the budgets switched off so the numbers are measured, not checked.
Also the kernel times of a pitch shift at the cfg4 shape (128 x 10 s mono at 44.1 kHz, +2 semitones).  Prints JSON
lines, with the GPU's name and power limit read in the same call.

    python tests/probes/pitch_accuracy_probe.py
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)


def emit(**kw):
    print(json.dumps(kw), flush=True)


def main():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine
    from tests import pitch64 as p64
    from tests import test_gpu_pitch_accuracy as G

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    emit(gpu=smi)
    eng = get_engine()
    p64.C_O = p64.C_R = 1e9
    kinds = ["noise", "tone+noise", "impulses", "noise_1e-3", "noise_1e-6"]
    for sr in (1000, 2000, 4000, 8000, 16000, 44100):
        W = p64.Geo(1, sr, 0.0).W
        T = 64 * W + 5
        for st in p64.SHIFTS:
            acc = G.check_pitch(eng, sr, st, T, kinds, seed=11)[0]
            sacc = G.check_stretch(eng, sr, G.factor_of(st), T, kinds, seed=12)
            g = p64.Geo(T, sr, st)
            emit(W=W, sr=sr, st=st, half=g.half, slack=round(acc["slack"], 4), C_o=round(acc["C_o"], 3),
                 C_o_stretch=round(sacc["C_o"], 3), C_r=round(acc["C_r"], 3), e_r_max=round(acc["C_r"] * 2 * g.half, 1),
                 flips=acc["flips"], searched=acc["searched"], fallback=acc["fallback"] + sacc["fallback"])

    # kernel times at the cfg4 shape
    x = 0.1 * torch.randn(128, 1, 441000, device="cuda:0")
    for _ in range(3):
        eng.pitch_shift(x, 44100, 2.0)
    torch.cuda.synchronize()
    reps = 20
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            eng.pitch_shift(x, 44100, 2.0)
        torch.cuda.synchronize()
    times = {}
    for ev in prof.events():
        if ev.device_type.name == "CUDA" and any(k in ev.name for k in ("wsola", "rate_kernel", "nominal")):
            name = ev.name.split("(")[0]
            times[name] = times.get(name, 0.0) + ev.device_time / reps
    emit(cfg4_kernel_us={k: round(v, 1) for k, v in times.items()}, gpu=smi)


if __name__ == "__main__":
    main()
