"""Accuracy table of the time-domain engines against float64 (DESIGN.md "Time-domain accuracy"): the worst budget
ratio of every check in tests/test_gpu_timedomain_accuracy.py, in units of its constant C, the K-weighting's per-block
error next to the sequential float32 cascade's, and the loudness offsets of bass tones against the oracle.  Prints JSON
lines, with the GPU's name and power limit.

    python tests/probes/timedomain_accuracy_probe.py
"""
import json
import math
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
    from oracle import signal_path as sp
    from tests import test_gpu_timedomain_accuracy as G
    from tests import timedomain64 as td

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    emit(gpu=smi)
    eng = get_engine()
    worst = 0.0
    for K in G.FIR_K:
        for st in G.FIR_STRIDE:
            for T in (2047, 2049, 3 * 2048 * st + 5):
                if eng.lib.b2a_fir_direct_supported(T, K, st):
                    worst = max(worst, G.check_fir_direct(eng, T, K, st))
    emit(route="fir_direct", C_measured=worst, budget=td.BUDGET_C["fir_direct"])
    worst = 0.0
    for L in G.FFT_L:
        for T in G.FFT_T:
            worst = max(worst, G.check_fftconv(eng, T, L, offset0=L // 2))
    emit(route="fftconv", C_measured=worst, budget=td.BUDGET_C["fftconv"])
    worst = max(G.check_circconv(eng, T, L, n) for T, L in ((3000, 3000), (5000, 1200), (2000, 4500)) for n in (1, 2))
    emit(route="circconv", C_measured=worst, budget=td.BUDGET_C["circconv"])
    for rt in ("fir_direct", "resample"):
        w = 0.0
        for old, new in G.RESAMPLE:
            if td.resample_route(eng.lib, 50000, old, new) == rt:
                w = max(w, G.check_resample(eng, old, new, 50000))
        emit(route=f"resample via {rt}", C_measured=w, budget=td.BUDGET_C[rt])
    for old, new in ((48000, 16000), (44100, 16000), (16000, 44100), (11025, 96000)):
        kt = eng._resample_kernel(old, new, "cuda:0")[0]
        g = torch.randn(2, new * 20000 // old, dtype=torch.float64).float()
        gx, a = td.resample_backward64(g, 20000, old, new, kt)
        c = td.direct_errors(eng.resample_backward(g.cuda(), 20000, old, new), gx, a).max() / (td.U * math.sqrt(kt.shape[0]))
        emit(route=f"resample_backward {old}->{new}", C_measured=c, budget=td.BUDGET_C["resample"])
    for sr in G.KW_RATES:
        T = int(2.5 * sr)
        sig = G.kw_signals(sr, T)
        names = list(sig)
        b, v, e = G.check_kweight(eng, sr, T)
        torch.cuda.synchronize()
        x = np.stack([sig[n] for n in names])[:, None].astype(np.float32)
        z64 = td.kweight_blocks64(x, sr)
        zr = td.kweight_blocks64(x, sr, filtered=td.kweight_seq32(x, td.kweight_coef(sr)))
        er = td.kweight_block_errors(zr, z64).max(-1)[:, 0] / td.U
        emit(route="kweight", rate=sr, per_signal_u={n: [round(float(a)), round(float(c))] for n, a, c in
                                                     zip(names, e[:, 0], er)},
             worst_budget_ratio=b, worst_vs_seq32=v)
    for sr in (44100, 48000):
        T = 3 * sr
        t = np.arange(T) / sr
        g = np.random.default_rng(1)
        x = np.stack([0.5 * np.sin(2 * np.pi * f * t) + 0.05 * g.standard_normal(T) for f in (20.0, 30.0, 45.0)])
        x = torch.from_numpy(x[:, None, :].astype(np.float32))
        ours = eng.lufs(x.cuda(), sr)["loud"].cpu().double()
        ref = sp.loudness(x, sr).double()
        z64 = td.kweight_blocks64(x.double().numpy(), sr)
        l64 = [G.loudness64(z64[b], sr, 1) for b in range(3)]
        emit(loudness_rate=sr, tones_hz=[20, 30, 45], ours_minus_fp32_oracle_db=(ours - ref).tolist(),
             ours_minus_float64_db=(ours.numpy() - np.array(l64)).tolist(),
             fp32_oracle_minus_float64_db=(ref.numpy() - np.array(l64)).tolist())
    # kernel time: 64 clips x 1 ch x 10 s at 44.1 kHz (the loudness stage of a batch), CUDA events over many launches
    x = (0.1 * torch.randn(64, 1, 441000)).cuda()
    for _ in range(5):
        eng.lufs(x, 44100)
    torch.cuda.synchronize()
    s, e_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(200):
        eng.lufs(x, 44100)
    e_.record()
    torch.cuda.synchronize()
    emit(lufs_call_ms_64x10s=s.elapsed_time(e_) / 200)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            eng.lufs(x, 44100)
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        if "kweight" in ev.key or "lufs_gate" in ev.key:
            emit(kernel=ev.key[:60], mean_us=ev.device_time_total / max(ev.count, 1), count=ev.count)


if __name__ == "__main__":
    main()
