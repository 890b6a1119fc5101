"""Time ``Engine.true_peak`` (csrc/truepeak.cu) with CUDA events at the bench shape (64 x 2 x 10 s at 44.1 kHz) and a
long-form shape (8 x 2 x 1 h at 48 kHz), against the two floors computed from the shape (HBM: 4 bytes read per sample
at 3.35 TB/s; FP32: 3 (L - 1) x 12 FMA = 2 x 36 FLOP per sample at 67 TFLOP/s, the H100 SXM data sheet's figures for a
700 W card) and against a torch ``conv1d`` polyphase of the same taps on the same GPU (one conv1d with L - 1 output
channels and the max of |.| over all of it, the instant rules aside).  Prints one JSON line with the GPU's name, power
limit and SM clock limit, read in the same run.

    python tests/probes/true_peak_probe.py [--reps 200] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)

SHAPES = {"bench": (64, 2, 441000, 44100), "long": (8, 2, 3600 * 48000, 48000)}
HBM_BPS = 3.35e12
FP32_FLOPS = 67e12


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def time_ms(fn, reps):
    """Mean time of one call over ``reps`` back-to-back calls between two events."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this probe measures on a GPU"
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    eng = get_engine()
    res = {"gpu": gpu_info(), "reps": args.reps, "shapes": {}}
    for name, (B, C, T, sr) in SHAPES.items():
        g = torch.Generator(device="cuda").manual_seed(0)
        x = 0.1 * torch.randn(B, C, T, device="cuda", generator=g)
        L = int(eng.lib.b2a_true_peak_factor(float(sr)))
        taps = torch.from_numpy(eng.true_peak_taps(sr)).cuda()
        w = taps.flip(-1)[:, None, :]  # conv1d correlates: y[n] = sum_m w[m] x[n - 6 + m] = sum_d h[d] x[n - d]
        xr = x.view(B * C, 1, T)

        def kernel():
            eng.true_peak(x, sr)

        def torch_conv():
            y = torch.nn.functional.conv1d(xr, w, padding=6)
            return torch.maximum(y.abs().amax(dim=(1, 2)), xr.abs().amax(dim=(1, 2)))

        with_conv = name == "bench"  # the long shape's conv1d output alone would take 33 GB
        for f in (kernel, torch_conv, kernel, torch_conv) if with_conv else (kernel, kernel):  # warm-up
            f()
        torch.cuda.synchronize()
        t_k, t_t = [], []
        for _ in range(args.rounds):  # alternate the two
            t_k.append(time_ms(kernel, args.reps))
            if with_conv:
                t_t.append(time_ms(torch_conv, max(args.reps // 10, 5)))
        n = B * C * T
        hbm_ms = 4.0 * n / HBM_BPS * 1e3
        fma_ms = 2.0 * 12 * (L - 1) * n / FP32_FLOPS * 1e3
        k = min(t_k)
        res["shapes"][name] = {"B": B, "C": C, "T": T, "rate": sr, "L": L, "bytes": 4 * n,
                               "kernel_ms": k, "kernel_ms_rounds": t_k, "hbm_floor_ms": hbm_ms, "fp32_floor_ms": fma_ms,
                               "kernel_over_larger_floor": k / max(hbm_ms, fma_ms),
                               "achieved_TBps": 4.0 * n / (k * 1e-3) / 1e12,
                               "achieved_fp32_TFLOPs": 2.0 * 12 * (L - 1) * n / (k * 1e-3) / 1e12}
        if with_conv:
            ref = eng.true_peak(x, sr)["rows"].reshape(-1)
            res["shapes"][name].update(torch_conv1d_ms=min(t_t), torch_conv1d_ms_rounds=t_t,
                                       max_rel_diff_vs_conv1d=float(((ref - torch_conv()).abs() / ref).max()))
        del x, xr
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
