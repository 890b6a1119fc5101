"""Time ``metrics.LoudnessLoss`` forward + backward (``Engine.lufs(want_blocks=True)`` + ``Engine.lufs_backward``)
against ``loudness()`` alone (``Engine.lufs``) with CUDA events, alternating after warm-up, on the bench batch
(64 x 2 x 10 s at 44.1 kHz), and the backward alone.  Also prints the bytes the backward must move (x read twice, u
written, u read twice, grad_x written: 24 B per sample) and the time that takes at 3.35 TB/s -- arithmetic, not a
measurement.  One JSON line with the GPU's name and power limit, read in the same run.

    python tests/probes/loudness_grad_probe.py [--reps 30] [--out result.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)

HBM_BYTES_PER_S = 3.35e12  # H100 SXM 80 GB HBM3, the data sheet's figure
BYTES_PER_SAMPLE = 24


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def time_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from audiotools_b200.engine import get_engine

    eng = get_engine()
    B, C, T, sr = 64, 2, 441000, 44100
    g = torch.Generator(device="cuda").manual_seed(0)
    x = 0.1 * torch.randn(B, C, T, device="cuda", generator=g)
    ones = torch.ones(B, device="cuda")

    def loud():
        return eng.lufs(x, sr)

    def fwd_bwd():
        out = eng.lufs(x, sr, want_blocks=True)
        return eng.lufs_backward(ones, x, sr, out["blocks"], out["lufs"])

    out = eng.lufs(x, sr, want_blocks=True)

    def bwd():
        return eng.lufs_backward(ones, x, sr, out["blocks"], out["lufs"])

    for _ in range(5):
        loud(), fwd_bwd(), bwd()
    torch.cuda.synchronize()
    t = {"loudness": [], "forward_backward": [], "backward": []}
    for _ in range(args.reps):
        t["loudness"].append(time_ms(loud))
        t["forward_backward"].append(time_ms(fwd_bwd))
        t["backward"].append(time_ms(bwd))
    n = B * C * T
    res = {
        "gpu": gpu_info(),
        "shape": [B, C, T, sr],
        "median_ms": {k: round(statistics.median(v), 4) for k, v in t.items()},
        "min_ms": {k: round(min(v), 4) for k, v in t.items()},
        "backward_bytes": BYTES_PER_SAMPLE * n,
        "backward_hbm_floor_ms_arithmetic": round(BYTES_PER_SAMPLE * n / HBM_BYTES_PER_S * 1e3, 4),
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
