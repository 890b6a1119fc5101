"""Times ``Engine.sos_filter`` (csrc/iir.cu, DESIGN.md K19) on the GPU, with CUDA events, against
``torchaudio.functional.lfilter`` on the GPU and ``scipy.signal.sosfilt`` on the CPU on the same input.

Shapes: 64 x 2 x 10 s at 44.1 kHz with S = 1, 4 and 8 cookbook sections, and 8 x 2 x 1 h at 48 kHz with S = 4.  The
compulsory traffic is 12 B per sample (x read twice, y written once); the ratio to its time at 3.35 TB/s is printed.
Each measurement is repeated ``--repeats`` times to show the spread; ``--out`` also writes the results as JSON.
`python tests/probes/iir_probe.py [--repeats 5] [--no-compare] [--out results.json]`"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
import __graft_entry__ as graft  # noqa: E402

HBM = 3.35e12


def cookbook_sos(S, sr, seed=0):
    from tests import iir64

    rng = np.random.default_rng(seed)
    kinds = ("peaking", "low_shelf", "high_shelf", "peaking")
    return np.stack([iir64.cookbook(kinds[s % 4], float(rng.uniform(40, 8000)), float(rng.uniform(-12, 12)),
                                    float(rng.uniform(0.5, 4)), sr) for s in range(S)])


def time_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-compare", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    graft.build()
    from audiotools_b200.engine import get_engine

    eng = get_engine()
    dev = "cuda:0"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "runs": []}
    for B, C, sr, secs, Ss, iters in ((64, 2, 44100, 10, (1, 4, 8), 20), (8, 2, 48000, 3600, (4,), 3)):
        T = int(sr * secs)
        x = (0.1 * torch.randn(B, C, T, device=dev))
        for S in Ss:
            sos = torch.from_numpy(cookbook_sos(S, sr)).to(dev)
            out = torch.empty_like(x)
            ms = [time_ms(lambda: eng.sos_filter(x, sos, out=out), iters) for _ in range(args.repeats)]
            floor = 12 * x.numel() / HBM * 1e3
            row = {"shape": [B, C, T], "sr": sr, "S": S, "ms": ms, "floor_ms": floor,
                   "ratio_median": float(np.median(ms) / floor)}
            print(json.dumps(row), flush=True)
            res["runs"].append(row)
        del x
        torch.cuda.empty_cache()
    if not args.no_compare:
        B, C, sr, S = 64, 2, 44100, 4
        T = sr * 10
        x = 0.1 * torch.randn(B, C, T, device=dev)
        sos = cookbook_sos(S, sr)
        try:
            import torchaudio.functional as AF

            def ta():
                y = x
                for s in range(S):
                    b = torch.tensor(sos[s, :3] / sos[s, 3], device=dev, dtype=torch.float32)
                    a = torch.tensor(sos[s, 3:] / sos[s, 3], device=dev, dtype=torch.float32)
                    y = AF.lfilter(y, a, b, clamp=False)
                return y

            res["torchaudio_lfilter_ms"] = time_ms(ta, 2)
        except Exception as e:  # torchaudio may be missing
            res["torchaudio_lfilter_ms"] = f"not measured: {type(e).__name__}: {e}"
        from scipy import signal as sps

        xc = x.cpu().numpy()
        t0 = time.perf_counter()
        sps.sosfilt((sos / sos[:, 3:4]).astype(np.float32), xc, axis=-1)
        res["scipy_sosfilt_cpu_ms"] = (time.perf_counter() - t0) * 1e3
        print(json.dumps({k: v for k, v in res.items() if k != "runs"}), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
