"""Times ``core.room.image_source_ir`` with octave bands (csrc/rir.cu, DESIGN.md K20 "Bands") on the GPU with CUDA
events, at B = 64 items, C = 1, no high-pass: for each room, the flat call (``bands=None``), ``bands=1`` and ``bands=6``
(beta 0.95 falling to 0.6 over the bands, air absorption 0 to 0.1 dB/m), images only and with ``diffuse_after=0.05``.
A second pass under ``torch.profiler`` splits the 6-band hybrid's time between its kernels.  The GPU's name and power
limit are read in the same run.  Prints JSON lines.
`python tests/probes/rir_bands_probe.py [--repeats 3] [--out results.json]`"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
import __graft_entry__ as graft  # noqa: E402
from tests.probes.rir_probe import events_ms  # noqa: E402

B, TD = 64, 0.05
ROOMS = [([5.0, 4.0, 3.0], [1.0, 1.0, 1.5], [3.0, 2.5, 1.2], 16000, 0.5),
         ([5.0, 4.0, 3.0], [1.0, 1.0, 1.5], [3.0, 2.5, 1.2], 16000, 1.0),
         ([6.0, 5.0, 3.0], [1.0, 1.0, 1.5], [4.0, 3.0, 1.2], 48000, 0.5),
         ([4.0, 3.0, 2.5], [1.0, 1.0, 1.2], [3.0, 2.0, 1.5], 48000, 1.0)]
BETA6 = np.linspace(0.95, 0.6, 6)
AIR6 = np.array([0.0, 0.001, 0.003, 0.01, 0.03, 0.1])


def kernel_ms(fn, n=3):
    """Mean GPU time per call of each kernel fn launches, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and "b2a" in e.key:
            out[e.key.split("(")[0]] = e.device_time_total / 1e3 / n
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    graft.build()
    from audiotools_b200.core.room import image_source_ir

    dev = "cuda:0"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "runs": []}
    print(json.dumps({"gpu": smi}), flush=True)
    walls = {"flat": dict(beta=np.full(6, 0.9)), "K1": dict(beta=np.full((6, 1), 0.9), bands=1),
             "K6": dict(beta=np.tile(BETA6, (6, 1)), bands=6, air_absorption=AIR6)}
    for room, src, mic, fs, secs in ROOMS:
        L = int(secs * fs)
        row = {"room": room, "fs": fs, "L": L, "B": B}
        for tname, tail in (("images", {}), ("hybrid", dict(diffuse_after=TD, seed=np.arange(B)))):
            for wname, w in walls.items():
                call = lambda tail=tail, w=w: image_source_ir([room] * B, src, [mic], fs, L, high_pass=False,  # noqa
                                                              device=dev, **w, **tail)
                call()
                torch.cuda.synchronize()
                n = 1 if not tail and L > 40000 else 5
                reps = 1 if not tail and L > 40000 else args.repeats
                row[f"{tname}_{wname}_ms"] = [events_ms(call, n) for _ in range(reps)]
                if tail and wname == "K6":
                    row["hybrid_K6_kernels_ms"] = kernel_ms(call)
        res["runs"].append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
