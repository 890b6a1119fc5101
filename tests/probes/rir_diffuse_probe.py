"""Times ``core.room.image_source_ir`` with and without the diffuse tail (csrc/rir.cu, DESIGN.md K20 "Hybrid") on the
GPU with CUDA events: K20's four rooms at B = 64 items, C = 1, beta = 0.9 on every wall, no high-pass, images only
against ``diffuse_after=0.05``.  A second pass under ``torch.profiler`` splits the hybrid's time between the image
kernel and the tail kernel.  The GPU's name and power limit are read in the same run.  Prints JSON lines.
`python tests/probes/rir_diffuse_probe.py [--repeats 3] [--out results.json]`"""
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
from tests.probes.rir_probe import BETA, ROOMS, events_ms  # noqa: E402

B, TD = 64, 0.05


def kernel_ms(fn, n=3):
    """Mean GPU time per call of each kernel fn launches, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and "rir" in e.key:
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
    for room, src, mic, fs, secs in ROOMS:
        L = int(secs * fs)
        row = {"room": room, "fs": fs, "L": L, "B": B}
        for name, tail in (("images_ms", {}), ("hybrid_ms", dict(diffuse_after=TD, seed=np.arange(B)))):
            call = lambda tail=tail: image_source_ir([room] * B, src, [mic], fs, L, beta=np.full(6, BETA),  # noqa
                                                     high_pass=False, device=dev, **tail)
            call()
            torch.cuda.synchronize()
            n = 1 if not tail and L > 40000 else 5
            row[name] = [events_ms(call, n) for _ in range(args.repeats)]
            if tail:
                row["hybrid_kernels_ms"] = kernel_ms(call)
        res["runs"].append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
