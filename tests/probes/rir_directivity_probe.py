"""Times ``core.room.image_source_ir`` with and without directivity (csrc/rir.cu, DESIGN.md K20 "Directivity") on the
GPU with CUDA events: K20's four rooms at B = 64 items, C = 1, beta = 0.9 on every wall, no high-pass, images only and
``diffuse_after=0.05``; directional means a cardioid microphone and a hypercardioid source with random orientations per
item.  The two variants are timed in the same run, alternated, ``--repeats`` times each.  The GPU's name and power
limit are read in the same run.  Prints JSON lines.  Timing only, not a test.
`python tests/probes/rir_directivity_probe.py [--repeats 3] [--out results.json]`"""
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
    rng = np.random.default_rng(0)
    mo = rng.standard_normal((B, 1, 3))
    so = rng.standard_normal((B, 3))
    directional = dict(mic_pattern="cardioid", mic_orientation=mo, source_pattern="hypercardioid",
                       source_orientation=so)
    for room, src, mic, fs, secs in ROOMS:
        L = int(secs * fs)
        for kind, tail in (("images", {}), ("hybrid", dict(diffuse_after=TD, seed=np.arange(B)))):
            row = {"room": room, "fs": fs, "L": L, "B": B, "kind": kind, "plain_ms": [], "directional_ms": []}
            calls = {}
            for name, d in (("plain_ms", {}), ("directional_ms", directional)):
                calls[name] = lambda tail=tail, d=d: image_source_ir(  # noqa: E731
                    [room] * B, src, [mic], fs, L, beta=np.full(6, BETA), high_pass=False, device=dev, **tail, **d)
                calls[name]()
            torch.cuda.synchronize()
            n = 1 if not tail and L > 40000 else 5
            for _ in range(args.repeats):
                for name in ("plain_ms", "directional_ms"):
                    row[name].append(events_ms(calls[name], n))
            row["ratio"] = float(np.median(row["directional_ms"]) / np.median(row["plain_ms"]))
            res["runs"].append(row)
            print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
