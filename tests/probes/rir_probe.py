"""Times ``core.room.image_source_ir`` (csrc/rir.cu, DESIGN.md K20) on the GPU with CUDA events, for the rooms below at
B = 64 items with C = 1 and 2 microphones, without the high-pass (the image sum alone), and reports taps per second:
the oracle's image count (tests/rir64.py, enumerated on the CPU) times the window Tw, per IR.  For comparison, one IR's
taps are scattered on the GPU with torch ``index_add_`` (indices and values precomputed, only the scatter timed), and
the float64 oracle renders one IR on the CPU (first two rooms only).  The GPU's name and power limit are read in the
same run.  Prints JSON lines.
`python tests/probes/rir_probe.py [--repeats 3] [--out results.json]`"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
import __graft_entry__ as graft  # noqa: E402
from tests import rir64  # noqa: E402

# (room, source, microphone, fs, seconds)
ROOMS = [([5.0, 4.0, 3.0], [1.0, 1.0, 1.5], [3.0, 2.5, 1.2], 16000, 0.5),
         ([6.0, 5.0, 3.0], [1.0, 1.0, 1.5], [4.0, 3.0, 1.2], 48000, 0.5),
         ([10.0, 8.0, 4.0], [2.0, 2.0, 1.5], [7.0, 5.0, 1.2], 44100, 1.0),
         ([4.0, 3.0, 2.5], [1.0, 1.0, 1.2], [3.0, 2.0, 1.5], 48000, 1.0)]
BETA = 0.9


def events_ms(fn, n):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(n):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / n


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
    B = 64
    for i, (room, src, mic, fs, secs) in enumerate(ROOMS):
        L = int(secs * fs)
        Tw = rir64.window(fs)
        d, g, o = rir64.images(room, src, mic, np.full(6, BETA), fs, L)
        taps = len(d) * Tw
        row = {"room": room, "fs": fs, "L": L, "images": len(d), "images_order_le_20": int((o <= 20).sum()),
               "taps_per_ir": taps}
        for C in (1, 2):
            mics = [mic] if C == 1 else [mic, [mic[0] - 0.1, mic[1], mic[2]]]
            call = lambda: image_source_ir(room, src, mics, fs, L, beta=np.full(6, BETA), high_pass=False,  # noqa
                                           device=dev)
            call()
            torch.cuda.synchronize()
            n = 1 if taps * B * C > 2e10 else 3
            ms = [events_ms(call, n) for _ in range(args.repeats)]
            row[f"C{C}_ms"] = ms
            row[f"C{C}_taps_per_s"] = taps * B * C / (min(ms) * 1e-3)
        if taps <= 2.5e8:  # a scatter of one IR's taps with torch, for comparison
            n = np.arange(Tw)
            fl = np.floor(d)
            idx = (fl[:, None] - Tw // 2 + 1 + n)
            f = (d - fl)[:, None]
            h = 0.5 * (1 - np.cos(2 * math.pi * (n + 1 - f) / Tw)) * np.sinc(n + 1 - f - Tw / 2) * g[:, None]
            ok = (idx >= 0) & (idx < L)
            it = torch.from_numpy(idx[ok].astype(np.int64)).to(dev)
            vt = torch.from_numpy(h[ok].astype(np.float32)).to(dev)
            del idx, h, f, ok
            out = torch.zeros(L, device=dev)
            row["torch_index_add_one_ir_ms"] = min(events_ms(lambda: out.zero_().index_add_(0, it, vt), 3)
                                                   for _ in range(args.repeats))
            del it, vt
        if i < 2:
            t0 = time.perf_counter()
            rir64.render(d, g, Tw, L)
            row["oracle_cpu_one_ir_s"] = time.perf_counter() - t0
        res["runs"].append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
