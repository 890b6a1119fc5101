"""Times ``Engine.sos_filtfilt`` and its backward (csrc/iir.cu, DESIGN.md K19) against one ``sos_filter`` pass on the
GPU with CUDA events, and optionally compares ``sos_filter`` bit for bit with another build of libb2a (the parent
commit's) on seeded inputs for S = 1 .. 8, forwards and backwards, with and without a gain.

Shapes: 64 x 2 x 10 s at 44.1 kHz with S = 1, 4 and 8 cookbook sections, and 8 x 2 x 1 h at 48 kHz with S = 4.  Each
time is the mean of back-to-back calls, repeated ``--repeats`` times to show the spread; with ``--parent`` the parent
build's ``sos_filter`` is timed too, alternating with this build's.  The GPU's name and power limit are read in the
same run.  Prints JSON lines; exits 1 when an output differs.
`python tests/probes/iir_state_probe.py [--parent LIB] [--repeats 3] [--out results.json]`"""
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
from tests.probes.iir_probe import cookbook_sos, time_ms  # noqa: E402


def parity(eng, ref, dev):
    """sos_filter of this build against ``ref``'s on seeded inputs: the number of calls that differ."""
    from tests import test_gpu_iir as G

    bad = 0
    rng = np.random.default_rng(0)
    for S in range(1, 9):
        for T in (1, 1000, 1024, 1025, 33 * 1024 + 7, 441000):
            x = torch.from_numpy(G.make_batch(rng, 48000, 2, T)).to(dev)
            sos = G.random_sos(rng, 48000, S, x.shape[0])
            gain = torch.from_numpy(rng.uniform(0.25, 4.0, x.shape[0]).astype(np.float32)).to(dev)
            for kw in ({}, {"reverse": True}, {"gain": gain}):
                a, b = eng.sos_filter(x, sos, **kw), ref.sos_filter(x, sos, **kw)
                same = torch.equal(a.view(torch.int32), b.view(torch.int32))  # bit for bit, NaN payloads included
                bad += not same
    return bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default=None, help="another build of libb2a.so to compare sos_filter with")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    graft.build()
    from audiotools_b200 import _lib
    from audiotools_b200.engine import Engine, get_engine

    eng = get_engine()
    dev = "cuda:0"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "runs": []}
    ref = None
    if args.parent:  # an older build lacks this change's entry points: bind only the symbols it exports
        import ctypes

        exported = ctypes.CDLL(args.parent)
        full = dict(_lib.SIGNATURES)
        _lib.SIGNATURES = {k: v for k, v in full.items() if hasattr(exported, k)}
        try:
            ref = Engine(_lib.B2ALibrary(args.parent))
        finally:
            _lib.SIGNATURES = full
    if ref is not None:
        res["parity_calls_differing"] = parity(eng, ref, dev)
        print(json.dumps({"gpu": smi, "parity_calls_differing": res["parity_calls_differing"]}), flush=True)
    for B, C, sr, secs, Ss, iters in ((64, 2, 44100, 10, (1, 4, 8), 20), (8, 2, 48000, 3600, (4,), 3)):
        T = int(sr * secs)
        x = 0.1 * torch.randn(B, C, T, device=dev)
        out = torch.empty_like(x)
        for S in Ss:
            sos = torch.from_numpy(cookbook_sos(S, sr)).to(dev)
            row = {"shape": [B, C, T], "sr": sr, "S": S, "sos_filter_ms": [], "sosfiltfilt_ms": [],
                   "backward_ms": []}
            if ref is not None:
                row["parent_sos_filter_ms"] = []
            for _ in range(args.repeats):
                row["sos_filter_ms"].append(time_ms(lambda: eng.sos_filter(x, sos, out=out), iters))
                if ref is not None:
                    row["parent_sos_filter_ms"].append(time_ms(lambda: ref.sos_filter(x, sos, out=out), iters))
                row["sosfiltfilt_ms"].append(time_ms(lambda: eng.sos_filtfilt(x, sos, out=out), iters))
                row["backward_ms"].append(time_ms(lambda: eng.sos_filtfilt_backward(x, sos), iters))
            row["filtfilt_over_one_pass"] = float(np.median(row["sosfiltfilt_ms"]) / np.median(row["sos_filter_ms"]))
            print(json.dumps(row), flush=True)
            res["runs"].append(row)
            torch.cuda.empty_cache()
        del x, out
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    sys.exit(1 if res.get("parity_calls_differing") else 0)


if __name__ == "__main__":
    main()
