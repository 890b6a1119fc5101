"""Time ``Engine.limit`` (csrc/limiter.cu) with CUDA events at the bench shape (64 x 2 x 10 s at 44.1 kHz) with none,
about 1 % and all of the chunks limited, and at a long-form shape (8 x 2 x 1 h at 48 kHz), against the time the
compulsory traffic (read x, write out: 8 C bytes per item-sample) takes at 3.35 TB/s, the H100 SXM data sheet's HBM
figure for a 700 W card.  The bytes the three launches move are counted from the shape: 4 C + 4 (envelope and hold: read
x, write h) + 4 + 4 C + 4 C (release and apply: read h and x, write out) = 12 C + 8 per item-sample when every chunk is
limited; a quiet chunk still reads x twice and h once and writes out.  Prints one JSON line with the GPU's name, power
limit and SM clock limit, read in the same run.  Without a GPU it fails.

    python tests/probes/limiter_probe.py [--reps 200] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)

CHUNK = 4096
HBM_BPS = 3.35e12
CASES = {  # name: (B, C, T, rate, share of the chunks with an over)
    "bench_0pct": (64, 2, 441000, 44100, 0.0),
    "bench_1pct": (64, 2, 441000, 44100, 0.01),
    "bench_100pct": (64, 2, 441000, 44100, 1.0),
    "long_1pct": (8, 2, 3600 * 48000, 48000, 0.01),
}


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


def make(B, C, T, share):
    """Noise well under the ceiling, with one 1.5-amplitude click in ``share`` of the (item, chunk) pairs."""
    g = torch.Generator(device="cuda").manual_seed(0)
    x = 0.05 * torch.randn(B, C, T, device="cuda", generator=g)
    n_chunks = (T + CHUNK - 1) // CHUNK
    if share > 0:
        pick = torch.rand(B, n_chunks, device="cuda", generator=g) < share
        b, k = pick.nonzero(as_tuple=True)
        pos = (k * CHUNK + CHUNK // 2).clamp(max=T - 1)
        x[b, 0, pos] = 1.5
    return x


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
    res = {"gpu": gpu_info(), "reps": args.reps, "cases": {}}
    for name, (B, C, T, sr, share) in CASES.items():
        x = make(B, C, T, share)
        out = torch.empty_like(x)
        reps = args.reps if name.startswith("bench") else max(args.reps // 10, 5)

        def kernel():
            eng.limit(x, sr, -1.0, out=out)

        kernel()
        kernel()
        torch.cuda.synchronize()
        _, red = eng.limit(x, sr, -1.0, want_reduction=True)
        limited = float((red.view(B, -1)[:, : T // CHUNK * CHUNK].view(B, -1, CHUNK).amax(-1) > 0).float().mean())
        del red
        t = [time_ms(kernel, reps) for _ in range(args.rounds)]
        n = B * T
        compulsory, moved = 8.0 * C * n, (12.0 * C + 8) * n
        k = min(t)
        res["cases"][name] = {"B": B, "C": C, "T": T, "rate": sr, "chunks_limited": limited, "limit_ms": k,
                              "limit_ms_rounds": t, "compulsory_bytes": compulsory, "moved_bytes": moved,
                              "compulsory_ms": compulsory / HBM_BPS * 1e3,
                              "limit_over_compulsory": k / (compulsory / HBM_BPS * 1e3),
                              "achieved_TBps_moved": moved / (k * 1e-3) / 1e12}
        del x, out
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
