"""Time ``Engine.lufs`` (what ``AudioSignal.loudness()`` runs) against ``Engine.loudness_stats`` (``loudness_stats()``)
with CUDA events, alternating the two after warm-up, at the bench shape (64 x 2 x 10 s at 44.1 kHz) and a long-form
shape (8 x 2 x 1 h at 48 kHz, ~36 k short-term blocks per item).  Prints one JSON line with the GPU's name and power
limit, read in the same run.

    python tests/probes/loudness_stats_probe.py [--reps 20] [--out result.json]
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


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def time_ms(fn, reps):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    out = []
    for a, b in ev:
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this probe measures on a GPU"
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    eng = get_engine()
    res = {"gpu": gpu_info(), "shapes": {}}
    for name, (B, C, T, sr) in SHAPES.items():
        g = torch.Generator(device="cuda").manual_seed(0)
        x = 0.1 * torch.randn(B, C, T, device="cuda", generator=g)
        lufs = lambda: eng.lufs(x, sr)  # noqa: E731
        stats = lambda: eng.loudness_stats(x, sr)  # noqa: E731
        for f in (lufs, stats, lufs, stats):  # warm-up
            f()
        torch.cuda.synchronize()
        t_l, t_s = [], []
        for _ in range(args.rounds):  # alternate the two
            t_l += time_ms(lufs, args.reps)
            t_s += time_ms(stats, args.reps)
        med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
        st = eng.loudness_stats(x, sr)
        same = bool(torch.equal(st["I"], eng.lufs(x, sr)["lufs"]))
        res["shapes"][name] = {"B": B, "C": C, "T": T, "rate": sr,
                               "n_short_term": int(eng.lib.b2a_loudness_stats_num_short_term(T, float(sr))),
                               "lufs_ms_median": med(t_l), "lufs_ms_min": min(t_l),
                               "stats_ms_median": med(t_s), "stats_ms_min": min(t_s),
                               "ratio_median": med(t_s) / med(t_l), "I_bit_identical": same,
                               "LRA_item0": st["LRA"][0].item()}
        del x
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
