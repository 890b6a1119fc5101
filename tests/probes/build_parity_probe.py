"""Compare two builds of libb2a bit for bit on the per-item element-wise effects, the true-peak meter, the limiter and
the gain pass of the LARGE / DENSE spectral routes, and optionally time the element-wise effects on both.  A change
that is meant to keep every output (a refactor) passes when build A is the parent commit's library, compiled with the
same flags, and build B the changed one.

The inputs drive both branches of the element-wise walk: 16-byte-aligned tensors and views offset by one float, and
per-item lengths of 0, 1, 2 and 3 mod 4.  They include T = 1 and the true-peak / limiter chunk length (4096) +- 1, and
an item with NaN and inf samples.

    python tests/probes/build_parity_probe.py LIB_A LIB_B [--sim] [--time] [--out result.json]

--sim: both libraries are CPU-simulator builds (tests/cusim/build_sim.py) and the tensors live on the CPU.
--time: also time gain, mix and quantize at 64 x 2 x 10 s at 44.1 kHz on the GPU, alternating the two builds, with CUDA
events (mean of --reps back-to-back calls, best of --rounds); the GPU's name and power limit are read in the same run.
Prints one JSON line; exits 1 when an output differs.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)

from audiotools_b200 import _lib  # noqa: E402
from audiotools_b200.engine import Engine  # noqa: E402

B, C, SR = 3, 2, 44100
LENGTHS = (1, 2, 3, 4, 5, 4095, 4096, 4097, 4098, 9001)
LIMIT_LENGTHS = (1, 6, 4095, 4097, 9002)
LOOKAHEADS = (0, 1, 66, 1024)  # samples
SPECTRAL = {"large": (8192, 2048, 20001), "dense": (1000, 250, 5002)}  # n_fft, hop, T


def make(T, seed):
    """[B, C, T]: a quiet, a loud and a very loud item; the second has a NaN and an inf sample."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, T, generator=g) * torch.tensor([0.05, 0.5, 1.0])[:, None, None]
    x[1, 0, T // 2] = float("nan")
    x[1, 1, T // 3] = float("inf")
    return x


def place(x, off, dev):
    """x on dev as a view `off` floats into a fresh buffer (the buffer itself is 16-byte aligned)."""
    buf = torch.zeros(x.numel() + 4, device=dev)
    v = buf[off:off + x.numel()].view(x.shape)
    v.copy_(x)
    assert v.data_ptr() % 16 == 4 * off
    return v


def outputs(eng, dev):
    """Every output of the covered entry points, by case name, on the CPU."""
    res = {}
    gains = torch.tensor([0.5, 2.0, -1.25], device=dev)
    chans = torch.tensor([8.0, 256.0, 3.0], device=dev)
    lo, hi = torch.tensor([-0.5, -1.0, -0.1], device=dev), torch.tensor([0.5, 1.0, 0.2], device=dev)
    for T in LENGTHS:
        x, o = make(T, T), make(T, T + 1)
        for off in (0, 1):
            k = f"T{T}/off{off}"
            xd, od = place(x, off, dev), place(o, off, dev)
            res[f"gain/{k}"] = eng.gain(xd, gains)
            res[f"gain_out_offset/{k}"] = eng.gain(place(x, 0, dev), gains, out=place(torch.zeros_like(x), off, dev))
            res[f"mix/{k}"] = eng.mix(xd, od)
            res[f"mix_gain/{k}"] = eng.mix(xd, od, gains)
            res[f"clamp_items/{k}"] = eng.clamp_items(xd, lo, hi)
            res[f"quantize/{k}"] = eng.quantize(xd, chans)
            res[f"quantize_mulaw/{k}"] = eng.quantize(xd, chans, mulaw=True)
            res[f"row_absmax/{k}"] = eng.row_absmax(xd)
            res[f"limit_peak/{k}"] = eng.limit_peak(xd, 0.7)
            for rate in (44100, 96000, 192000):
                tp = eng.true_peak(xd, rate)
                res[f"true_peak_rows/{rate}/{k}"], res[f"true_peak_db/{rate}/{k}"] = tp["rows"], tp["db"]
    for T in LIMIT_LENGTHS:
        x = make(T, 7 * T)
        for off in (0, 1):
            for A in LOOKAHEADS:
                k, la = f"T{T}/off{off}/A{A}", A / SR
                xd = place(x, off, dev)
                res[f"limit/{k}"], res[f"limit_reduction/{k}"] = eng.limit(xd, SR, -1.0, lookahead=la,
                                                                              want_reduction=True)
                res[f"limit_gain/{k}"] = eng.limit(xd, SR, -1.0, lookahead=la, gain=gains)
                y = place(x, off, dev)
                eng.limit(y, SR, -1.0, lookahead=la, out=y)
                res[f"limit_in_place/{k}"] = y
                y = place(x, off, dev)
                eng.limit(y, SR, -1.0, lookahead=la, gain=gains, out=y)
                res[f"limit_gain_in_place/{k}"] = y
    for name, (n_fft, hop, T) in SPECTRAL.items():
        x = make(T, n_fft).nan_to_num(0.0, 1.0, -1.0)  # finite: a NaN would fill every bin of its frames
        win = torch.hann_window(n_fft, device=dev)
        for off in (0, 1):
            xd = place(x, off, dev)
            r = eng.spectral(xd, n_fft, hop, win, gain=gains, want_scaled=True)
            res[f"spectral_{name}_stft/off{off}"] = torch.view_as_real(r["stft"])
            res[f"spectral_{name}_scaled/off{off}"] = r["scaled"]
            r = eng.spectral(xd, n_fft, hop, win, gain=gains)
            res[f"spectral_{name}_stft_ws_gain/off{off}"] = torch.view_as_real(r["stft"])
    return {k: v.detach().cpu().contiguous() for k, v in res.items()}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def time_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def timings(engines, reps, rounds):
    """gain, mix (with a gain), linear and mu-law quantize at 64 x 2 x 10 s at 44.1 kHz, the builds alternating."""
    g = torch.Generator(device="cuda").manual_seed(0)
    x = 0.1 * torch.randn(64, 2, 441000, device="cuda", generator=g)
    o = 0.1 * torch.randn(64, 2, 441000, device="cuda", generator=g)
    gains = torch.rand(64, device="cuda", generator=g) + 0.5
    chans = torch.full((64,), 256.0, device="cuda")
    ops = {"gain": lambda e: e.gain(x, gains), "mix": lambda e: e.mix(x, o, gains),
           "quantize": lambda e: e.quantize(x, chans), "quantize_mulaw": lambda e: e.quantize(x, chans, mulaw=True)}
    t = {name: {lab: [] for lab in engines} for name in ops}
    for name, f in ops.items():
        for e in engines.values():
            f(e), f(e)
        torch.cuda.synchronize()
        for _ in range(rounds):
            for lab, e in engines.items():
                t[name][lab].append(time_ms(lambda: f(e), reps))
    return {name: {lab: {"ms": min(v), "rounds": v} for lab, v in d.items()} for name, d in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("lib_a")
    ap.add_argument("lib_b")
    ap.add_argument("--sim", action="store_true")
    ap.add_argument("--time", action="store_true")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = "cpu" if args.sim else "cuda"
    assert args.sim or torch.cuda.is_available(), "without --sim this probe runs on a GPU"
    engines = {lab: Engine(_lib.B2ALibrary(p), require_cuda=not args.sim) for lab, p in
               (("a", args.lib_a), ("b", args.lib_b))}
    ra, rb = outputs(engines["a"], dev), outputs(engines["b"], dev)
    assert ra.keys() == rb.keys()
    bits = lambda t: t.view(torch.int32)  # noqa: E731  (every output is float32)
    bad = [k for k in ra if ra[k].shape != rb[k].shape or not torch.equal(bits(ra[k]), bits(rb[k]))]
    res = {"device": "cpu simulator" if args.sim else gpu_info(), "outputs": len(ra),
           "values": int(sum(v.numel() for v in ra.values())), "differ": bad}
    if args.time:
        res["timing"] = timings(engines, args.reps, args.rounds)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
