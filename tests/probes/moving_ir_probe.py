"""Times the moving impulse response (DESIGN.md K22) on the GPU with CUDA events, at 64 items x 2 channels x 10 s at
44.1 kHz, 1 s responses, a waypoint every 0.05 s (200 waypoints): the hybrid room responses for all B K waypoints
(``image_source_ir``, one call), the path convolution (``Engine.circular_convolve_moving``: spectra and convolution),
and a static ``circular_convolve`` of the first waypoints, the cost of ``apply_ir``'s convolution.  A second pass
under ``torch.profiler`` splits the path convolution by kernel.  Peak memory, the GPU's name and power limit are read
in the same run.  Prints JSON lines.
`python tests/probes/moving_ir_probe.py [--repeats 3] [--out results.json]`"""
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

B, C, SR, SECONDS, IR_SECONDS, HOP_S = 64, 2, 44100, 10.0, 1.0, 0.05


def kernel_ms(fn, n=2):
    """Mean GPU time per call of each kernel fn launches, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA":
            out[e.key.split("(")[0][:80]] = round(e.device_time_total / 1e3 / n, 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    graft.build()
    from audiotools_b200.core.room import image_source_ir
    from audiotools_b200.engine import get_engine

    dev = "cuda:0"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    eng = get_engine()
    T, L, hop = int(SECONDS * SR), int(IR_SECONDS * SR), int(round(HOP_S * SR))
    K = (T - 1) // hop + 1
    rng = np.random.default_rng(0)
    room = np.array([8.0, 6.0, 3.0])
    start, end = rng.uniform(0.5, room - 0.5, (B, 3)), rng.uniform(0.5, room - 0.5, (B, 3))
    src = start[:, None] + np.linspace(0, 1, K)[None, :, None] * (end - start)[:, None]  # [B, K, 3]
    mics = np.array([[3.9, 3.0, 1.5], [4.1, 3.0, 1.5]])
    seed = np.repeat(np.arange(B), K)

    def gen():
        return image_source_ir(room, src.reshape(-1, 3), mics, SR, L, rt60=0.6, diffuse_after=0.05, seed=seed,
                               device=dev).audio_data

    x = 0.1 * torch.randn(B, C, T, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    irs = gen().reshape(B, K, C, L)
    ir0 = irs[:, 0].contiguous()

    def moving():
        return eng.circular_convolve_moving(x, irs, hop)

    def static():
        return eng.circular_convolve(x, ir0)

    for fn in (gen, moving, static):  # warm every shape
        fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    moving()
    torch.cuda.synchronize()
    peak_conv = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    rows = []
    for rep in range(args.repeats):
        rows.append({"rep": rep, "ir_generation_ms": round(events_ms(gen, 3), 3),
                     "moving_convolution_ms": round(events_ms(moving, 5), 3),
                     "static_convolution_ms": round(events_ms(static, 5), 3)})
        print(json.dumps(rows[-1]), flush=True)
    kern = kernel_ms(moving)
    res = {"gpu": smi, "B": B, "C": C, "T": T, "L": L, "hop": hop, "K": K,
           "irs_GB": round(irs.numel() * 4 / 2 ** 30, 3),
           "moving_convolution_peak_extra_MB": round(peak_conv, 1),
           "median": {k: float(np.median([r[k] for r in rows])) for k in rows[0] if k != "rep"},
           "moving_kernels_ms": kern}
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"runs": rows, "summary": res}, f, indent=1)


if __name__ == "__main__":
    main()
