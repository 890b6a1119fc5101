"""Worst error over its unit budget (tests/effects64.py) for each check of tests/test_gpu_effects_accuracy.py, with the
budget constants lifted: the table of DESIGN.md "Effect kernel accuracy".  Exact checks are asserted, not measured.
`python tests/probes/effects_accuracy_probe.py [--sim] [--json PATH]`  (--sim: the CPU-simulated kernels)."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import tests.test_gpu_effects_accuracy as G  # noqa: E402
from tests import effects64 as o  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sim", action="store_true")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if args.sim:
        from tests.cusim.sim_engine import sim_engine

        G.DEV = "cpu"
        eng = sim_engine()
    else:
        import __graft_entry__ as graft

        graft.build()
        from audiotools_b200.engine import get_engine

        eng = get_engine()
        print(torch.cuda.get_device_name(0))
    for c in ("C_Q", "C_DRR", "C_PS", "C_DCT"):
        setattr(o, c, float("inf"))
    acc = {}
    big = 10 ** 6 if args.sim else 30_000_000
    for T in (1023, 1025, 10 ** 6, big):
        row = G.rng(T).standard_normal(T).astype("float32")
        G.check_quantile(eng, row, [0.0, 0.05, 0.333, 0.5, 0.95, 1.0], acc)
    for T in G.DRR_T:
        G.check_drr(eng, G.ir_like(3, 2, T, T, peaks=[T // 3, T // 3 + 7]), 44100, [-5.0, 3.0, 12.0], acc)
    for C in (1, 2, 5):
        G.check_drr(eng, G.ir_like(7, C, 2049, 20 + C, peaks=[200 + 13 * c for c in range(C)]), 48000,
                    torch.linspace(-10, 15, 7), acc)
    G.check_drr(eng, G.ir_like(35000, 2, 300, 16, peaks=[40, 45]), 16000, torch.linspace(-6, 12, 35000), acc)
    for T in G.PS_T + [100_000]:
        g, y, x = G.ps_data(5, T, T)
        G.check_ps(eng, g, y, acc=acc, key="peak_scale limit")
        G.check_ps(eng, g, y, max_abs=0.25, acc=acc, key="peak_scale limit")
        G.check_ps(eng, g, y, x, acc=acc, key="peak_scale restore")
    for n_mfcc in G.MFCC:
        for n_mels in G.MELS:
            G.check_dct(eng, 2, n_mels, n_mfcc, 129, n_mfcc + n_mels, acc)
    G.check_dct(eng, 1, 256, 200, 130, 8, acc)
    G.check_dct(eng, 65535, 4, 3, 2, 9, acc)
    for q in G.Q_LEVELS:
        G.check_quant(eng, G.quant_inputs(q).reshape(1, 1, -1), q, True, acc)
    for k, v in sorted(acc.items()):
        print(f"{k:32s} {v:.3g}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(acc, f, indent=1)


if __name__ == "__main__":
    main()
