"""Accuracy table of STOI and its backward against float64 (DESIGN.md "STOI accuracy"): per check group of
tests/test_gpu_stoi_accuracy.py, the worst error of each stage in its budget units (tests/stoi64.py), with the budgets
switched off so the numbers are measured, not checked.  Prints JSON lines, with the GPU's name and power limit read in
the same call.  ``--sim`` runs the same groups, at the simulator's sizes, on the CPU-simulated build.

    python tests/probes/stoi_accuracy_probe.py [--sim]
"""
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)


def emit(**kw):
    print(json.dumps(kw), flush=True)


def main():
    sim = "--sim" in sys.argv
    import audiotools_b200.engine as engine_mod
    from tests import stoi64 as s
    from tests import test_gpu_stoi_accuracy as G

    if sim:
        from tests.cusim.sim_engine import sim_engine

        eng = engine_mod._ENGINE = sim_engine()
        G.DEV = "cpu"
        emit(gpu="CPU simulator")
    else:
        import __graft_entry__ as graft

        graft.build()
        eng = engine_mod.get_engine()
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip()
        emit(gpu=smi)
    for k in ("RESAMPLE_ULP", "ENERGY_DB", "C_B", "F_B", "SCORE_ABS", "C_G", "C_H", "C_Y", "C_X"):
        setattr(s, k, 1e30)
    total = {}

    def row(group, acc):
        emit(group=group, **{k: float(f"{v:.4g}") for k, v in sorted(acc.items())})
        for k, v in acc.items():
            total[k] = max(total.get(k, 0.0), v)

    rates = [8000, 10000, 12345, 22050, 44100, 96000] if sim else s.RATES + [7999]
    for sr in rates:
        row(f"rate {sr}", G.check_rate(eng, sr, 0.8 if sim else 2.0))
    for sr in ([8000, 10000, 7999] if sim else [8000, 10000, 12345, 44100, 192000, 7999]):
        row(f"resampler tiles {sr}", G.check_resampler_tiles(eng, sr))
    for sr in ([8000] if sim else [8000, 16000, 44100]):
        row(f"input tiles {sr}", G.check_input_tiles(eng, sr))
    for n_fr in [1, 2, 255, 256, 257, 512, 513]:
        row(f"mask n_fr={n_fr}", G.check_mask_chunks(eng, n_fr))
    acc = {}
    for M in G.M_EDGES if not sim else [0, 1, 29, 30, 31, 32, 33, 46, 47, 36, 38, 64, 65]:
        G.check_m(eng, M, acc)
    row("band / score M edges", acc)
    emit(group="worst", **{k: float(f"{v:.4g}") for k, v in sorted(total.items())})


if __name__ == "__main__":
    main()
