"""Accuracy table of the spectral masks and the spectral gate against float64 (DESIGN.md "Spectral mask accuracy"): per
check group of tests/test_gpu_specmask_accuracy.py, the worst error of each stage in its budget units
(tests/specmask64.py), with the budgets switched off so the numbers are measured, not checked.  Prints JSON lines, with
the GPU's name and power limit read in the same call.  ``--sim`` runs the same groups, at the simulator's sizes, on the
CPU-simulated build.

    python tests/probes/specmask_accuracy_probe.py [--sim]
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
    import torch

    from audiotools_b200.ml.layers.spectral_gate import _ramp
    from tests import specmask64 as s
    from tests import test_gpu_specmask_accuracy as G

    if sim:
        from tests.cusim.sim_engine import sim_engine

        eng = sim_engine()
        G.DEV = "cpu"
        emit(gpu="CPU simulator")
    else:
        import __graft_entry__ as graft

        graft.build()
        from audiotools_b200.engine import get_engine

        eng = get_engine()
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip()
        emit(gpu=smi)
    for k in ("C_ROT", "C_KEEP", "C_MLBWD", "C_TH", "C_S", "C_OUT"):
        setattr(s, k, 1e30)
    total = {}

    def row(group, acc):
        emit(group=group, **{k: float(f"{v:.4g}") for k, v in sorted(acc.items())})
        for k, v in acc.items():
            total[k] = max(total.get(k, 0.0), v)

    acc = {}
    for shape, per_cell, smax in G.ROTATE_CASES:
        G.check_rotate(eng, shape, per_cell, smax, acc=acc)
    row("rotate", acc)
    acc = {}
    shapes = [(2, 1, 33, 70), (3, 2, 17, 65)] + ([] if sim else [(3, 1, 513, 400)])
    for shape in shapes:
        G.check_mask_low(eng, G.ramped(shape, 1 + shape[-1]), torch.linspace(-60.0, -20.0, shape[0]), 0.5, shape,
                         acc=acc)
    X, two = G.margin_cells((1, 1, 33, 70), -30.0, 5)
    G.check_mask_low(eng, X, [-30.0], 0.5, "margin", acc=acc, max_undecided=0.06, must_decide=two)
    row("mask_low", acc)
    acc = {}
    Fs, Ns = ([1, 16, 17, 33], [1, 64, 65, 130]) if sim else (G.F_EDGES, G.N_EDGES)
    for F in Fs:
        for N in Ns:
            G.gate_case(eng, 2, 2, F, N, (1, 1, F, 50), F + N, hf=3, ht=5, acc=acc)
    row("gate tiles", acc)
    acc = {}
    for hf in G.HALVES:
        for ht in G.HALVES:
            G.gate_case(eng, 2, 1, 17, 65, (1, 1, 17, 50), 3 * hf + ht + 17, hf=hf, ht=ht, acc=acc)
    G.gate_case(eng, 2, 2, 33, 130, (1, 1, 33, 50), 21, sf=G.ASYM_F, st=G.ASYM_T, acc=acc)
    row("gate smoothing widths", acc)
    acc = {}
    for nz_N in G.NZ_FRAMES:
        G.gate_case(eng, 2, 2, 33, 130, (2, 2, 33, nz_N), 40 + nz_N, n_std=1.5, acc=acc)
    for nz_shape in [(1, 1), (3, 1), (1, 2), (3, 2)]:
        G.gate_case(eng, 3, 2, 17, 65, nz_shape + (17, 50), 31, amount=(1.0, 0.3, 0.8), acc=acc)
    row("gate noise", acc)
    acc = {}
    for where, value in G.NONFINITE:
        G.check_gate_nonfinite(eng, where, value, acc=acc)
    row("gate non-finite", acc)
    if not sim:
        acc = {}
        G.check_gate(eng, G.gate_signal(65535, 1, 3, 5, 90), G.gate_noise((1, 1, 3, 50), 91), 1.0, 0.8,
                     _ramp(1).tolist(), _ramp(2).tolist(), "65535 rows", acc=acc, max_undecided=2e-3)
        row("gate 65535 rows", acc)
    emit(group="worst", **{k: float(f"{v:.4g}") for k, v in sorted(total.items())})


if __name__ == "__main__":
    main()
