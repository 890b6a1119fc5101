"""Prints the table of DESIGN.md "Loss accuracy": for every window, mode and case of tests/test_gpu_loss_accuracy.py,
the worst kept-cell error of dL/dX and dL/dY in units of tests/loss64.py's model (ours / torch's FP32 arithmetic), each
loss term's error in the same units (ours / torch's, on the noise rows), and the cells dropped by reason.  The device
name and power limit are read in the same run.  Usage: python tests/probes/loss_accuracy_probe.py [out.md]"""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import tests.test_gpu_loss_accuracy as G  # noqa: E402
from tests import loss64 as L  # noqa: E402


def main():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    eng = get_engine()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    lines = [f"device: {q}", "",
             "| n_fft | mode | case | hop | c dL/dX ours / torch | c dL/dY ours / torch | log term ours / torch | "
             "mag term ours / torch | dropped sign / mag / clamp / zero of cells |",
             "|---|---|---|---|---|---|---|---|---|"]
    worst = {}
    for n in G.WINDOWS:
        for mode in ("stft", "mel"):
            for case in G.cases(eng, n, mode == "mel"):
                o = G.run_case(eng, n, case, G.DEV)
                lo = o["loss"]
                d = o["dropped"]
                lines.append(f"| {n} | {mode} | {case[0]} | {case[3]} | {o['c_x']:.3f} / {o['c_x_torch']:.3f} | "
                             f"{o['c_y']:.3f} / {o['c_y_torch']:.3f} | {lo['log'][0]:.1e} ({lo['log'][1]:.1e} / "
                             f"{lo['log'][2]:.1e}) | {lo['mag'][0]:.1e} ({lo['mag'][1]:.1e} / {lo['mag'][2]:.1e}) | "
                             f"{d['sign']} / {d['mag']} / {d['clamp']} / {d['zero']} of {o['cells']} |")
                for k, v in (("cell", max(o["c_x"], o["c_y"])), ("loss", max(lo["log"][0], lo["mag"][0]))):
                    key = (k, mode)
                    worst[key] = max(worst.get(key, 0.0), v)
                print(lines[-1], flush=True)
    lines += ["", "worst: " + ", ".join(f"{k[0]} {k[1]} {v:.3f}" for k, v in sorted(worst.items())),
              f"device: {q}"]
    text = "\n".join(lines)
    print(text)
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        with open(sys.argv[1], "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
