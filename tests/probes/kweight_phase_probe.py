"""Phase clock of the K-weighting energy kernel `kweight_energy_warp_kernel<2>` (K2) at the bench shape.

Builds a separate copy of the library with -DB2A_K2_PROBE into OUT (libb2a.so and its digest in the source tree are
not touched), runs `eng.lufs` once on bench.py's batch (64 clips x 2 ch x 10 s at 44.1 kHz) and prints, for each phase
of a 2048-sample segment, the median and p90 of the cycles lane 0 of a warp spends in it, next to the phase's static
SASS instruction count in the same build (cuobjdump).  Each warp stamps clock64() at the 7 phase boundaries of the
first 16 energy segments of its run (warm-up segments are not stamped).

  python tests/probes/kweight_phase_probe.py --out DIR [--lib DIR/libb2a.so]   (--lib: reuse a probe build)

Needs a GPU for the run; the build and the SASS count work without one.
"""
import argparse
import ctypes
import glob
import json
import os
import re
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
CSRC = os.path.join(REPO, "audiotools_b200", "csrc")
KERNEL = "kweight_energy_warp_kernelILi2E"  # the two-biquad K-weighting instantiation
PHASES = ["scan", "start states + carry", "span wait", "recursion + next map", "bin atomics", "next issue"]


def build(out):
    sys.path.insert(0, REPO)
    from audiotools_b200 import _build

    nvcc = _build._nvcc()
    flags = _build.NVCC_FLAGS + ["-DB2A_K2_PROBE"]
    os.makedirs(out, exist_ok=True)
    procs, objs = [], []
    for s in sorted(glob.glob(os.path.join(CSRC, "*.cu"))):
        o = os.path.join(out, os.path.basename(s)[:-3] + ".o")
        procs.append((s, subprocess.Popen([nvcc] + flags + ["-c", s, "-o", o], stdout=subprocess.PIPE,
                                          stderr=subprocess.STDOUT)))
        objs.append(o)
    for s, p in procs:
        msg, _ = p.communicate()
        if p.returncode:
            raise RuntimeError(f"nvcc failed on {s}:\n{msg.decode()}")
    lib = os.path.join(out, "libb2a.so")
    subprocess.check_call([nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", lib] + objs)
    return lib


def sass_phase_counts(binary):
    """Static instruction counts between consecutive clock reads of K2 in program order."""
    cuobjdump = os.path.join(os.path.dirname(os.path.realpath(subprocess.check_output(
        ["bash", "-c", "command -v nvcc || echo /usr/local/cuda/bin/nvcc"]).decode().strip())), "cuobjdump")
    if not os.path.exists(cuobjdump):
        cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    txt = subprocess.check_output([cuobjdump, "-sass", binary]).decode()
    funcs = [f for f in txt.split("Function : ")[1:] if f.split(None, 1)[0].find(KERNEL) >= 0]
    instr = [ln for ln in funcs[0].splitlines() if re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+\S", ln)]
    clocks = [i for i, ln in enumerate(instr) if "SR_CLOCKLO" in ln]
    return len(instr), [clocks[i + 1] - clocks[i] for i in range(len(clocks) - 1)], len(clocks)


def power_limit():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                                        "--format=csv,noheader"]).decode().strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--lib", default=None, help="an existing -DB2A_K2_PROBE build of libb2a.so")
    ap.add_argument("--label", default="")
    args = ap.parse_args()
    lib = args.lib or build(args.out)
    os.makedirs(args.out, exist_ok=True)
    lufs_o = os.path.join(os.path.dirname(lib), "lufs.o")
    n_instr, per_phase_instr, n_clocks = sass_phase_counts(lufs_o if os.path.exists(lufs_o) else lib)

    os.environ["B2A_LIB_PATH"] = lib
    sys.path.insert(0, REPO)
    import numpy as np
    import torch

    from audiotools_b200.engine import get_engine

    dll = ctypes.CDLL(lib)
    segs, wpb, ns = dll.b2a_k2_probe_segs(), dll.b2a_k2_probe_wpb(), dll.b2a_k2_probe_stamps()
    import bench

    eng = get_engine()
    x = bench.make_batch(64, 0, "cuda")
    target = torch.tensor([bench.TARGET_DB], device="cuda")

    def call():
        return eng.lufs(x, bench.SR, target_db=target)

    for _ in range(3):
        call()
    torch.cuda.synchronize()
    last = (ctypes.c_int * 3)()
    dll.b2a_k2_probe_last(last)
    occ, grid, smem = list(last)
    buf = torch.zeros(grid * wpb * segs * ns, dtype=torch.int64, device="cuda")
    assert dll.b2a_k2_probe_set(ctypes.c_void_p(buf.data_ptr())) == 0
    call()
    torch.cuda.synchronize()
    assert dll.b2a_k2_probe_set(ctypes.c_void_p(0)) == 0
    st = buf.view(grid, wpb, segs, ns).cpu().numpy().astype(np.int64)
    done = st[..., ns - 1] != 0  # segments the warp ran
    d = np.diff(st, axis=-1)[done]  # [n, ns - 1]
    seg_cycles = (st[..., ns - 1] - st[..., 0])[done]
    period = np.diff(st[..., 0], axis=-1)[(st[..., 1:, 0] != 0) & (st[..., :-1, 0] != 0)]  # segment-to-segment

    rows = []
    print(f"K2 phase clock {args.label}: {torch.cuda.get_device_name()} | nvidia-smi name, power limit, max SM clock: "
          f"{power_limit()}")
    print(f"occupancy {occ} CTAs/SM x {wpb} warps (cudaOccupancyMaxActiveBlocksPerMultiprocessor), grid {grid}, "
          f"dynamic smem {smem} B, {int(done.sum())} warp-segments stamped")
    if len(per_phase_instr) != len(PHASES):
        print(f"note: {n_clocks} clock reads in the SASS (expected {len(PHASES) + 1}): static counts are not split "
              "per phase")
    print(f"{'phase':<24}{'median cyc':>12}{'p90 cyc':>10}{'SASS instr':>12}")
    for i, name in enumerate(PHASES):
        med, p90 = float(np.median(d[:, i])), float(np.percentile(d[:, i], 90))
        ins = per_phase_instr[i] if len(per_phase_instr) == len(PHASES) else None
        rows.append({"phase": name, "median": med, "p90": p90, "sass": ins})
        print(f"{name:<24}{med:>12.0f}{p90:>10.0f}{'' if ins is None else ins:>12}")
    print(f"{'segment (first -> last)':<24}{np.median(seg_cycles):>12.0f}{np.percentile(seg_cycles, 90):>10.0f}"
          f"{n_instr:>12} (whole kernel)")
    print(f"{'segment period':<24}{np.median(period):>12.0f}{np.percentile(period, 90):>10.0f}")
    res = {"label": args.label, "device": torch.cuda.get_device_name(), "nvidia_smi": power_limit(),
           "occupancy": occ, "warps_per_cta": wpb, "grid": grid, "smem": smem, "phases": rows,
           "segment_median": float(np.median(seg_cycles)), "period_median": float(np.median(period)),
           "sass_total": n_instr}
    with open(os.path.join(args.out, f"k2_phase{('_' + args.label) if args.label else ''}.json"), "w") as f:
        json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
