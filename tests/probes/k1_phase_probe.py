"""Phase clock of the fused log-mel kernel `spectral_warp_kernel<10,0>` (K1) at the bench shape.

Builds a separate copy of the library with -DB2A_K1_PROBE into OUT (libb2a.so and its digest in the source tree are
not touched), runs bench.py's step once (64 clips x 2 ch x 10 s: LUFS-normalise, then log-mel 2048 / 512 / 128) and
prints, for each phase of a tile, the median and p90 of the cycles lane 0 of a warp spends in it, next to the phase's
static SASS instruction count in the same build (cuobjdump).  Each warp stamps clock64() at the 11 phase boundaries of
its first 64 tiles.

  python tests/probes/k1_phase_probe.py --out DIR [--lib DIR/libb2a.so]   (--lib: reuse a probe build)

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
KERNEL = "_ZN3b2a8spectral20spectral_warp_kernelILi10ELi0EEEvNS0_6ParamsE"
PHASES = ["span wait", "barrier", "writeback", "frame load", "barrier + TMA issue", "FFT + untangle",
          "barrier", "mel (+ store)", "barrier", "store"]


def build(out):
    sys.path.insert(0, REPO)
    from audiotools_b200 import _build

    nvcc = _build._nvcc()
    flags = _build.NVCC_FLAGS + ["-DB2A_K1_PROBE"]
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
    """Static instruction counts between consecutive clock reads of K1 in program order."""
    cuobjdump = os.path.join(os.path.dirname(os.path.realpath(subprocess.check_output(
        ["bash", "-c", "command -v nvcc || echo /usr/local/cuda/bin/nvcc"]).decode().strip())), "cuobjdump")
    if not os.path.exists(cuobjdump):
        cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    txt = subprocess.check_output([cuobjdump, "-sass", "-fun", KERNEL, binary]).decode()
    instr = [ln for ln in txt.splitlines() if re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+\S", ln)]
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
    ap.add_argument("--lib", default=None, help="an existing -DB2A_K1_PROBE build of libb2a.so")
    ap.add_argument("--label", default="")
    args = ap.parse_args()
    lib = args.lib or build(args.out)
    os.makedirs(args.out, exist_ok=True)
    spectral_o = os.path.join(os.path.dirname(lib), "spectral.o")
    n_instr, per_phase_instr, n_clocks = sass_phase_counts(spectral_o if os.path.exists(spectral_o) else lib)

    os.environ["B2A_LIB_PATH"] = lib
    sys.path.insert(0, REPO)
    import numpy as np
    import torch

    from audiotools_b200 import AudioSignal

    dll = ctypes.CDLL(lib)
    tiles = dll.b2a_k1_probe_tiles()
    sys.path.insert(0, REPO)
    import bench

    x = bench.make_batch(64, 0, "cuda")

    def step():
        sig = AudioSignal(x, bench.SR)
        sig.normalize(bench.TARGET_DB)
        return sig.mel_spectrogram(n_mels=bench.N_MELS, window_length=bench.N_FFT, hop_length=bench.HOP,
                                   window_type="hann", log=True)

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    last = (ctypes.c_int * 3)()
    dll.b2a_k1_probe_last(last)
    occ, grid, smem = list(last)
    buf = torch.zeros(grid * 8 * tiles * 11, dtype=torch.int64, device="cuda")
    assert dll.b2a_k1_probe_set(ctypes.c_void_p(buf.data_ptr())) == 0
    step()
    torch.cuda.synchronize()
    assert dll.b2a_k1_probe_set(ctypes.c_void_p(0)) == 0
    st = buf.view(grid, 8, tiles, 11).cpu().numpy().astype(np.int64)
    done = st[..., 10] != 0  # tiles the CTA ran (a CTA runs ceil(total / grid) or one fewer)
    d = np.diff(st, axis=-1)[done]  # [n, 10]
    tile_cycles = (st[..., 10] - st[..., 0])[done]
    per_tile_total = np.diff(st[:, 0, :, 0], axis=-1)  # tile-to-tile period of warp 0
    per_tile_total = per_tile_total[(st[:, 0, 1:, 0] != 0) & (st[:, 0, :-1, 0] != 0)]

    rows = []
    print(f"K1 phase clock {args.label}: {torch.cuda.get_device_name()} | nvidia-smi name, power limit, max SM clock: "
          f"{power_limit()}")
    print(f"occupancy {occ} CTAs/SM (cudaOccupancyMaxActiveBlocksPerMultiprocessor), grid {grid}, "
          f"dynamic smem {smem} B, {int(done.sum())} warp-tiles stamped")
    if len(per_phase_instr) != len(PHASES):
        print(f"note: {n_clocks} clock reads in the SASS (expected 11): static counts are not split per phase")
    print(f"{'phase':<22}{'median cyc':>12}{'p90 cyc':>10}{'SASS instr':>12}")
    for i, name in enumerate(PHASES):
        med, p90 = float(np.median(d[:, i])), float(np.percentile(d[:, i], 90))
        ins = per_phase_instr[i] if len(per_phase_instr) == len(PHASES) else None
        rows.append({"phase": name, "median": med, "p90": p90, "sass": ins})
        print(f"{name:<22}{med:>12.0f}{p90:>10.0f}{'' if ins is None else ins:>12}")
    print(f"{'tile (stamp 0 -> 10)':<22}{np.median(tile_cycles):>12.0f}{np.percentile(tile_cycles, 90):>10.0f}"
          f"{n_instr:>12} (whole kernel)")
    print(f"{'tile period (warp 0)':<22}{np.median(per_tile_total):>12.0f}{np.percentile(per_tile_total, 90):>10.0f}")
    res = {"label": args.label, "device": torch.cuda.get_device_name(), "nvidia_smi": power_limit(),
           "occupancy": occ, "grid": grid, "smem": smem, "phases": rows,
           "tile_median": float(np.median(tile_cycles)), "period_median": float(np.median(per_tile_total)),
           "sass_total": n_instr}
    with open(os.path.join(args.out, f"k1_phase{('_' + args.label) if args.label else ''}.json"), "w") as f:
        json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
