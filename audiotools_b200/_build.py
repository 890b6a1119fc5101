"""In-tree build of ``audiotools_b200/csrc/libb2a.so`` for sm_90a (H100; nvcc cross-compiles
without a GPU).  The .so is a build product and is git-ignored."""
import glob
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(CSRC, "libb2a.so")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


def _digest(files):
    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    for f in sorted(files):
        with open(f, "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    """Build (if stale) and return the path of libb2a.so.  Safe to call from several processes at once (the ranks of a
    torchrun launch, the two ranks of a gloo test): an exclusive file lock serialises the builders and the library is
    moved into place atomically, so a concurrent importer never sees a half-written file."""
    import fcntl

    if not force and _up_to_date(_deps()):  # a built tree may be read-only: take no lock unless there is work
        return OUT
    with open(os.path.join(CSRC, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            return _build_locked(force, verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


STAMP = os.path.join(CSRC, ".libb2a.stamp")


def _deps():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu"))) + sorted(glob.glob(os.path.join(CSRC, "*.h"))) + sorted(
        glob.glob(os.path.join(CSRC, "*.cuh"))) + [os.path.join(os.path.dirname(HERE), "include", "b2a.h")]


def _up_to_date(deps):
    if not (os.path.exists(OUT) and os.path.exists(STAMP)):
        return False
    with open(STAMP) as f:
        return f.read() == _digest(deps)


def _build_locked(force: bool, verbose: bool) -> str:
    srcs = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
    deps = _deps()
    if not force and _up_to_date(deps):
        return OUT
    dig = _digest(deps)
    nvcc = _nvcc()
    objs, procs = [], []
    for s in srcs:
        o = s[:-3] + ".o"
        cmd = [nvcc] + NVCC_FLAGS + ["-c", s, "-o", o]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(o)
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {s}:\n{out.decode()}")
    tmp = OUT + ".tmp.%d" % os.getpid()
    cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", tmp] + objs
    subprocess.check_call(cmd)
    os.replace(tmp, OUT)
    with open(STAMP, "w") as f:
        f.write(dig)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
