"""Where the K-weighting kernel (csrc/lufs.cu) loses accuracy: its algorithm evaluated in numpy with each stage of the
state path switched between float32 and float64, and in the state basis the kernel uses.  Prints per-block errors
|z^ - z| / z against the float64 cascade, in units of u = 2^-24 (worst / median over the blocks of each signal).

    python tests/probes/kweight_state_probe.py

Stages: ``tables`` (the end-state map Wa and the powers of A, rounded once from float64), ``endstate`` (each lane's
66-tap dot product), ``scan`` (the affine scan over the 32 lanes), ``start`` (the lane start state from the carried
state), ``carry`` (the state carried to the next segment), ``rec`` (the DF-I recursion); ``Wa_split`` / ``lo_apart``
split the end-state table into float32 high and low halves (summed in the same or in a separate accumulator),
``cols64`` keeps some state components of the end-state map in float64, ``d2`` evaluates the high-pass's feed-forward
sum as a second difference (the kernel's difference form).  ``basis`` = "y" is the output history
(y[n-1], y[n-2]) of every biquad; "s" is (y[n-1] - rho y[n-2], y[n-2]) with rho the stage's largest pole radius, in
which the powers of a near-double pole at rho ~ 1 carry no cancellation."""
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)

from tests import timedomain64 as td  # noqa: E402

L2, LANES = 64, 32
SEG = L2 * LANES
U = 2.0 ** -24


def rnd(v, f32):
    return v.astype(np.float32).astype(np.float64) if f32 else v


def emulate(x, coef, f32, basis="y"):
    """The kernel's outputs y [T] for one row walked as one run from a zero state (no warm-up)."""
    b0, b1, b2, a1, a2 = (np.asarray(c, np.float64) for c in coef)
    NS = len(b0)
    D = 2 * NS
    A, Wa = td.kweight_state_maps(coef, L2)
    P = td.kweight_basis(coef) if basis == "s" else np.eye(D)
    Pi = np.linalg.inv(P)
    W = Wa @ P.T  # [66, D]: end state in the basis
    Wt = rnd(W, f32.get("Wa", f32["tables"]))
    Wlo = rnd(W - Wt, True) if f32.get("Wa_split") else np.zeros_like(W)  # float-float table: hi + lo
    Ap = np.linalg.matrix_power
    M64 = P @ Ap(A, L2) @ Pi
    Mlane = [rnd(np.linalg.matrix_power(M64, lane), f32.get("Mlane", f32["tables"])) for lane in range(LANES)]
    Mscan = [rnd(np.linalg.matrix_power(M64, 1 << k), f32.get("Mscan", f32["tables"])) for k in range(5)]
    Mseg = rnd(np.linalg.matrix_power(M64, LANES), f32.get("Mseg", f32["tables"]))
    T = x.shape[-1]
    nseg = (T + SEG - 1) // SEG
    xp = np.zeros(nseg * SEG + 2)
    xp[2:2 + T] = x
    # the 66 inputs of every lane chunk: two history samples then its 64
    idx = np.arange(nseg * LANES)[:, None] * L2 + np.arange(L2 + 2)[None, :]
    chunks = xp[idx].reshape(nseg, LANES, L2 + 2)
    g = np.zeros((nseg, LANES, D))
    glo = np.zeros((nseg, LANES, D))
    c64 = list(f32.get("cols64", []))  # components whose map and sum are float64
    Wt[:, c64] = W[:, c64]
    for j in range(L2 + 2):  # sequential fma chain over the taps, as the kernel
        gn = rnd(g + Wt[j] * chunks[..., j:j + 1], f32["endstate"])
        if not f32.get("lo_apart"):
            gn = rnd(gn + Wlo[j] * chunks[..., j:j + 1], f32["endstate"])
        gn[..., c64] = g[..., c64] + Wt[j, c64] * chunks[..., j:j + 1]
        g = gn
        glo = rnd(glo + Wlo[j] * chunks[..., j:j + 1], True)
    if f32.get("lo_apart"):  # the low halves of the split table in an accumulator of their own
        g = rnd(g + glo, f32["endstate"])
    g = rnd(g, f32["scan"])  # the scan runs on float32 states
    for k in range(5):
        s = 1 << k
        o = np.zeros_like(g)
        o[:, s:] = g[:, :-s]
        add = rnd(np.einsum("ij,slj->sli", Mscan[k], o), f32["scan"])
        g = np.where(np.arange(LANES)[None, :, None] >= s, rnd(g + add, f32["scan"]), g)
    ex = np.zeros_like(g)
    ex[:, 1:] = g[:, :-1]
    agg = g[:, -1]
    carry = np.zeros((nseg, D))
    c = np.zeros(D)
    for sgi in range(nseg):
        carry[sgi] = c
        c = rnd(agg[sgi] + rnd(Mseg @ c, f32["carry"]), f32["carry"])
    st = rnd(ex + rnd(np.einsum("lij,sj->sli", np.stack(Mlane), carry), f32["start"]), f32["start"])
    st = rnd(np.einsum("ij,slj->sli", Pi, st), f32["start"])  # back to (y[n-1], y[n-2])
    y1 = [st[..., 2 * s] for s in range(NS)]
    y2 = [st[..., 2 * s + 1] for s in range(NS)]
    out = np.zeros((nseg, LANES, L2))
    r = lambda v: rnd(v, f32["rec"])  # noqa: E731
    for i in range(L2):
        in0, in1, in2 = chunks[..., i + 2], chunks[..., i + 1], chunks[..., i]
        for s in range(NS):
            if f32.get("d2") and b1[s] == -2 * b0[s] and b2[s] == b0[s]:  # b0 (in0 - 2 in1 + in2): second difference
                f = r(b0[s] * r(r(in0 - in1) - r(in1 - in2)))
            else:
                f = r(r(b0[s] * in0) + r(r(b1[s] * in1) + r(b2[s] * in2)))
            y0 = r(r(f - r(a2[s] * y2[s])) - r(a1[s] * y1[s]))
            in0, in1, in2 = y0, y1[s], y2[s]
            y2[s], y1[s] = y1[s], y0
        out[..., i] = in0
    return out.reshape(-1)[:T]


def blocks(y, sr):
    K, st = int(0.4 * sr), int(0.1 * sr)
    n = (max(len(y), K) - K + st - 1) // st + 1
    yy = np.pad(y, (0, max(0, (n - 1) * st + K - len(y))))
    return np.array([(yy[j * st:j * st + K] ** 2).sum() for j in range(n)])


def main():
    sr, T = 48000, 96000
    g = np.random.default_rng(0)
    t = np.arange(T) / sr
    sigs = {"0.2 noise": 0.2 * g.standard_normal(T),
            "0.9 sin 20 Hz": 0.9 * np.sin(2 * np.pi * 20 * t),
            "0.5 sin 30 Hz + 0.05 noise": 0.5 * np.sin(2 * np.pi * 30 * t) + 0.05 * g.standard_normal(T)}
    coef = td.kweight_coef(sr)
    all32 = dict(tables=True, endstate=True, scan=True, start=True, carry=True, rec=True)
    variants = [("all float32, basis y (before)", all32, "y")]
    for k in all32:
        variants.append((f"{k} in float64", dict(all32, **{k: False}), "y"))
    variants.append(("state path in float64", dict(all32, tables=False, endstate=False, scan=False, start=False,
                                                   carry=False), "y"))
    variants.append(("all float32, basis s", all32, "s"))
    variants.append(("basis s, split table (as shipped)", dict(all32, Wa_split=True, lo_apart=True), "s"))
    for name, x in sigs.items():
        x = x.astype(np.float32).astype(np.float64)
        z = blocks(td.kweight64(x, coef), sr)
        zr = blocks(td.kweight_seq32(x, coef), sr)
        print(f"{name}: sequential float32 lfilter worst {np.max(np.abs(zr - z) / z) / U:.0f} u")
        for vname, f32, basis in variants:
            e = np.abs(blocks(emulate(x, coef, f32, basis), sr) - z) / z / U
            print(f"  {vname:34s} worst {e.max():9.0f} u  median {np.median(e):8.0f} u")


if __name__ == "__main__":
    main()
