"""Float64 per-stage model of csrc/stoi.cu (STOI and its backward), shared by tests/test_gpu_stoi_accuracy.py, its
simulator twin tests/test_sim_stoi_accuracy.py and tests/probes/stoi_accuracy_probe.py.

Each stage is recomputed in float64 from the kernel's OWN output of the stage before it (read from the workspaces),
so an error is charged to the stage that made it:
  - ``resample_kernel``: the 10 kHz rows ``sig10`` against the zero-padded polyphase FIR in float64 of the float32
    channel mean, in float32 ulps plus the float64 accumulation's own bound;
  - ``mask_kernel``: the frame energies in dB, the kept lists and counts;
  - ``band_kernel``: every band envelope ``tob[s][b][i]`` in units of u ||X_i|| (the frame's spectral norm over its 257
    bins), and against the error of a float32 ``torch.fft.rfft`` of the same frames;
  - ``score_kernel``: the score from the kernel's own envelopes;
  - ``score_bwd_kernel``: dL/dtob of the estimate (``gbar``) in units of u sum_j |cell_j| |scale|, with the float64
    per-segment cells of autograd;
  - ``band_bwd_kernel``: the frame gradients ``ghat`` against a float64 inverse real FFT of W_k = gbar Y_k / tob, in
    units of u (||W|| + ||cf|| ||Y||), cf the per-bin weights gbar / tob;
  - ``unframe_kernel``: ``gy`` against a float64 gather of the kernel's ``ghat``, in units of u times the sum of the
    absolute terms (so samples no kept STOI frame covers must be exactly 0);
  - ``resample_bwd_kernel``: the gradient against a float64 transposed FIR of the kernel's ``gy``, in float32 ulps.

The budgets below are the constants the tests hold the kernels to.  Measured values are from
tests/probes/stoi_accuracy_probe.py (DESIGN.md "STOI accuracy").
"""
import numpy as np
import torch

from audiotools_b200.engine import Engine, _dptr
from tests import stoi_grad_cases as sg
from tests import stoi_oracle as so

FRAME, HOP, NBAND, SEG = 256, 128, 15, 30
EDGES = so.band_edges()  # band b covers bins [EDGES[b], EDGES[b + 1])
WIN = np.hanning(FRAME + 2)[1:-1]
U = 2.0 ** -24       # float32 unit roundoff
U64 = 2.0 ** -53

# ---- budgets.  Measured worst values by tests/probes/stoi_accuracy_probe.py (DESIGN.md "STOI accuracy"), on an
# NVIDIA H100 80GB HBM3 at a 700 W power limit over the GPU tests' cases, and on the CPU simulator (simulator only)
# over its rate and resampler-tile groups at its shapes.
RESAMPLE_ULP = 0.5   # sig10: the float64 sum rounded once, plus the float64 noise; H100 0.5, simulator 0.5
ENERGY_DB = 1e-9     # mask energies, absolute dB; H100 9.9e-14, simulator 2.8e-14
THRESH_DB = 1e-6     # kept decisions are exact for frames farther than this from max - 40 dB
C_B = 8.0            # tob, units of u ||X_i||; H100 4.74 (a tone at 7999 Hz), simulator 4.38
F_B = 8.0            # worst tob error / worst error of a float32 torch.fft.rfft of the same frames (floored at
#                      0.5 u ||X||) per call; H100 4.36, simulator 3.29
SCORE_ABS = 1e-12    # score from the kernel's own tob; H100 4.4e-16, simulator 3.3e-16
C_G = 2.0            # gbar, units of u sum_j |cell_j| |scale|; H100 1.08, simulator 0.99
C_H = 2.5            # ghat, units of u (||W|| + ||cf|| ||Y||); H100 1.28, simulator 1.04
C_Y = 5.0            # gy, units of u sum |terms|; H100 3.34, simulator 3.07
C_X = 1.0            # final gradient, float32 ulps (plus the float64 noise); H100 0.5, simulator 0.5


# ---------------------------------------------------------------------------------------------- workspaces
def align256(v):
    return (v + 255) & ~255


class Layout:
    """The forward workspace of ``b2a_stoi_f32``: sig10 [2][B][n10] float32 (the estimates' rows first), energy
    [B][n_fr] float64, kept [B][n_fr] int32, count [B] int32, tob [2][B][15][n_fr] float32, each at a 256-byte
    aligned offset; and the backward's scratch: cell [B][n_fr][15][30] float32, gbar [B][15][n_fr] float64, pos
    [B][n_fr] int32, ghat [B][n_fr][256] float32, gy [B][n10] float32."""

    def __init__(self, B, T, up, down):
        self.B, self.T = B, T
        self.n10 = -(-T * up // down)
        self.n_fr = (self.n10 - FRAME + HOP - 1) // HOP if self.n10 > FRAME else 0
        o = align256(2 * B * self.n10 * 4)
        self.off_energy = o
        o = align256(o + B * self.n_fr * 8)
        self.off_kept = o
        o = align256(o + B * self.n_fr * 4)
        self.off_count = o
        o = align256(o + B * 4)
        self.off_tob = o
        self.bytes = o + 2 * B * NBAND * self.n_fr * 4
        o = align256(B * self.n_fr * NBAND * SEG * 4)
        self.off_gbar = o
        o = align256(o + B * NBAND * self.n_fr * 8)
        self.off_pos = o
        o = align256(o + B * self.n_fr * 4)
        self.off_ghat = o
        o = align256(o + B * self.n_fr * FRAME * 4)
        self.off_gy = o
        self.bwd_bytes = o + B * self.n10 * 4


def _view(ws, off, n, dtype, shape):
    size = torch.tensor([], dtype=dtype).element_size()
    return ws[off: off + n * size].view(dtype).reshape(shape)


class Forward:
    """One ``Engine.stoi`` call and its workspace, read back to the host (numpy)."""

    def __init__(self, eng, est, ref, sr, extended, dev):
        B, C, T = est.shape
        self.sr, self.extended, self.shape = sr, extended, est.shape
        self.up, self.down = Engine.stoi_ratio(sr)
        L = self.L = Layout(B, T, self.up, self.down)
        e = torch.from_numpy(np.ascontiguousarray(est)).to(dev)
        r = torch.from_numpy(np.ascontiguousarray(ref)).to(dev)
        score, kept, short, ws = eng.stoi(e, r, sr, extended, return_workspace=True)
        assert ws.numel() == L.bytes == eng.lib.b2a_stoi_workspace_bytes(B, T, self.up, self.down)
        self.ws = ws
        self.score, self.kept_out, self.short = score.cpu().numpy(), kept.cpu().numpy(), short.cpu().numpy()
        n10, n_fr = L.n10, L.n_fr
        self.sig10 = _view(ws, 0, 2 * B * n10, torch.float32, (2, B, n10)).cpu().numpy()
        self.energy = _view(ws, L.off_energy, B * n_fr, torch.float64, (B, n_fr)).cpu().numpy()
        self.count = _view(ws, L.off_count, B, torch.int32, (B,)).cpu().numpy()
        kl = _view(ws, L.off_kept, B * n_fr, torch.int32, (B, n_fr)).cpu().numpy()
        self.kept = [kl[b, :self.count[b]].astype(np.int64) for b in range(B)]
        self.tob = _view(ws, L.off_tob, 2 * B * NBAND * n_fr, torch.float32, (2, B, NBAND, n_fr)).cpu().numpy()
        self.M = self.count.astype(np.int64) - 1


class Backward:
    """``b2a_stoi_backward_f32`` with a scratch workspace the caller keeps (filled with NaN bytes first, so a value
    a kernel reads without another having written it shows up), read back to the host."""

    def __init__(self, eng, fwd, grad_score, dev):
        B, C, T = fwd.shape
        L = fwd.L
        nbytes = eng.lib.b2a_stoi_backward_workspace_bytes(B, T, fwd.up, fwd.down)
        assert nbytes == L.bwd_bytes
        taps = eng._stoi_taps(fwd.sr, fwd.ws.device)
        g = torch.as_tensor(np.asarray(grad_score, np.float64)).to(fwd.ws.device)
        bws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=fwd.ws.device)
        gx = torch.empty(B, C, T, dtype=torch.float32, device=fwd.ws.device)
        eng._call(eng.lib.b2a_stoi_backward_f32, _dptr(g), _dptr(fwd.ws), fwd.ws.numel(), B, C, T,
                  int(fwd.extended), _dptr(taps), taps.numel(), fwd.up, fwd.down, _dptr(gx), _dptr(bws), nbytes,
                  eng._stream(fwd.ws))
        # the engine's own entry point computes the same gradient
        again = eng.stoi_backward(g, fwd.ws, (B, C, T), fwd.sr, fwd.extended)
        assert torch.equal(gx.view(torch.int32), again.view(torch.int32))  # bit for bit, NaN included
        n_fr, n10 = L.n_fr, L.n10
        self.grad_score = np.asarray(grad_score, np.float64)
        self.gbar = _view(bws, L.off_gbar, B * NBAND * n_fr, torch.float64, (B, NBAND, n_fr)).cpu().numpy()
        self.pos = _view(bws, L.off_pos, B * n_fr, torch.int32, (B, n_fr)).cpu().numpy()
        self.ghat = _view(bws, L.off_ghat, B * n_fr * FRAME, torch.float32, (B, n_fr, FRAME)).cpu().numpy()
        self.gy = _view(bws, L.off_gy, B * n10, torch.float32, (B, n10)).cpu().numpy()
        self.grad = gx.cpu().numpy()


# ---------------------------------------------------------------------------------------------- float64 stages
def mono32(x):
    """The kernel's float32 channel mean of x [C, T]: a running float32 sum over channels, then / C."""
    s = x[0].astype(np.float32).copy()
    for c in range(1, x.shape[0]):
        s += x[c]
    return (s / np.float32(x.shape[0])).astype(np.float32)


def _fir_index(T, up, down, n_taps, m):
    """Input sample and tap of every (output m, slot k) of the zero-padded polyphase FIR, and their validity."""
    half = (n_taps - 1) // 2
    kp = -(-n_taps // up)
    a = m * down + half
    nh = a // up
    t = (a - nh * up)[:, None] + up * np.arange(kp)[None, :]
    n = nh[:, None] - np.arange(kp)[None, :]
    valid = (t < n_taps) & (n >= 0) & (n < T)
    return np.where(valid, n, 0), np.where(valid, t, 0), valid


def _chunks(n_out, kp, budget=1 << 22):
    step = max(1, budget // kp)
    for m0 in range(0, n_out, step):
        yield np.arange(m0, min(n_out, m0 + step), dtype=np.int64)


def resample64(x, sr):
    """x [T] (any float) at sr -> (its 10 kHz row in float64, sum_k |tap_k x_k| per output)."""
    up, down = Engine.stoi_ratio(sr)
    taps = Engine.stoi_taps(sr)
    x = np.asarray(x, np.float64)
    T = x.size
    n10 = -(-T * up // down)
    out, mag = np.empty(n10), np.empty(n10)
    kp = -(-taps.size // up)
    for m in _chunks(n10, kp):
        n, t, valid = _fir_index(T, up, down, taps.size, m)
        v = np.where(valid, x[n] * taps[t], 0.0)
        out[m], mag[m] = v.sum(1), np.abs(v).sum(1)
    return out, mag


def resample_transpose64(gy, T, sr):
    """The transposed FIR: g[n] = sum_m taps[m down + half - n up] gy[m] -> (g [T] float64, sum of |terms| [T])."""
    up, down = Engine.stoi_ratio(sr)
    taps = Engine.stoi_taps(sr)
    gy = np.asarray(gy, np.float64)
    g, mag = np.zeros(T), np.zeros(T)
    kp = -(-taps.size // up)
    for m in _chunks(gy.size, kp):
        n, t, valid = _fir_index(T, up, down, taps.size, m)
        v = (taps[t] * gy[m][:, None])[valid]
        g += np.bincount(n[valid], weights=v, minlength=T)
        mag += np.bincount(n[valid], weights=np.abs(v), minlength=T)
    return g, mag


def energies64(x10, n_fr):
    """Frame energies in dB of a 10 kHz row (float64)."""
    x = np.asarray(x10, np.float64)
    idx = HOP * np.arange(n_fr)[:, None] + np.arange(FRAME)[None, :]
    return 20 * np.log10(np.sqrt(((x[idx] * WIN) ** 2).sum(1)) + so.EPS)


def stoi_frames64(x10, kept):
    """The M = K - 1 windowed STOI frames [M, 256] (float64) of the silence-removed row built from kept frames."""
    x = np.asarray(x10, np.float64)
    K = len(kept)
    if K < 2:
        return np.zeros((0, FRAME))
    F = x[HOP * np.asarray(kept)[:, None] + np.arange(FRAME)[None, :]] * WIN  # [K, 256]
    rb = np.zeros((K + 1, HOP))
    rb[:K] += F[:, :HOP]
    rb[1:] += F[:, HOP:]
    return np.concatenate([rb[:K - 1], rb[1:K]], axis=1) * WIN


def band_envelopes(P):
    """[M, 257] power spectra -> [15, M] band envelopes."""
    return np.sqrt(np.stack([P[:, EDGES[b]:EDGES[b + 1]].sum(1) for b in range(NBAND)]))


def tob64(frames):
    """(tob [15, M], spectra [M, 257] complex, ||X_i|| [M]) of the frames, float64."""
    X = np.fft.rfft(frames, n=so.NFFT)
    P = X.real ** 2 + X.imag ** 2
    return band_envelopes(P), X, np.sqrt(P.sum(1))


def tob32_rfft(frames):
    """The same envelopes from a float32 torch.fft.rfft of the frames rounded to float32 (the comparison FFT)."""
    X = torch.fft.rfft(torch.from_numpy(frames.astype(np.float32)), n=so.NFFT)
    P = (X.real ** 2 + X.imag ** 2).double().numpy()
    return band_envelopes(P)


def score64(xt, yt, extended):
    """Score from [15, M] envelopes (float64 torch restatement)."""
    return float(sg._score(torch.from_numpy(np.asarray(xt, np.float64)),
                           torch.from_numpy(np.asarray(yt, np.float64)), extended))


def cells64(xt, yt, extended):
    """Per-segment cells [J, 15, 30] (float64 autograd): cell_j[b][t] = d term_j / d y[b][j + t], term_j the sum of
    segment j's band correlations (standard) or of its column correlations / 30 (extended)."""
    xs = sg._segments(torch.from_numpy(np.asarray(xt, np.float64)))
    ys = sg._segments(torch.from_numpy(np.asarray(yt, np.float64))).clone().requires_grad_()
    if extended:
        def rc(v):
            v = v - v.mean(-1, keepdim=True)
            v = v / torch.sqrt((v ** 2).sum(-1, keepdim=True))
            v = v - v.mean(1, keepdim=True)
            return v / torch.sqrt((v ** 2).sum(1, keepdim=True))

        total = (rc(xs) * rc(ys)).sum() / SEG
    else:
        c = torch.linalg.norm(xs, dim=2, keepdim=True) / (torch.linalg.norm(ys, dim=2, keepdim=True) + so.EPS)
        yp = torch.minimum(ys * c, xs * sg.CLIP)
        yp = yp - yp.mean(2, keepdim=True)
        xc = xs - xs.mean(2, keepdim=True)
        yp = yp / (torch.linalg.norm(yp, dim=2, keepdim=True) + so.EPS)
        xc = xc / (torch.linalg.norm(xc, dim=2, keepdim=True) + so.EPS)
        total = (yp * xc).sum()
    (cells,) = torch.autograd.grad(total, ys)
    return cells.numpy()


def gather_cells(cells, M):
    """sum_j cells[j][b][i - j] over the segments j covering frame i -> [15, M] (and the same of |cells|)."""
    J = cells.shape[0]
    out, mag = np.zeros((NBAND, M)), np.zeros((NBAND, M))
    for t in range(SEG):
        out[:, t:t + J] += cells[:, :, t].T
        mag[:, t:t + J] += np.abs(cells[:, :, t]).T
    return out, mag


_E = np.exp(2j * np.pi * np.arange(EDGES[0], EDGES[-1])[:, None] * np.arange(FRAME)[None, :] / so.NFFT)


def unframe64(ghat, kept, M, n10):
    """The adjoint of the silence removal: dL/dy [n10] (float64) from the frame gradients ghat [M, 256], and the sum
    of the absolute terms."""
    K = len(kept)
    gy, mag = np.zeros(n10), np.zeros(n10)
    if M < SEG:
        return gy, mag
    g = np.asarray(ghat[:M], np.float64)
    dr = np.zeros((K + 1, HOP))  # dL/d removed signal, in blocks of 128
    dr[:M] += g[:, :HOP]
    dr[1:M + 1] += g[:, HOP:]
    ar = np.zeros((K + 1, HOP))
    ar[:M] += np.abs(g[:, :HOP])
    ar[1:M + 1] += np.abs(g[:, HOP:])
    nb = -(-n10 // HOP) + 2
    gb, mb = np.zeros((nb, HOP)), np.zeros((nb, HOP))
    k = np.asarray(kept)
    np.add.at(gb, k, WIN[:HOP] * dr[:K])
    np.add.at(gb, k + 1, WIN[HOP:] * dr[1:K + 1])
    np.add.at(mb, k, WIN[:HOP] * ar[:K])
    np.add.at(mb, k + 1, WIN[HOP:] * ar[1:K + 1])
    gy[:] = gb.reshape(-1)[:n10]
    mag[:] = mb.reshape(-1)[:n10]
    return gy, mag


# ---------------------------------------------------------------------------------------------- per-stage checks
def _ulp32(v):
    return np.spacing(np.abs(np.asarray(v, np.float64)).astype(np.float32)).astype(np.float64)


def _units(got, want, unit, where):
    """max |got - want| / unit over the finite entries of want; the non-finite entries of got and want must agree."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    fin = np.isfinite(want)
    assert np.array_equal(np.isfinite(got), fin), (where, "non-finite entries differ", np.nonzero(~fin)[0][:4])
    unit = np.broadcast_to(unit, want.shape)[fin]
    r = np.abs(got - want)[fin] / np.maximum(unit, np.finfo(float).tiny)
    return float(r.max(initial=0.0))


def _merge(acc, **kw):
    for k, v in kw.items():
        acc[k] = max(acc.get(k, 0.0), float(v))
    return acc


def check_forward(fwd, est, ref, where, acc=None):
    """Every forward stage of every item against float64 from the kernel's own previous stage -> worst values in
    budget units."""
    acc = {} if acc is None else acc
    B, C, T = fwd.shape
    L = fwd.L
    n10, n_fr = L.n10, L.n_fr
    kp = -(-Engine.stoi_taps(fwd.sr).size // fwd.up)
    worst_b, worst_f32 = 0.0, 0.0
    for b in range(B):
        w = (where, b)
        # resample_kernel
        for s, x in enumerate((est, ref)):
            m32 = mono32(x[b])
            got = fwd.sig10[s, b].astype(np.float64)
            if fwd.up == fwd.down == 1:
                assert np.array_equal(fwd.sig10[s, b], m32), w  # 10 kHz: the mono mix, bit for bit
                continue
            want, mag = resample64(m32, fwd.sr)
            err = np.abs(got - want)
            noise = 2 * kp * U64 * mag
            fin = np.isfinite(want)
            assert np.array_equal(np.isfinite(got), fin), w
            ulps = np.maximum(err[fin] - noise[fin], 0) / _ulp32(want[fin])
            assert ulps.max(initial=0) <= RESAMPLE_ULP, (w, s, float(ulps.max()), int(ulps.argmax()))
            _merge(acc, resample_ulp=ulps.max(initial=0))
        # mask_kernel
        e64 = energies64(fwd.sig10[1, b], n_fr)
        fin = np.isfinite(e64)
        assert np.array_equal(np.isfinite(fwd.energy[b]), fin), w
        de = np.abs(fwd.energy[b][fin] - e64[fin])
        assert de.max(initial=0) <= ENERGY_DB, (w, float(de.max()))
        _merge(acc, energy_db=de.max(initial=0))
        kept = fwd.kept[b]
        assert fwd.kept_out[b] == fwd.count[b] == len(kept)
        if np.isnan(e64).any():
            assert len(kept) == 0, w  # np.max of a NaN energy: no frame kept
        else:
            d = e64.max() - so.DYN_RANGE - e64
            want = d < 0
            got_mask = np.zeros(n_fr, bool)
            assert (np.diff(kept) > 0).all() and (len(kept) == 0 or (kept[0] >= 0 and kept[-1] < n_fr)), w
            got_mask[kept] = True
            clear = np.abs(d) > THRESH_DB
            assert np.array_equal(got_mask[clear], want[clear]), (w, np.nonzero(got_mask != want)[0][:8])
        M = int(fwd.M[b])
        assert fwd.short[b] == (M < SEG), w
        if M < 1:
            continue
        # band_kernel
        tob = {}
        for s in range(2):
            fr = stoi_frames64(fwd.sig10[s, b], kept)
            t64, _, nX = tob64(fr)
            got = fwd.tob[s, b, :, :M].astype(np.float64)
            unit = U * nX[None, :]
            r = _units(got, t64, unit, (w, s, "tob"))
            fin = np.isfinite(t64)
            r32 = np.abs(tob32_rfft(fr) - t64)[fin] / np.maximum(np.broadcast_to(unit, t64.shape)[fin], 1e-300)
            assert r <= C_B, (w, s, r)
            worst_b, worst_f32 = max(worst_b, r), max(worst_f32, r32.max(initial=0))
            tob[s] = got
        _merge(acc, C_B=worst_b)
        # score_kernel
        if M >= SEG:
            want = score64(tob[1], tob[0], fwd.extended)
            if np.isnan(want):
                assert np.isnan(fwd.score[b]), w
            else:
                assert abs(fwd.score[b] - want) <= SCORE_ABS, (w, fwd.score[b], want)
                _merge(acc, score_abs=abs(fwd.score[b] - want))
        else:
            assert fwd.score[b] == 1e-5, w
    if worst_b > 0:
        assert worst_b <= F_B * max(worst_f32, 0.5), (where, worst_b, worst_f32)
        _merge(acc, F_B=worst_b / max(worst_f32, 0.5))
    return acc


def check_backward(fwd, bwd, where, acc=None):
    """Every backward stage of every item against float64 from the kernel's own inputs to that stage."""
    acc = {} if acc is None else acc
    B, C, T = fwd.shape
    n10 = fwd.L.n10
    for b in range(B):
        w = (where, b)
        M, kept = int(fwd.M[b]), fwd.kept[b]
        # the frame -> kept position map
        pos = np.full(fwd.L.n_fr, -1)
        pos[kept] = np.arange(len(kept))
        assert np.array_equal(bwd.pos[b], pos), w
        if M >= SEG:
            xt, yt = fwd.tob[1, b, :, :M].astype(np.float64), fwd.tob[0, b, :, :M].astype(np.float64)
            J = M - SEG + 1
            # score_bwd_kernel
            cells = cells64(xt, yt, fwd.extended)
            scale = bwd.grad_score[b] / (J if fwd.extended else J * NBAND)
            g64, mag = gather_cells(cells, M)
            g64, mag = g64 * scale, mag * abs(scale)
            gk = bwd.gbar[b, :, :M]
            r = _units(gk, g64, U * mag, (w, "gbar"))
            assert r <= C_G, (w, r)
            _merge(acc, C_G=r)
            # band_bwd_kernel, from the kernel's gbar and tob
            _, Y, _ = tob64(stoi_frames64(fwd.sig10[0, b], kept))
            tk = fwd.tob[0, b, :, :M]
            cf_band = np.where(tk > 0, (gk / np.where(tk > 0, tk, 1).astype(np.float64)).astype(np.float32), 0)
            cf = np.zeros((M, Y.shape[1]))
            for band in range(NBAND):
                cf[:, EDGES[band]:EDGES[band + 1]] = cf_band[band][:, None]
            W = cf * Y
            h64 = (W[:, EDGES[0]:EDGES[-1]] @ _E).real * WIN
            unit = U * (np.linalg.norm(W, axis=1) + np.linalg.norm(cf, axis=1) * np.linalg.norm(Y, axis=1))
            r = _units(bwd.ghat[b, :M], h64, unit[:, None], (w, "ghat"))
            assert r <= C_H, (w, r)
            _merge(acc, C_H=r)
        # unframe_kernel, from the kernel's ghat
        y64, mag = unframe64(bwd.ghat[b], kept, M, n10)
        assert (bwd.gy[b][mag == 0] == 0).all(), w  # samples no kept STOI frame covers, and short items: exactly 0
        r = _units(bwd.gy[b], y64, U * mag, (w, "gy"))
        assert r <= C_Y, (w, r)
        _merge(acc, C_Y=r)
        # resample_bwd_kernel, from the kernel's gy
        x64, xmag = resample_transpose64(bwd.gy[b], T, fwd.sr)
        x64, xmag = x64 / C, xmag / C
        kp = -(-Engine.stoi_taps(fwd.sr).size // fwd.up)
        gk = bwd.grad[b].astype(np.float64)
        for c in range(1, C):
            assert np.array_equal(bwd.grad[b, c], bwd.grad[b, 0], equal_nan=True), w  # every channel the same
        assert (gk[0][xmag == 0] == 0).all(), w
        fin = np.isfinite(x64)
        assert np.array_equal(np.isfinite(gk[0]), fin), (w, "grad")
        noise = 2 * (kp + 1) * U64 * xmag[fin]
        ulps = np.maximum(np.abs(gk[0][fin] - x64[fin]) - noise, 0) / _ulp32(x64[fin])
        assert ulps.max(initial=0) <= C_X, (w, float(ulps.max()), int(ulps.argmax()))
        _merge(acc, C_X=ulps.max(initial=0))
    return acc


# ---------------------------------------------------------------------------------------------- signals
RATES = [8000, 10000, 11025, 12345, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 192000]


def _noise(n, seed):
    return np.random.default_rng(seed).standard_normal(n)


def _tone(sr, T, k, seed, amp=0.3):
    """A tone on 10 kHz STFT bin k (k * 10000 / 512 Hz, kept under 0.45 sr), over a -70 dB noise floor."""
    f = min(k * so.FS / so.NFFT, 0.45 * sr)
    t = np.arange(T) / sr
    return amp * np.sin(2 * np.pi * f * t + 0.3) + 1e-4 * _noise(T, seed)


def signal(kind, sr, T, seed):
    """[T] float32 clean signal of a kind (all reach every band unless the kind says otherwise)."""
    from tests.golden import make_golden_quality as mg

    if kind == "speech":
        x = mg.speech(sr, T, seed, ((0.25 * T / sr, 0.4 * T / sr),)).astype(np.float64)
    elif kind == "noise":
        x = 0.1 * _noise(T, seed)
    elif kind.startswith("tone"):
        x = _tone(sr, T, int(kind[4:]), seed)
    elif kind == "deep":  # one loud tone, every other band about 100 dB under it
        x = _tone(sr, T, 30, seed, amp=1.0) - 1e-4 * _noise(T, seed) + 1e-5 * _noise(T, seed + 1)
    elif kind == "silence":
        x = np.zeros(T)
    elif kind == "alternate":  # loud and silent stretches of 2.5 frames at 10 kHz
        n = int(round(320 * sr / so.FS))
        x = 0.1 * _noise(T, seed) * ((np.arange(T) // n) % 2 == 0)
    elif kind == "burst":  # one burst leaving about 31 kept frames in a long row
        n0, n = T // 3, int(round(29 * HOP * sr / so.FS))
        x = np.zeros(T)
        x[n0:n0 + n] = 0.1 * _noise(n, seed)
    else:
        raise ValueError(kind)
    return x.astype(np.float32)


def item(kind, sr, T, C, seed, snr=5.0):
    """(est [C, T], ref [C, T]) float32: the clean signal in every channel (scaled per channel) and a noisy
    estimate."""
    ref = np.stack([signal(kind, sr, T, seed) * np.float32(1.0 - 0.1 * c) for c in range(C)])
    n = 0.1 * _noise(C * T, seed + 99).reshape(C, T)
    p = float((ref.astype(np.float64) ** 2).mean())
    g = np.sqrt(p / 10 ** (snr / 10)) if p > 0 else 1e-3
    est = (ref + g * n / 0.1).astype(np.float32)
    return est, ref


def batch(kinds, sr, T, C, seed):
    pairs = [item(k, sr, T, C, seed + 17 * i) for i, k in enumerate(kinds)]
    return np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])


def bursts_10k(n10, spans, seed, tone=None):
    """A 10 kHz clean row with noise on the sample ranges [128 a, 128 b + 256) of frame spans (a, b): each span keeps
    frames a - 1 .. b + 1 (the half-covered neighbours are 3 dB down), everything else is digital silence.  A span
    (a, None) is one sample at 128 a + 64, which keeps frames a - 1 and a; (a, -1) is one sample at 128 a, which keeps
    frame a - 1 alone (the window's first tap is 76 dB under its middle).  ``tone``: the bursts are a tone on that
    STFT bin over a -50 dB noise floor instead of noise."""
    x = np.zeros(n10)
    r = np.random.default_rng(seed)
    for a, b in spans:
        if b is None:
            x[HOP * a + 64] = 0.5
        elif b == -1:
            x[HOP * a] = 0.5
        else:
            n = np.arange(HOP * a, HOP * b + FRAME)
            v = 0.1 * r.standard_normal(n.size)
            if tone is not None:
                v = 0.3 * np.sin(2 * np.pi * tone * n / so.NFFT + 0.7) + 0.003 * v
            x[n] = v
    return x.astype(np.float32)


def spans_for(M, n_fr, gap=False):
    """Spans of bursts_10k keeping exactly K = M + 1 frames (two separated spans when gap is set and M allows)."""
    K = M + 1
    if K == 1:
        return [(2, -1)]
    if K == 2:
        return [(2, None)]
    if gap and K >= 8:
        k1 = K // 2
        a1 = 2
        b1 = a1 + k1 - 3
        a2 = b1 + 7
        spans = [(a1, b1), (a2, a2 + (K - k1) - 3)]
    else:
        spans = [(2, 2 + K - 3)]
    assert spans[-1][1] + 2 < n_fr, (M, n_fr)
    return spans


def n10_for(n_fr):
    """The shortest 10 kHz length with n_fr frames."""
    return HOP * n_fr + 129
