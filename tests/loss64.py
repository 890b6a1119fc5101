"""Float64 references and the per-cell error model of the fused spectral losses (``spectral_loss_kernel<LOG2N, MEL>``,
csrc/loss.cu), shared by tests/test_gpu_loss_accuracy.py (H100), tests/test_sim_loss_accuracy.py (simulator) and
tests/probes/loss_accuracy_probe.py.

The reference takes the float64 STFTs X, Y of the float32 inputs (``spectral64.stft_ref``, the engine's framing), one
scale's loss from them by the reference's arithmetic (``metrics_cases.scale_loss64`` restated on spectra), and
dL/dX, dL/dY by ``torch.autograd.grad`` in torch's complex convention, the one the kernel writes.

Error model.  The kernel's spectra carry the per-bin error of its FFT: beta = ``spectral64.budget(n_fft)`` times the
frame's RMS bin magnitude (the same bound as the STFT's), and its mels ``spectral64.mel_bound``'s delta.  With v the
float64 magnitude (or mel) of a cell, d = dL/dv (a log part d_log and a magnitude part) and g its gradient:
  - STFT mode:  |g^ - g| <= C (|d_log| beta / v + |g| (beta / v + u)): the 1 / v of the log term's derivative, the
    direction X / |X| (|X^/|X^| - X/|X|| <= 2 beta / v) and a few roundings;
  - mel mode:   |g^_k - g_k| <= C (sum_m fb[m, k] (|d_log,m| delta_m / mel_m + |d_m| u) + |g_k| beta_k / |X_k|): the
    same terms of every mel cell through the transposed projection, and the bin's own direction;
  - loss, per term:  |L^ - L| <= C_LOSS (sum_cells e + n u sum_cells |t|) / numel, e the cell's term error
    (log: pow (beta_x / v_x + beta_y / v_y) / ln 10 + a few ulp of log10f / powf; magnitude: beta_x + beta_y), t the
    term and n the cells of one frame (the kernel's float accumulation).
The C's are set from the H100 run in DESIGN.md ("Loss accuracy").

Keep mask: a cell counts when its derivative is decided above FP32 resolution (``grad_cases.undecided`` with these
bounds as tolerances): the log term's L1 sign, the magnitude term's L1 sign (beta plus the rounding of |X| itself,
a few u |X|: a loud bin's two FP32 magnitudes can be one float apart), each side's clamp step, and (log term
only) a magnitude within 2 beta of 0, where 1 / v^ is unbounded.  In the mel mode a bin is dropped when any mel cell
whose band holds it is dropped.  A dropped STFT-mode cell must still match one of the float64 gradients with each
undecided branch taken either way, within twice the kept cells' budget."""
import itertools
import math

import torch

from tests import grad_cases as gc
from tests import spectral64 as s64

U = s64.U
LN10 = math.log(10.0)
# log10f and powf (or the square) of one side: a few ulp of lg = pow log10 max(v, eps), absolute in lg units
LG_ULP = 4 * U

# Budget constants of the model above: set from the H100 measurement in DESIGN.md "Loss accuracy" (NVIDIA H100 80GB
# HBM3, 700 W power limit) with about 2x headroom over the worst case measured there and on the simulator (kept
# cells: 1.33 / 1.22 in the STFT mode, 0.89 / 0.84 in the mel mode).  A loss term's errors mostly cancel across cells
# (0.055 on the H100), except in a frame that holds one input sample (T = 1 under constant match_stride padding):
# its spectrum is an impulse's, every bin carries the same rounding, and the term's error reaches 0.146 of the sum of
# the cells' bounds (simulator, four rows; the sum itself, C_LOSS = 1, is the bound with no cancellation).
C_CELL = {"stft": 2.5, "mel": 2.0}
C_LOSS = 0.3
# ours <= TORCH_FACTOR x torch's FP32 error (torch.stft in float32 and the same loss on the same input), per kept cell
# and per loss term, each in the model's units.  Torch's error is floored (TORCH_FLOOR, LOSS_FLOOR units): a frame that
# reflect padding makes symmetric has a real spectrum, which cuFFT returns with exact zero imaginary parts, and a
# loss term over a few cells is the rounding of those cells, of either sign
TORCH_FACTOR = 2.0
TORCH_FLOOR = 0.6
LOSS_FLOOR = 0.01
MIN_LOSS_CELLS = 4096  # a loss term over fewer cells is compared with its budget alone
MAX_DROP = 0.01  # the share of noise cells the keep mask may drop

# rows of ``batch``: the signals of spectral64.signals (y: the same kinds at another seed; the alternating sequence
# has no noise, so its x == y), noise with a stretch of exact zeros over whole frames in both (collate's padding),
# x == y, and a row that is silent in x only / in y only
NOISE = ("noise", "noise_1e-3", "noise_1e-6")
KINDS = NOISE + ("tones_120dB", "dc", "nyquist", "gap", "same", "x_zero", "y_zero")


def batch(n_fft: int, hop: int, T: int, kinds=KINDS, seed: int = 0):
    """x, y [len(kinds), 1, T] float32, one row per kind."""
    frames = max(2, -(-(T - 1) // hop) + 1)
    sx, sy = s64.signals(n_fft, hop, frames, seed), s64.signals(n_fft, hop, frames, seed + 1)
    xs, ys = [], []
    for k in kinds:
        src = k if k in sx else "noise"
        a, b = sx[src][0, 0, :T].clone(), sy[src][1, 0, :T].clone()
        if k == "same":
            b = a.clone()
        elif k == "x_zero":
            a.zero_()
        elif k == "y_zero":
            b.zero_()
        elif k == "gap":
            a[T // 4:T // 4 + n_fft + 2 * hop] = 0
            b[T // 4:T // 4 + n_fft + 2 * hop] = 0
        xs.append(a)
        ys.append(b)
    return torch.stack(xs)[:, None], torch.stack(ys)[:, None]


def mel_tables(mel, n_fft: int, dev):
    """(fb, lo, hi) of mel = (sr, n_mels, fmin, fmax) on dev."""
    from audiotools_b200 import AudioSignal

    sr, nm, fmin, fmax = mel
    return AudioSignal._mel_tables(sr, n_fft, nm, float(fmin), fmax, torch.device(dev))


def max_mels(eng, n_fft: int, hop: int) -> int:
    """The largest n_mels ``b2a_spectral_loss_supported`` accepts for the window and hop."""
    lo, hi = 1, 1 << 15
    assert eng.spectral_loss_supported(n_fft, hop, lo) and not eng.spectral_loss_supported(n_fft, hop, hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if eng.spectral_loss_supported(n_fft, hop, mid) else (lo, mid)
    return lo


def reference(x, y, n_fft, hop, window, geo=(0, 0, "reflect", 0), fb=None, clamp_eps=1e-5, pow=2.0, log_weight=1.0,
              mag_weight=1.0, frac=1.0, dtype=torch.float64):
    """One scale's loss from the STFTs of x, y [R, C, T] (float32) in ``dtype`` (float64: the reference; float32:
    torch's FP32 arithmetic) -> dict: the spectra X, Y, dL/dX, dL/dY, the cells' magnitudes (or mels) vx, vy, the
    cells' log and magnitude terms, and the two terms' means.  ``frac`` scales the weights: the rows of a strided
    subset of a launch have the gradient of the whole launch when frac = subset rows / launch rows."""
    X = s64.stft_ref(x, n_fft, hop, window, *geo, dtype=dtype).detach().requires_grad_()
    Y = s64.stft_ref(y, n_fft, hop, window, *geo, dtype=dtype).detach().requires_grad_()

    def mag(S):
        v = S.abs()
        return v if fb is None else (v.transpose(-1, -2) @ fb.to(v.device, dtype).T).transpose(-1, -2)

    vx, vy = mag(X), mag(Y)
    lg = lambda v: v.clamp(clamp_eps).pow(pow).log10()  # noqa: E731
    tl, tm = (lg(vx) - lg(vy)).abs(), (vx - vy).abs()
    L = frac * (log_weight * tl.mean() + mag_weight * tm.mean())
    gX, gY = torch.autograd.grad(L, (X, Y))
    return dict(X=X.detach(), Y=Y.detach(), gX=gX, gY=gY, vx=vx.detach(), vy=vy.detach(), tl=tl.detach(),
                tm=tm.detach(), log=tl.mean().item(), mag=tm.mean().item())


def model(ref, n_fft, fb=None, clamp_eps=1e-5, pow=2.0, log_weight=1.0, mag_weight=1.0, frac=1.0):
    """The per-cell bounds and the keep mask of a float64 ``reference`` -> dict (see the module's docstring)."""
    X, Y, vx, vy = ref["X"], ref["Y"], ref["vx"], ref["vy"]
    dev = X.device
    bud = s64.budget(n_fft)
    beta_x = bud * X.abs().pow(2).mean(-2, keepdim=True).sqrt()  # [..., 1, N]
    beta_y = bud * Y.abs().pow(2).mean(-2, keepdim=True).sqrt()
    if fb is None:
        dx, dy = beta_x.expand_as(vx), beta_y.expand_as(vy)
    else:
        fb = fb.double().to(dev)
        dx = s64.mel_bound(fb, X, bud, s64.MEL_RTOL)[0].to(dev)
        dy = s64.mel_bound(fb, Y, bud, s64.MEL_RTOL)[0].to(dev)
    numel = vx.numel()
    cl, cm = frac * log_weight / numel, frac * mag_weight / numel
    lx, ly = pow * vx.clamp(clamp_eps).log10(), pow * vy.clamp(clamp_eps).log10()
    s_l, s_m = torch.sign(lx - ly), torch.sign(vx - vy)
    on_x, on_y = vx >= clamp_eps, vy >= clamp_eps
    tiny = torch.finfo(torch.float64).tiny

    def dlog(v, on):  # d(lg v)/dv where the clamp passes the gradient
        return torch.where(on, pow / (LN10 * v.clamp_min(tiny)), torch.zeros_like(v))

    rel_x, rel_y = dx / vx.clamp_min(tiny), dy / vy.clamp_min(tiny)
    # the keep mask (in log10 v units for the sign and the clamp)
    tol_log = (dx / vx.clamp(clamp_eps) + dy / vy.clamp(clamp_eps)) / LN10 + LG_ULP * (lx.abs() + ly.abs() + 1) / pow
    sign, clamp_x, clamp_y, magu = gc.undecided(vx, vy, clamp_eps, tol_log, (rel_x + 2 * U) / LN10,
                                                (rel_y + 2 * U) / LN10, dx + dy + 2 * U * (vx + vy))
    none = torch.zeros_like(sign)
    if log_weight == 0:
        sign = clamp_x = clamp_y = none
    if mag_weight == 0:
        magu = none
    zero = (vx < 2 * dx) | (vy < 2 * dy) if log_weight != 0 else none
    drop = {"sign": sign, "mag": magu & ~sign, "clamp": (clamp_x | clamp_y) & ~sign & ~magu}
    drop["zero"] = zero & ~(sign | magu | clamp_x | clamp_y)
    cell_drop = sign | magu | clamp_x | clamp_y | zero
    # dL/dv of each cell: its log part and the whole
    dl_x, dl_y = cl * s_l * dlog(vx, on_x), -cl * s_l * dlog(vy, on_y)
    d_x, d_y = dl_x + cm * s_m, dl_y - cm * s_m
    gx, gy = ref["gX"].abs(), ref["gY"].abs()
    if fb is None:
        unit_x = dl_x.abs() * rel_x + gx * (rel_x + U)
        unit_y = dl_y.abs() * rel_y + gy * (rel_y + U)
        bin_drop = cell_drop
    else:
        def back(t):  # sum_m fb[m, k] t[m] over the bins
            return (t.transpose(-1, -2) @ fb).transpose(-1, -2)

        unit_x = back(dl_x.abs() * rel_x + d_x.abs() * U) + gx * beta_x / X.abs().clamp_min(tiny)
        unit_y = back(dl_y.abs() * rel_y + d_y.abs() * U) + gy * beta_y / Y.abs().clamp_min(tiny)
        bin_drop = back(cell_drop.double()) > 0
    n_acc = vx.shape[-2]
    e_log = pow * (dx / vx.clamp(clamp_eps) + dy / vy.clamp(clamp_eps)) / LN10 + LG_ULP * (lx.abs() + ly.abs() + 1)
    e_mag = dx + dy
    return dict(unit_x=unit_x, unit_y=unit_y, keep=~bin_drop, cell_drop=cell_drop, drop=drop, numel=numel,
                loss_unit={"log": (e_log.sum() + n_acc * U * ref["tl"].sum()).item() / numel,
                           "mag": (e_mag.sum() + n_acc * U * ref["tm"].sum()).item() / numel},
                undecided=dict(sign=sign, mag=magu, clamp_x=clamp_x, clamp_y=clamp_y, zero=zero),
                parts=dict(s_l=s_l, s_m=s_m, on_x=on_x, on_y=on_y, cl=cl, cm=cm, dlog=dlog, rel_x=rel_x, rel_y=rel_y))


def ratio(got, want, unit, keep):
    """The worst |got - want| / unit over the kept cells (inf where unit = 0 and got != want: those must be exact)."""
    err = (got.to(torch.complex128) - want).abs()
    r = torch.where(unit > 0, err / unit.clamp_min(torch.finfo(torch.float64).tiny),
                    torch.where(err > 0, math.inf, 0.0))
    r = torch.where(keep, r, torch.zeros_like(r))
    return r.max().item() if r.numel() else 0.0


def unexplained(got, ref, m, side, c):
    """Dropped STFT-mode cells (sign, magnitude or clamp undecided; not the zero rule) whose gradient matches none of
    the float64 gradients with the undecided branches taken either way, within c model units."""
    p, und = m["parts"], m["undecided"]
    S = ref["X"] if side == "x" else ref["Y"]
    v = S.abs()
    rel = p["rel_x"] if side == "x" else p["rel_y"]
    on = p["on_x"] if side == "x" else p["on_y"]
    und_c = und["clamp_x"] if side == "x" else und["clamp_y"]
    sg = 1.0 if side == "x" else -1.0
    unit_dir = torch.where(v > 0, S / v.clamp_min(torch.finfo(torch.float64).tiny), torch.zeros_like(S))
    got = got.to(torch.complex128)
    check = m["cell_drop"] & ~und["zero"]
    ok = torch.zeros_like(check)
    for s_l, c_on, s_m in itertools.product((-1.0, 0.0, 1.0), (False, True), (-1.0, 0.0, 1.0)):
        allowed = ((und["sign"] | (p["s_l"] == s_l)) & (und_c | (on == c_on)) & (und["mag"] | (p["s_m"] == s_m)))
        dl = sg * p["cl"] * s_l * (p["dlog"](v, torch.ones_like(on)) if c_on else torch.zeros_like(v))
        d = dl + sg * p["cm"] * s_m
        g = d * unit_dir
        unit = dl.abs() * rel + g.abs() * (rel + U)
        ok |= allowed & ((got - g).abs() <= c * unit)
    return int((check & ~ok).sum())


def check(eng, x, y, n_fft, hop, window, geo=(0, 0, "reflect", 0), mel=None, clamp_eps=1e-5, pow=2.0,
          log_weight=1.0, mag_weight=1.0, kinds=None, rows=None, torch32=True):
    """Run ``Engine.spectral_loss`` on x, y [R, 1, T] (on the engine's device) with both gradients and per term, and
    hold it against the float64 reference -> dict of measurements (model units; see the module's docstring):
      c_x, c_y: worst kept-cell error of dL/dX, dL/dY; c_x_torch, c_y_torch: torch's FP32 arithmetic's;
      loss: {"log" / "mag": (ours in model units; ours and torch's in model units on the noise rows)},
        "total": ours in model units for the given weights;
      dropped: cells dropped by reason; noise_drop: the dropped share of the noise rows' bins;
      unexplained: dropped STFT-mode cells matching no branch; zero_bad: nonzero gradients of x == y rows.
    ``rows``: compare a strided subset of the rows only (the loss values are then not compared)."""
    dev = x.device
    tab = mel_tables(mel, n_fft, dev) if mel is not None else None
    fb = tab[0] if tab is not None else None
    kw = dict(clamp_eps=clamp_eps, pow=pow)
    loss, gX, gY = eng.spectral_loss(x, y, n_fft, hop, window, *geo, mel=tab, log_weight=log_weight,
                                     mag_weight=mag_weight, want_grad_x=True, want_grad_y=True, **kw)
    sel = slice(None) if rows is None else rows
    xs, ys = x[sel], y[sel]
    frac = xs.shape[0] / x.shape[0]
    wk = dict(kw, log_weight=log_weight, mag_weight=mag_weight, frac=frac)
    ref = reference(xs, ys, n_fft, hop, window, geo, fb, **wk)
    m = model(ref, n_fft, fb, **wk)
    gX, gY = gX[sel], gY[sel]
    out = {"c_x": ratio(gX, ref["gX"], m["unit_x"], m["keep"]), "c_y": ratio(gY, ref["gY"], m["unit_y"], m["keep"])}
    if torch32:
        r32 = reference(xs, ys, n_fft, hop, window, geo, fb, dtype=torch.float32, **wk)
        out["c_x_torch"] = ratio(r32["gX"], ref["gX"], m["unit_x"], m["keep"])
        out["c_y_torch"] = ratio(r32["gY"], ref["gY"], m["unit_y"], m["keep"])
    if rows is None:
        out["loss"] = {}
        # torch's FP32 loss is compared on the noise rows: where bins sit at the FFTs' error floor (tones over noise
        # 120 dB down, DC, silent stretches) each loss's error is those few bins' rounding, of either sign
        dense = [i for i in range(x.shape[0]) if kinds and i < len(kinds) and kinds[i] in NOISE] or list(range(len(x)))
        rd = reference(x[dense], y[dense], n_fft, hop, window, geo, fb, **kw) if len(dense) < x.shape[0] else ref
        rd32 = reference(x[dense], y[dense], n_fft, hop, window, geo, fb, dtype=torch.float32, **kw) if torch32 else None
        for term, w in (("log", (1.0, 0.0)), ("mag", (0.0, 1.0))):
            lt = eng.spectral_loss(x, y, n_fft, hop, window, *geo, mel=tab, log_weight=w[0], mag_weight=w[1], **kw)[0]
            ld = eng.spectral_loss(x[dense], y[dense], n_fft, hop, window, *geo, mel=tab, log_weight=w[0],
                                   mag_weight=w[1], **kw)[0] if rd is not ref else lt
            md = m if rd is ref else model(rd, n_fft, fb, **kw)
            out["dense_cells"] = rd["vx"].numel()
            scale = md["loss_unit"][term]
            e32 = abs(rd32[term] - rd[term]) / scale if torch32 else None
            out["loss"][term] = (abs(lt.item() - ref[term]) / m["loss_unit"][term], abs(ld.item() - rd[term]) / scale,
                                 e32)
        want = log_weight * ref["log"] + mag_weight * ref["mag"]
        unit = abs(log_weight) * m["loss_unit"]["log"] + abs(mag_weight) * m["loss_unit"]["mag"]
        out["loss"]["total"] = (abs(loss.item() - want) / unit, None, None)
    out["dropped"] = {k: int(v.sum()) for k, v in m["drop"].items()}
    out["cells"] = m["cell_drop"].numel()
    kinds = kinds if kinds is not None else []
    sub = list(range(x.shape[0]))[sel]
    noise = [i for i, r in enumerate(sub) if r < len(kinds) and kinds[r] in NOISE]
    out["noise_drop"] = (float((~m["keep"][noise]).double().mean()) if noise else 0.0)
    same = [i for i, r in enumerate(sub) if r < len(kinds) and kinds[r] in ("same", "nyquist")]
    out["zero_bad"] = int(torch.count_nonzero(gX[same]) + torch.count_nonzero(gY[same])) if same else 0
    if fb is None:
        un = unexplained(gX, ref, m, "x", 2 * C_CELL["stft"]) + unexplained(gY, ref, m, "y", 2 * C_CELL["stft"])
        out["unexplained"] = un
    else:
        out["unexplained"] = 0
    return out


def assert_within(out, mode, what):
    """The budgets of the model and the comparison with torch's FP32 arithmetic."""
    c = C_CELL[mode]
    for side in ("x", "y"):
        ours = out["c_" + side]
        assert ours <= c, (what, side, ours, out)
        if "c_%s_torch" % side in out:
            theirs = out["c_%s_torch" % side]
            assert ours <= TORCH_FACTOR * max(theirs, TORCH_FLOOR), (what, side, ours, theirs)
    for term, (ours, dense, dense32) in out.get("loss", {}).items():
        assert ours <= C_LOSS, (what, term, ours, out["loss"])
        if dense32 is not None and out["dense_cells"] >= MIN_LOSS_CELLS:
            assert dense <= TORCH_FACTOR * max(dense32, LOSS_FLOOR), (what, term, dense, dense32)
    assert out["noise_drop"] <= MAX_DROP, (what, out["noise_drop"], out["dropped"])
    assert out["unexplained"] == 0, (what, out["unexplained"], out["dropped"])
    assert out["zero_bad"] == 0, (what, "x == y rows must have a zero gradient")
