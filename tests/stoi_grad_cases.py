"""Checks of metrics.quality.STOILoss (the STOI backward of csrc/stoi.cu) shared by the simulator tests
(tests/test_sim_stoi_grad.py) and the GPU tests (tests/test_gpu_stoi_grad.py), and their float64 yardstick: a torch
restatement of ``tests/stoi_oracle.py`` (pystoi's algorithm) that autograd differentiates.

The restatement is dtype-generic and differentiable with respect to the estimate:
  - mono: the mean over channels;
  - resampling: the kernel's zero-padded polyphase gather out[m] = sum_n taps[m down + half - n up] x[n] with the
    engine's taps (pystoi's Octave design; checked against ``scipy.signal.resample_poly`` to 1e-12);
  - silence removal: the mask comes from the reference alone (a constant), the kept frames of both signals are
    windowed and overlap-added;
  - the 512-point rFFT of the frames, the third-octave envelopes, and the segment correlations (standard: scale,
    clip at -15 dB SDR, correlate; extended: row then column normalisation), as ``stoi_oracle.stoi_detail``;
  - an item with fewer than 30 STFT frames scores the constant 1e-5.
"""
import numpy as np
import torch

from audiotools_b200 import AudioSignal, metrics
from audiotools_b200.core import grad as _grad
from audiotools_b200.engine import Engine, get_engine
from tests import stoi_oracle as so
from tests.golden import make_golden_quality as mg

CLIP = 1.0 + 10 ** (-so.BETA / 20)
GLOBAL_TOL = 1e-4  # |g_kernel - g64| / |g64| over a case
ROW_TOL = 1e-3     # max_n |g_kernel - g64| per item, relative to max_n |g64| of the item


# ---------------------------------------------------------------------------------------------- float64 restatement
def _resample_index(T, up, down, n_taps):
    n10 = -(-T * up // down)
    half = (n_taps - 1) // 2
    kp = -(-n_taps // up)
    a = np.arange(n10, dtype=np.int64) * down + half
    nh = a // up
    t = (a - nh * up)[:, None] + up * np.arange(kp)[None, :]
    n = nh[:, None] - np.arange(kp)[None, :]
    valid = (t < n_taps) & (n >= 0) & (n < T)
    return np.where(valid, n, 0), np.where(valid, t, 0), valid


def resample(x: torch.Tensor, sample_rate: int) -> torch.Tensor:
    """x [..., T] -> [..., ceil(T up / down)] at 10 kHz, the kernel's polyphase gather (differentiable)."""
    up, down = Engine.stoi_ratio(sample_rate)
    if up == down == 1:
        return x
    taps = Engine.stoi_taps(sample_rate)
    n, t, valid = _resample_index(x.shape[-1], up, down, taps.size)
    w = torch.from_numpy(taps[t]).to(x)
    # the padding slots are a where, not a zero weight: autograd then sends them nothing, where 0 * a NaN gradient
    # would reach sample 0
    v = torch.from_numpy(valid).to(x.device)
    return torch.where(v, x[..., torch.from_numpy(n).to(x.device)] * w, 0.0).sum(-1)


def _window(like):
    return torch.from_numpy(np.hanning(so.N_FRAME + 2)[1:-1].copy()).to(like)


def _frames(x):
    n_fr = max(-(-(x.shape[-1] - so.N_FRAME) // so.HOP), 0)  # len(range(0, len(x) - 256, 128))
    return x.unfold(-1, so.N_FRAME, so.HOP)[:n_fr] * _window(x)


def kept_frames(x10: torch.Tensor) -> np.ndarray:
    """Indices of the frames the silence removal keeps, from the clean 10 kHz signal (float64 numpy)."""
    xf = _frames(x10.detach().double()).cpu().numpy()
    e = 20 * np.log10(np.linalg.norm(xf, axis=1) + so.EPS)
    return np.nonzero((np.max(e) - so.DYN_RANGE - e) < 0)[0]


def _removed(x10, kept):
    f = _frames(x10)[torch.from_numpy(kept).to(x10.device)]
    a, b = f[:, :so.HOP], f[:, so.HOP:]
    return torch.cat([a[0], (a[1:] + b[:-1]).reshape(-1), b[-1]])


def _tob(r):
    spec = torch.fft.rfft(_frames(r), n=so.NFFT)
    p = spec.real ** 2 + spec.imag ** 2
    return torch.sqrt(p @ torch.from_numpy(so.OBM.T.copy()).to(p)).T  # [15, M]


def _segments(tob):
    return tob.unfold(1, so.N, 1).permute(1, 0, 2)  # [J, 15, 30]


def _score(xt, yt, extended):
    xs, ys = _segments(xt), _segments(yt)
    if extended:
        def rc(v):
            v = v - v.mean(-1, keepdim=True)
            v = v / torch.sqrt((v ** 2).sum(-1, keepdim=True))
            v = v - v.mean(1, keepdim=True)
            return v / torch.sqrt((v ** 2).sum(1, keepdim=True))

        xn, yn = rc(xs), rc(ys)
        return (xn * yn / so.N).sum() / xn.shape[0]
    c = torch.linalg.norm(xs, dim=2, keepdim=True) / (torch.linalg.norm(ys, dim=2, keepdim=True) + so.EPS)
    yp = torch.minimum(ys * c, xs * CLIP)
    yp = yp - yp.mean(2, keepdim=True)
    xs = xs - xs.mean(2, keepdim=True)
    yp = yp / (torch.linalg.norm(yp, dim=2, keepdim=True) + so.EPS)
    xs = xs / (torch.linalg.norm(xs, dim=2, keepdim=True) + so.EPS)
    return (yp * xs).sum() / (xs.shape[0] * xs.shape[1])


def item_stoi(est_mono, ref_mono, sample_rate, extended=False):
    """STOI of one item: est_mono / ref_mono [T] at sample_rate; differentiable with respect to est_mono."""
    y, x = resample(est_mono, sample_rate), resample(ref_mono, sample_rate)
    kept = kept_frames(x)
    if len(kept) - 1 < so.N:
        return est_mono.sum() * 0 + 1e-5
    return _score(_tob(_removed(x, kept)), _tob(_removed(y, kept)), extended)


def batch_stoi(est, ref, sample_rate, extended=False):
    """[B] scores of est / ref [B, C, T] (mixed to mono by the mean over channels)."""
    e, r = est.mean(1), ref.mean(1)
    return torch.stack([item_stoi(e[b], r[b], sample_rate, extended) for b in range(e.shape[0])])


def grad64(est32: np.ndarray, ref32: np.ndarray, sample_rate, extended, device="cpu"):
    """dscore/dest [B, C, T] float64 of the restatement at the float32 inputs (upstream 1 per item)."""
    e = torch.from_numpy(est32).to(device).double().requires_grad_()
    r = torch.from_numpy(ref32).to(device).double()
    out = torch.zeros_like(e)
    for b in range(e.shape[0]):  # item by item keeps the gather's memory to one item
        s = item_stoi(e[b].mean(0), r[b].mean(0), sample_rate, extended)
        out[b] = torch.autograd.grad(s, e, allow_unused=True)[0][b] if s.requires_grad else 0.0
    return out


def clip_margin(est32, ref32, sample_rate):
    """min over the standard-mode cells of |c y_t - clip x_t| / (clip x_t): how far each cell is from a clip flip."""
    e = torch.from_numpy(est32).double().mean(1)
    r = torch.from_numpy(ref32).double().mean(1)
    out = np.inf
    for b in range(e.shape[0]):
        y, x = resample(e[b], sample_rate), resample(r[b], sample_rate)
        kept = kept_frames(x)
        if len(kept) - 1 < so.N:
            continue
        xs, ys = _segments(_tob(_removed(x, kept))), _segments(_tob(_removed(y, kept)))
        c = torch.linalg.norm(xs, dim=2, keepdim=True) / (torch.linalg.norm(ys, dim=2, keepdim=True) + so.EPS)
        out = min(out, float(((ys * c - xs * CLIP).abs() / (xs * CLIP)).min()))
    return out


# ---------------------------------------------------------------------------------------------- checks
def signals(est, ref, sr, device, grad=False):
    e = torch.from_numpy(np.ascontiguousarray(est)).to(device)
    if grad:
        e.requires_grad_()
    return e, AudioSignal(e, sr), AudioSignal(torch.from_numpy(np.ascontiguousarray(ref)).to(device), sr)


def kernel_grad(est, ref, sr, extended, device):
    """(loss per item [B] float32, dloss.sum()/dest [B, C, T]) of STOILoss on the engine."""
    x, e, r = signals(est, ref, sr, device, grad=True)
    loss = metrics.STOILoss(extended, reduction="none")(e, r)
    (g,) = torch.autograd.grad(loss.sum(), x)
    return loss.detach(), g


def check_value(key, device):
    """STOILoss(reduction="none") is -stoi() cast to float32; the gradient path's engine scores are bit-identical to
    the no-gradient call's; the golden holds within 1e-5."""
    from tests.quality_cases import GOLDEN

    g = np.load(GOLDEN)
    est, ref, sr = mg.case_signals(key)
    for mode, ext in (("std", False), ("ext", True)):
        x, e, r = signals(est, ref, sr, device, grad=True)
        loss = metrics.STOILoss(ext, reduction="none")(e, r)
        assert loss.dtype == torch.float32 and loss.device == x.device and loss.requires_grad
        _, e0, r0 = signals(est, ref, sr, device)
        want = metrics.quality.stoi(e0, r0, ext)
        assert torch.equal(loss.detach().cpu(), (-want).float()), (key, mode)
        s_grad = _grad.STOI.apply(x, r.audio_data, sr, ext)
        s_plain = get_engine().stoi(x.detach(), r.audio_data, sr, ext)[0]
        assert torch.equal(s_grad.detach(), s_plain)
        assert np.abs(-loss.detach().cpu().double().numpy() - g[f"{key}_{mode}"]).max() < 1e-5
        for red, fn in (("mean", torch.mean), ("sum", torch.sum)):
            v = metrics.STOILoss(ext, reduction=red)(e, r)
            assert v.dtype == torch.float32 and v.shape == ()
            assert v.item() == fn(-want).float().item()


def gradient_errors(key, extended, device):
    """Kernel gradient against the float64 restatement's for golden case `key`: (global relative error, worst
    per-row error / max |g| of the row over the noisy rows, largest gradient norm of a row whose estimate is the
    reference or a scaled copy of it / largest of a noisy row).  Those rows sit at the score's maximum, where the exact
    gradient is 0 and both gradients are rounding noise, so they are held to a small norm instead of a per-row match."""
    est, ref, sr = mg.case_signals(key)
    _, gk = kernel_grad(est, ref, sr, extended, device)
    g64 = -grad64(est, ref, sr, extended, device)
    gk = gk.double()
    glob = float(torch.linalg.norm(gk - g64) / torch.linalg.norm(g64))
    worst, noisy, flat = 0.0, 0.0, 0.0
    for b, (kind, _, _) in enumerate(mg.CASES[key][3]):
        if kind != "snr":
            flat = max(flat, float(gk[b].norm()))
            continue
        noisy = max(noisy, float(g64[b].norm()))
        m = float(g64[b].abs().max())
        d = float((gk[b] - g64[b]).abs().max())
        worst = max(worst, d / m if m > 0 else (0.0 if d == 0 else np.inf))
    return glob, worst, flat / noisy


def check_gradient(key, extended, device):
    glob, worst, flat = gradient_errors(key, extended, device)
    assert glob <= GLOBAL_TOL and worst <= ROW_TOL and flat <= 1e-4, (key, extended, glob, worst, flat)


def check_directional(extended):
    """A central difference of the float64 numpy oracle along a random direction equals <g, v> of the restatement:
    the restatement's gradient is the derivative of the number the reference's goldens pin."""
    for key, b in (("sr16000", 0), ("sr44100", 0), ("snr16000", 3)):
        est, ref, sr = mg.case_signals(key)
        e = est[b, 0].astype(np.float64)
        r = ref[b, 0].astype(np.float64)
        et = torch.from_numpy(e).requires_grad_()
        (g,) = torch.autograd.grad(item_stoi(et, torch.from_numpy(r), sr, extended), et)
        v = np.random.default_rng(7).standard_normal(e.size) * np.abs(e).max()
        h = 1e-6
        fd = (so.stoi(r, e + h * v, sr, extended) - so.stoi(r, e - h * v, sr, extended)) / (2 * h)
        an = float((g.numpy() * v).sum())
        assert abs(fd - an) <= 1e-6 * abs(an), (key, extended, fd, an)


def check_properties(device, extended):
    """Scale invariance, a zero gradient at est = ref, exact zeros for a short item and for samples only silent
    (dropped) frames cover, and a batch row equal to the item alone."""
    # scale invariance: <g, est> = 0
    est, ref, sr = mg.case_signals("snr16000")
    _, g = kernel_grad(est, ref, sr, extended, device)
    x = torch.from_numpy(est).to(device)
    for b in range(est.shape[0]):
        dot = float((g[b].double() * x[b].double()).sum())
        assert abs(dot) <= 1e-5 * float(g[b].double().norm() * x[b].double().norm()), (b, dot)
    # est = ref: the maximum, so the gradient vanishes (relative to the gradient at 10 dB SNR)
    g10 = float(g[1].double().norm())
    _, g0 = kernel_grad(ref, ref, sr, extended, device)
    assert float(g0.double().norm(dim=(1, 2)).max()) <= 1e-6 * g10
    # a short item (M < 30) and an item beside it
    est, ref, sr = mg.case_signals("short16000")
    _, g = kernel_grad(est, ref, sr, extended, device)
    assert torch.equal(g[0], torch.zeros_like(g[0])) and bool(g[1].abs().max() > 0)
    # 10 kHz with a silent gap: samples that no kept frame covers get exactly 0
    sr, T = 10000, 24000
    ref = mg.speech(sr, T, 51, ((0.6, 1.3),))[None, None]
    est = mg.with_snr(ref, 5.0, 52)
    _, g = kernel_grad(est, ref, sr, extended, device)
    kept = kept_frames(torch.from_numpy(ref[0, 0]).double())
    covered = np.zeros(T, bool)
    for f in kept:
        covered[f * so.HOP:f * so.HOP + so.N_FRAME] = True
    assert (~covered).sum() > 3000
    gn = g[0, 0].cpu().numpy()
    assert (gn[~covered] == 0).all() and np.count_nonzero(gn[covered]) > 0.9 * covered.sum()
    # row r of a batch is the item run alone, bit for bit
    est, ref, sr = mg.case_signals("snr16000")
    _, g = kernel_grad(est, ref, sr, extended, device)
    _, g2 = kernel_grad(est[2:3], ref[2:3], sr, extended, device)
    assert torch.equal(g[2:3], g2)


def check_plumbing(device):
    """References requiring a gradient raise; the no-gradient path makes stoi()'s launches and no more; a deferred
    gain is differentiated through."""
    import pytest

    est, ref, sr = mg.case_signals("gaps16000")
    x, e, _ = signals(est, ref, sr, device, grad=True)
    _, r_grad, _ = signals(ref, ref, sr, device, grad=True)
    with pytest.raises(NotImplementedError, match="references"):
        metrics.STOILoss()(e, r_grad)
    eng = get_engine()
    for ext in (False, True):
        _, e0, r0 = signals(est, ref, sr, device)
        n0 = eng.launches
        metrics.quality.stoi(e0, r0, ext)
        n_stoi = eng.launches - n0
        n0 = eng.launches
        with torch.no_grad():
            a = metrics.STOILoss(ext)(e, r0)
        b = metrics.STOILoss(ext)(e0, r0)
        assert eng.launches - n0 == 2 * n_stoi and not a.requires_grad and not b.requires_grad
        # deferred gain vs the same gain applied explicitly (noisy rows: away from the score's maximum)
        ne, nr, nsr = mg.case_signals("snr16000")
        db = torch.tensor([-6.0, 3.0, 12.0, -20.0])
        gains = torch.exp(db * float(np.float32(AudioSignal.GAIN_FACTOR))).to(device)
        x2, _, r2 = signals(ne, nr, nsr, device, grad=True)
        sig = AudioSignal(x2 * gains[:, None, None], nsr)
        (g2,) = torch.autograd.grad(metrics.STOILoss(ext, reduction="sum")(sig, r2), x2)
        # on CUDA a gain set while grad mode is off is deferred, then applied by the loss (Gain's backward)
        for deferred in ((False, True) if x2.is_cuda else (False,)):
            x1, e1, r1 = signals(ne, nr, nsr, device, grad=True)
            with torch.set_grad_enabled(not deferred):
                e1.volume_change(db)
            assert (e1._pending_gain is not None) == deferred
            (g1,) = torch.autograd.grad(metrics.STOILoss(ext, reduction="sum")(e1, r1), x1)
            torch.testing.assert_close(g1, g2, rtol=1e-5, atol=1e-6 * float(g2.abs().max()))
