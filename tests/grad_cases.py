"""Shared by the gradient tests: float64 torch.autograd references through torch.stft / torch.istft (the reference's
own arithmetic, ref:audiotools/core/audio_signal.py:1123-1369), and the reference's two spectral losses restated over
an AudioSignal-like object (ref:audiotools/metrics/spectral.py:70-95 MultiScaleSTFTLoss.forward, 159-192
MelSpectrogramLoss.forward; the defaults of their constructors, :29-58 and :121-157)."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from audiotools_b200 import AudioSignal

# (window_length, hop_length, match_stride, padding_type, T): every backward route and padding mode
#   warp FFT 64 .. 2048, CTA kernel sizes 32 / 4096 (dense / large backward), dense (any length), large (8192+)
STFT_GEOMETRIES = [
    (2048, 512, False, "reflect", 9000),
    (512, 128, True, "reflect", 3000),
    (256, 64, True, "constant", 1000),
    (128, 96, False, "replicate", 700),
    (32, 8, False, "reflect", 300),
    (4096, 1024, False, "replicate", 9000),
    (400, 160, False, "constant", 3000),
    (400, 100, True, "replicate", 3000),
    (255, 60, False, "reflect", 1000),
    (8192, 2048, True, "reflect", 20000),
]


def window64(window_type, wl):
    return AudioSignal.get_window(window_type, wl, "cpu").double()


def padding(T, wl, hop, ms):
    if ms:
        return math.ceil(T / hop) * hop - T, (wl - hop) // 2
    return 0, 0


def stft64(x, wl, hop, window_type="hann", ms=False, pt="reflect"):
    """ref :1123-1212 in x's precision (float64 for the references here; float32 is the reference's own arithmetic)."""
    B, C, T = x.shape
    right_pad, pad = padding(T, wl, hop, ms)
    y = F.pad(x, (pad, pad + right_pad), mode=pt)
    X = torch.stft(y.reshape(-1, y.shape[-1]), wl, hop, window=window64(window_type, wl).to(x.device, x.dtype),
                   return_complex=True, center=True)
    X = X.reshape(B, C, *X.shape[1:])
    return X[..., 2:-2] if ms else X


def istft64(S, T, wl, hop, window_type="hann", ms=False):
    """ref :1214-1296 in float64 (S [B, C, F, N] complex128); T = the original signal length."""
    B, C = S.shape[:2]
    right_pad, pad = padding(T, wl, hop, ms)
    L = T + 2 * pad + right_pad
    s = S.reshape(B * C, *S.shape[2:])
    if ms:
        s = F.pad(s, (2, 2))
    y = torch.istft(s, wl, hop, window=window64(window_type, wl).to(S.device), center=True, length=L)
    y = y.reshape(B, C, -1)
    return y[..., pad:L - (pad + right_pad)] if ms else y


def mel64(x, sr, n_mels, wl, hop, window_type="hann", fmin=0.0, fmax=None):
    """ref :1333-1369 in float64: |X|^T @ mel_basis^T."""
    X = stft64(x, wl, hop, window_type)
    fb = torch.from_numpy(np.asarray(AudioSignal.get_mel_filters(sr, wl, n_mels, fmin, fmax), dtype=np.float64))
    return (X.abs().transpose(2, -1) @ fb.to(x.device, x.dtype).T).transpose(-1, 2)


def real_inner(X, G):
    """<X, G> of a complex output and its gradient in torch's convention (sum Re X Re G + Im X Im G), float64."""
    return (X.real.double() * G.real.double() + X.imag.double() * G.imag.double()).sum()


# --------------------------------------------------------------------------- the reference's losses, restated
MEL_LOSS_DEFAULT = dict(n_mels=[150, 80], window_lengths=[2048, 512], log_weight=1.0, mag_weight=1.0, pow=2.0)
MEL_LOSS_7SCALE = dict(n_mels=[5, 10, 20, 40, 80, 160, 320], window_lengths=[32, 64, 128, 256, 512, 1024, 2048],
                       log_weight=1.0, mag_weight=0.0, pow=1.0)


def mel_loss(x_mel, y_mel, n_mels, window_lengths, log_weight, mag_weight, pow, clamp_eps=1e-5, keep=None):
    """MelSpectrogramLoss.forward (spectral.py:159-192), loss_fn = L1, hop = window // 4, hann, fmin 0, fmax None.
    x_mel(n_mels, wl, hop) / y_mel(...) return the mel spectrograms of the estimate / the reference.  ``keep`` (one
    boolean mask per scale, see ``fp32_resolution_keep``) drops cells from the log term; the mean still divides by
    every cell, so the kept cells' gradients are those of the unmasked loss."""
    loss = 0.0
    for i, (nm, wl) in enumerate(zip(n_mels, window_lengths)):
        xm, ym = x_mel(nm, wl, wl // 4), y_mel(nm, wl, wl // 4)
        xl, yl = xm.clamp(clamp_eps).pow(pow).log10(), ym.clamp(clamp_eps).pow(pow).log10()
        if keep is None:
            loss = loss + log_weight * F.l1_loss(xl, yl)
        else:
            loss = loss + log_weight * ((xl - yl).abs() * keep[i]).sum() / xl.numel()
        loss = loss + mag_weight * F.l1_loss(xm, ym)
    return loss


def undecided(vx, vy, clamp_eps, tol_log, tol_clamp_x, tol_clamp_y=None, tol_mag=None):
    """The L1 cells whose derivative is decided below FP32 resolution, from the float64 magnitudes (or mels) vx, vy of
    the two signals: boolean masks (sign, clamp_x, clamp_y, mag).  Each tolerance is a scalar or a per-cell tensor:
      - sign:  |log10 max(vx, eps) - log10 max(vy, eps)| <= tol_log, unless both are clamped (no log gradient either
               way, and both sides' log terms are the same number);
      - clamp: |log10 v - log10 eps| <= tol_clamp on that side (the clamp's step); clamp_y only with tol_clamp_y;
      - mag:   |vx - vy| <= tol_mag (the magnitude term's sign), only with tol_mag; a cell whose tensor tolerance is 0
               (two silent frames: both spectra exactly 0) is decided."""
    lx, ly = vx.clamp(clamp_eps).log10(), vy.clamp(clamp_eps).log10()
    both_clamped = (vx < clamp_eps) & (vy < clamp_eps)
    sign = ((lx - ly).abs() <= tol_log) & ~both_clamped
    clamp_x = (vx.log10() - math.log10(clamp_eps)).abs() <= tol_clamp_x
    clamp_y = (vy.log10() - math.log10(clamp_eps)).abs() <= tol_clamp_y if tol_clamp_y is not None else None
    mag = None
    if tol_mag is not None:
        d = (vx - vy).abs()
        mag = (d <= tol_mag) & (tol_mag > 0) if torch.is_tensor(tol_mag) else (d <= tol_mag)
    return sign, clamp_x, clamp_y, mag


def fp32_resolution_keep(x, y, sr, n_mels, window_lengths, pow=2.0, tol=1e-4, clamp_eps=1e-5, **_):
    """The mel cells of MelSpectrogramLoss whose log-term gradient FP32 arithmetic can resolve, from the float64 mels
    of x and y: one boolean mask per scale, and the number of cells dropped for each reason.  A cell is dropped when
      - "sign":  |log10 x_mel - log10 y_mel| <= 2^-20 (four FP32 spacings of log10 values in [2, 4), about the mels'
                 own FP32 error): the L1 term's sign(x - y) is decided below FP32 resolution.  An FP32 log10 of two mels
                 3e-7 apart can return the same value, and the cell's gradient is then 0 instead of +-1 / (mel ln10 n);
      - "clamp": log10 x_mel is within 2^-20 of log10 clamp_eps: the clamp's step lies inside FP32 resolution;
      - "zero":  a filter of the cell holds a bin with |X_k| / rms_k |X_k| < C u log2(n_fft) / tol (C = 2: the FP32 FFT
                 error budget of tests/spectral64.py) and that bin carries at least half of the mel: d|X|/dX = X / |X|
                 is discontinuous at X = 0, so its direction is known to no better than tol.  A frame that reflect
                 padding makes symmetric (the first and last) has a real spectrum, where such bins are common."""
    keep, dropped = [], {"sign": 0, "clamp": 0, "zero": 0, "cells": 0}
    tau = 2.0 ** -20
    for nm, wl in zip(n_mels, window_lengths):
        hop = wl // 4
        fb = torch.from_numpy(np.asarray(AudioSignal.get_mel_filters(sr, wl, nm), dtype=np.float64)).to(x.device)
        X = stft64(x.double(), wl, hop).abs()
        xm = (X.transpose(2, -1) @ fb.T).transpose(-1, 2)
        ym = mel64(y.double(), sr, nm, wl, hop)
        sign, clamp, _, _ = undecided(xm, ym, clamp_eps, tau, tau)
        rms = X.pow(2).mean(-2, keepdim=True).sqrt()
        small = X < (2.0 * 2.0 ** -24 * math.log2(wl) / tol) * rms  # [B, C, F, N]
        share = ((X * small).transpose(2, -1) @ fb.T).transpose(-1, 2)  # the mel of the small bins
        zero = share >= 0.5 * xm
        k = ~(sign | clamp | zero)
        keep.append(k)
        dropped["sign"] += int(sign.sum())
        dropped["clamp"] += int((clamp & ~sign).sum())
        dropped["zero"] += int((zero & ~sign & ~clamp).sum())
        dropped["cells"] += k.numel()
    return keep, dropped


def stft_loss(x_mag, y_mag, window_lengths=(2048, 512), clamp_eps=1e-5, pow=2.0, log_weight=1.0, mag_weight=1.0):
    """MultiScaleSTFTLoss.forward (spectral.py:70-95), loss_fn = L1, hop = window // 4, hann."""
    loss = 0.0
    for wl in window_lengths:
        xm, ym = x_mag(wl, wl // 4), y_mag(wl, wl // 4)
        loss = loss + log_weight * F.l1_loss(xm.clamp(clamp_eps).pow(pow).log10(), ym.clamp(clamp_eps).pow(pow).log10())
        loss = loss + mag_weight * F.l1_loss(xm, ym)
    return loss


def signal_losses(x: torch.Tensor, y: torch.Tensor, sr: int, keep=(None, None)):
    """(mel default, 7-scale mel, multi-scale STFT) losses over this package's AudioSignal, each a fresh signal of x
    (which requires grad) and of y; ``keep``: the cell masks of the two mel losses (``mel_loss``)."""
    def sig_mel(t):
        return lambda nm, wl, hop: AudioSignal(t, sr).mel_spectrogram(nm, window_length=wl, hop_length=hop,
                                                                      window_type="hann")

    def sig_mag(t):
        def f(wl, hop):
            s = AudioSignal(t, sr)
            s.stft(wl, hop, "hann")
            return s.magnitude
        return f

    return (mel_loss(sig_mel(x), sig_mel(y), **MEL_LOSS_DEFAULT, keep=keep[0]),
            mel_loss(sig_mel(x), sig_mel(y), **MEL_LOSS_7SCALE, keep=keep[1]),
            stft_loss(sig_mag(x), sig_mag(y)))


def oracle_losses(x: torch.Tensor, y: torch.Tensor, sr: int, keep=(None, None)):
    """The same three losses through torch.stft in x's precision (float64: the exact reference; float32: the real
    reference's arithmetic)."""
    def o_mel(t):
        return lambda nm, wl, hop: mel64(t, sr, nm, wl, hop)

    def o_mag(t):
        return lambda wl, hop: stft64(t, wl, hop).abs()

    return (mel_loss(o_mel(x), o_mel(y), **MEL_LOSS_DEFAULT, keep=keep[0]),
            mel_loss(o_mel(x), o_mel(y), **MEL_LOSS_7SCALE, keep=keep[1]),
            stft_loss(o_mag(x), o_mag(y)))


# --------------------------------------------------------------------------- the real reference's gradients
def golden_errors(golden, device):
    """Every case of tests/golden/make_golden_grad.py recomputed through this package's AudioSignal on ``device``:
    {case: (rel_err, elementwise_ok)} against the real reference's gradients (and the loss values)."""
    from tests.conftest import elementwise_ok, rel_err
    from tests.golden import make_golden_grad as mg

    x, y = mg.make_input().to(device), mg.make_input(1).to(device)
    T, sr = mg.T, mg.SR

    def cmp(key, got, keep=None):
        got = got[mg.ROWS].detach().cpu()
        if keep is not None:
            got = got[..., keep]
        want = torch.from_numpy(golden[key])
        if torch.is_complex(got):
            return rel_err(torch.view_as_real(got), torch.view_as_real(want)), elementwise_ok(got.abs(), want.abs())
        return rel_err(got, want), elementwise_ok(got, want, frame_dim=-1)

    errs = {}
    for i, (key, wl, hop, wt, ms, pt) in enumerate(mg.STFT_CASES):
        xg = x.clone().requires_grad_()
        X = AudioSignal(xg, sr).stft(window_length=wl, hop_length=hop, window_type=wt, match_stride=ms, padding_type=pt)
        G = mg.cotangent(X.shape, 100 + i, complex_=True).to(device)
        (gx,) = torch.autograd.grad(real_inner(X, G), xg)
        errs[key + "_stft_vjp"] = cmp(key + "_stft_vjp", gx, mg.keep_index(T, mg.edge_of(wl, hop, ms)))
        if key in mg.ISTFT_CASES:
            S = X.detach().clone().requires_grad_()
            s = AudioSignal(x.clone(), sr)
            s.stft_data = S
            yy = s.istft(window_length=wl, hop_length=hop, window_type=wt, match_stride=ms).audio_data
            assert yy.shape[-1] == int(golden[key + "_istft_len"])
            (gS,) = torch.autograd.grad((yy * mg.cotangent(yy.shape, 200 + i).to(device)).sum(), S)
            errs[key + "_istft_vjp"] = cmp(key + "_istft_vjp", gS[..., ::mg.BIN_STRIDE, :])
    for i, (key, wl, nm) in enumerate(mg.MEL_CASES):
        for log in (False, True):
            xg = x.clone().requires_grad_()
            mel = AudioSignal(xg, sr).mel_spectrogram(nm, window_length=wl, hop_length=wl // 4)
            gm = mg.cotangent(mel.shape, 300 + i).to(device)
            out = mel.clamp(1e-5).pow(2).log10() if log else mel
            (gx,) = torch.autograd.grad((out * gm).sum(), xg)
            k = key + ("_log_vjp" if log else "_vjp")
            errs[k] = cmp(k, gx, mg.keep_index(T, wl))
    xg = x.clone().requires_grad_()
    mf = AudioSignal(xg, sr).mfcc(**mg.MFCC)
    (gx,) = torch.autograd.grad((mf * mg.cotangent(mf.shape, 400).to(device)).sum(), xg)
    errs["mfcc_vjp"] = cmp("mfcc_vjp", gx, mg.keep_index(T, mg.MFCC["window_length"]))
    for k, loss_of in enumerate(["loss_mel", "loss_mel7", "loss_stft"]):
        xg = x.clone().requires_grad_()
        loss = signal_losses(xg, y, sr)[k]
        (gx,) = torch.autograd.grad(loss, xg)
        want = float(golden[loss_of])
        errs[loss_of] = (abs(loss.item() - want) / abs(want), True)
        errs[loss_of + "_grad"] = cmp(loss_of + "_grad", gx, mg.keep_index(T, 2048))
    return errs


def check_golden(golden, device, tol=1e-4):
    """Assert every golden case at ``tol`` (global relative; element-wise too where the gradient is a transform's, not
    a loss's: an L1 loss's gradient flips sign between neighbouring cells).  The one exception is the gradient of
    MultiScaleSTFTLoss: log10 of single bins has d/dX = X / (|X|^2 ln10), and the real reference's own FP32 gradient is
    ~1e-4 away from the float64 one (measured on this golden: 1.05e-4).  There the check is that this package is as
    accurate as the reference: its distance to float64 at most 1.25x the reference's."""
    from tests.conftest import rel_err
    from tests.golden import make_golden_grad as mg

    errs = golden_errors(golden, device)
    bad = {k: v for k, v in errs.items() if k != "loss_stft_grad" and not (v[0] < tol and (v[1] or "loss" in k))}
    assert not bad, bad
    x, y = mg.make_input().to(device), mg.make_input(1).to(device)
    xd = x.double().requires_grad_()
    (w,) = torch.autograd.grad(oracle_losses(xd, y.double(), mg.SR)[2], xd)
    w = w[mg.ROWS][..., mg.keep_index(mg.T, 2048)].cpu()
    xg = x.clone().requires_grad_()
    (g,) = torch.autograd.grad(signal_losses(xg, y, mg.SR)[2], xg)
    g = g[mg.ROWS][..., mg.keep_index(mg.T, 2048)].cpu()
    ref_err = rel_err(torch.from_numpy(golden["loss_stft_grad"]), w)
    assert rel_err(g, w) <= max(tol, 1.25 * ref_err), (rel_err(g, w), ref_err, errs["loss_stft_grad"])
    return errs
