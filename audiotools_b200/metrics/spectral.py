"""The reference's spectral losses (ref:audiotools/metrics/spectral.py): ``MultiScaleSTFTLoss``, ``MelSpectrogramLoss``
and ``PhaseLoss``, with the reference's constructors, defaults and ``forward(x, y)``.

Each scale of the two L1 losses runs on ``csrc/loss.cu`` (``core.grad.SpectralLoss``) when its inputs allow it:
``loss_fn`` is an ``nn.L1Loss`` with ``reduction="mean"``, the window is a power of two in [64, 2048], x and y resolve
to the same geometry (sample rate, shape, window type, match_stride, padding type) and the rows / mel filters are
within the backward's limits.  One launch then gives the scale's loss and the gradient wrt the estimate's STFT, and the
backward is the STFT adjoint alone.  Every other scale runs the reference's arithmetic through the differentiable
``AudioSignal`` methods (``stft`` / ``mel_spectrogram``); there is no option to choose between the two.

Kept from the reference, on purpose:
  - the constructors' ``match_stride`` is stored but unused: the signals' own ``stft_params`` decide match_stride and
    padding, as ``x.stft(window_length, hop_length, window_type)`` does in the reference;
  - ``weight`` is stored and not applied (the caller weighs the losses);
  - ``PhaseLoss`` wraps with ``diff[diff > pi] -= -2 pi``, i.e. it ADDS 2 pi there.
One difference: the reference leaves the last scale's STFT in each signal's ``stft_data`` (a side effect of calling
``stft()``).  Here neither signal's ``stft_data`` changes, on either path, as ``mel_spectrogram`` already leaves it.
"""
import typing
from typing import List

import numpy as np
import torch
from torch import nn

from ..core import AudioSignal
from ..core import STFTParams
from ..core import grad as _grad


def _stft_args(s: STFTParams):
    return (s.window_length, s.hop_length, s.window_type, None, None)


def _stft(sig: AudioSignal, s: STFTParams) -> torch.Tensor:
    """``sig.stft(window_length, hop_length, window_type)`` without touching ``sig.stft_data``."""
    return sig._spectral(_stft_args(s), want_stft=True)["stft"]


def _fused(loss_fn, x: AudioSignal, y: AudioSignal, s: STFTParams, n_mels: int = 0):
    """The geometry (window_length, hop, window_type, match_stride, padding_type) of a scale that the fused kernel
    computes, or None when this scale runs the composed path."""
    from ..engine import get_engine

    if not (isinstance(loss_fn, nn.L1Loss) and loss_fn.reduction == "mean"):
        return None
    if not (isinstance(x, AudioSignal) and isinstance(y, AudioSignal)):
        return None
    geo = x._resolve_stft(*_stft_args(s))
    wl, hop = geo[0], geo[1]
    if not (64 <= wl <= 2048 and (wl & (wl - 1)) == 0):
        return None
    if geo != y._resolve_stft(*_stft_args(s)) or x.sample_rate != y.sample_rate:
        return None
    xa, ya = x._audio_data, y._audio_data
    if xa.shape != ya.shape or xa.device != ya.device:
        return None
    if xa.shape[0] * xa.shape[1] > _grad.MAX_ROWS or n_mels > _grad.MAX_MELS:
        return None
    if not get_engine().spectral_loss_supported(wl, hop, n_mels):
        return None
    return geo


def _fused_loss(x: AudioSignal, y: AudioSignal, geo, mel, clamp_eps, pow, log_weight, mag_weight):
    wl, hop, wt, ms, pt = geo
    xa, ya = x._materialized(), y._materialized()  # a deferred gain is applied first (no gain inside the kernel)
    window = AudioSignal.get_window(wt, wl, xa.device)
    right_pad, pad = x.compute_stft_padding(wl, hop, ms)
    args = (xa, ya, wl, hop, window, pad, right_pad, pt, 2 if ms else 0, mel, float(clamp_eps), float(pow),
            float(log_weight), float(mag_weight))
    if _grad.wants_grad(xa) or _grad.wants_grad(ya):
        return _grad.SpectralLoss.apply(*args)
    from ..engine import get_engine

    return get_engine().spectral_loss(*args)[0]


class MultiScaleSTFTLoss(nn.Module):
    """Computes the multi-scale STFT loss from [1] (ref:audiotools/metrics/spectral.py:11-95).

    Parameters
    ----------
    window_lengths : List[int], optional
        Length of each window of each STFT, by default [2048, 512]
    loss_fn : typing.Callable, optional
        How to compare each loss, by default nn.L1Loss()
    clamp_eps : float, optional
        Clamp on the log magnitude, below, by default 1e-5
    mag_weight : float, optional
        Weight of raw magnitude portion of loss, by default 1.0
    log_weight : float, optional
        Weight of log magnitude portion of loss, by default 1.0
    pow : float, optional
        Power to raise magnitude to before taking log, by default 2.0
    weight : float, optional
        Weight of this loss, by default 1.0 (stored, not applied)
    match_stride : bool, optional
        Stored, not used: the signals' ``stft_params`` decide match_stride, by default False
    window_type : str, optional
        Window of every scale; None: the signals' own, by default None

    References
    ----------
    1.  Engel, Jesse, Chenjie Gu, and Adam Roberts.
        "DDSP: Differentiable Digital Signal Processing."
        International Conference on Learning Representations. 2019.
    """

    def __init__(
        self,
        window_lengths: List[int] = [2048, 512],
        loss_fn: typing.Callable = nn.L1Loss(),
        clamp_eps: float = 1e-5,
        mag_weight: float = 1.0,
        log_weight: float = 1.0,
        pow: float = 2.0,
        weight: float = 1.0,
        match_stride: bool = False,
        window_type: str = None,
    ):
        super().__init__()
        self.stft_params = [
            STFTParams(window_length=w, hop_length=w // 4, match_stride=match_stride, window_type=window_type)
            for w in window_lengths
        ]
        self.loss_fn = loss_fn
        self.log_weight = log_weight
        self.mag_weight = mag_weight
        self.clamp_eps = clamp_eps
        self.weight = weight
        self.pow = pow

    def forward(self, x: AudioSignal, y: AudioSignal):
        """Multi-scale STFT loss between an estimate ``x`` and a reference ``y``."""
        loss = 0.0
        for s in self.stft_params:
            geo = _fused(self.loss_fn, x, y, s)
            if geo is not None:
                loss = loss + _fused_loss(x, y, geo, None, self.clamp_eps, self.pow, self.log_weight, self.mag_weight)
                continue
            xm, ym = _stft(x, s).abs(), _stft(y, s).abs()
            loss = loss + self.log_weight * self.loss_fn(
                xm.clamp(self.clamp_eps).pow(self.pow).log10(),
                ym.clamp(self.clamp_eps).pow(self.pow).log10(),
            )
            loss = loss + self.mag_weight * self.loss_fn(xm, ym)
        return loss


class MelSpectrogramLoss(nn.Module):
    """Distance between mel spectrograms, optionally at several scales (ref:audiotools/metrics/spectral.py:98-192).

    Parameters
    ----------
    n_mels : List[int]
        Number of mels per STFT, by default [150, 80],
    window_lengths : List[int], optional
        Length of each window of each STFT, by default [2048, 512]
    loss_fn : typing.Callable, optional
        How to compare each loss, by default nn.L1Loss()
    clamp_eps : float, optional
        Clamp on the log magnitude, below, by default 1e-5
    mag_weight : float, optional
        Weight of raw magnitude portion of loss, by default 1.0
    log_weight : float, optional
        Weight of log magnitude portion of loss, by default 1.0
    pow : float, optional
        Power to raise magnitude to before taking log, by default 2.0
    weight : float, optional
        Weight of this loss, by default 1.0 (stored, not applied)
    match_stride : bool, optional
        Stored, not used: the signals' ``stft_params`` decide match_stride, by default False
    mel_fmin, mel_fmax : List[float], optional
        Band edges of each scale's filterbank, by default [0.0, 0.0] and [None, None]
    window_type : str, optional
        Window of every scale; None: the signals' own, by default None
    """

    def __init__(
        self,
        n_mels: List[int] = [150, 80],
        window_lengths: List[int] = [2048, 512],
        loss_fn: typing.Callable = nn.L1Loss(),
        clamp_eps: float = 1e-5,
        mag_weight: float = 1.0,
        log_weight: float = 1.0,
        pow: float = 2.0,
        weight: float = 1.0,
        match_stride: bool = False,
        mel_fmin: List[float] = [0.0, 0.0],
        mel_fmax: List[float] = [None, None],
        window_type: str = None,
    ):
        super().__init__()
        self.stft_params = [
            STFTParams(window_length=w, hop_length=w // 4, match_stride=match_stride, window_type=window_type)
            for w in window_lengths
        ]
        self.n_mels = n_mels
        self.loss_fn = loss_fn
        self.clamp_eps = clamp_eps
        self.log_weight = log_weight
        self.mag_weight = mag_weight
        self.weight = weight
        self.mel_fmin = mel_fmin
        self.mel_fmax = mel_fmax
        self.pow = pow

    def forward(self, x: AudioSignal, y: AudioSignal):
        """Mel loss between an estimate ``x`` and a reference ``y``."""
        loss = 0.0
        for n_mels, fmin, fmax, s in zip(self.n_mels, self.mel_fmin, self.mel_fmax, self.stft_params):
            geo = _fused(self.loss_fn, x, y, s, n_mels)
            if geo is not None:
                mel = AudioSignal._mel_tables(x.sample_rate, geo[0], n_mels, fmin, fmax, x._audio_data.device)
                loss = loss + _fused_loss(x, y, geo, mel, self.clamp_eps, self.pow, self.log_weight, self.mag_weight)
                continue
            kwargs = {"window_length": s.window_length, "hop_length": s.hop_length, "window_type": s.window_type}
            x_mels = x.mel_spectrogram(n_mels, mel_fmin=fmin, mel_fmax=fmax, **kwargs)
            y_mels = y.mel_spectrogram(n_mels, mel_fmin=fmin, mel_fmax=fmax, **kwargs)
            loss = loss + self.log_weight * self.loss_fn(
                x_mels.clamp(self.clamp_eps).pow(self.pow).log10(),
                y_mels.clamp(self.clamp_eps).pow(self.pow).log10(),
            )
            loss = loss + self.mag_weight * self.loss_fn(x_mels, y_mels)
        return loss


class PhaseLoss(nn.Module):
    """Difference between phase spectrograms (ref:audiotools/metrics/spectral.py:195-247).

    Parameters
    ----------
    window_length : int, optional
        Length of STFT window, by default 2048
    hop_length : int, optional
        Hop length of STFT window, by default 512
    weight : float, optional
        Weight of loss, by default 1.0 (stored, not applied)
    """

    def __init__(self, window_length: int = 2048, hop_length: int = 512, weight: float = 1.0):
        super().__init__()
        self.weight = weight
        self.stft_params = STFTParams(window_length, hop_length)

    def forward(self, x: AudioSignal, y: AudioSignal):
        """Magnitude-weighted squared phase error between an estimate ``x`` and a reference ``y``."""
        s = self.stft_params
        X, Y = _stft(x, s), _stft(y, s)
        diff = torch.angle(X) - torch.angle(Y)
        diff[diff < -np.pi] += 2 * np.pi
        diff[diff > np.pi] -= -2 * np.pi  # the reference's sign, kept
        mag = X.abs()
        x_min, x_max = mag.min(), mag.max()
        weights = (mag - x_min) / (x_max - x_min)
        return ((weights * diff) ** 2).mean()
