"""Spectral noise gate (ref:audiotools/ml/layers/spectral_gate.py:10-127; after noisereduce / Audacity's noise
reduction): a per-bin threshold from a noise excerpt's STFT statistics, a smoothed binary mask, applied to the
signal's STFT.  Both STFTs and the inverse run on the engine (``csrc/spectral.cu``, ``csrc/istft.cu``), and so does the
mask algebra in between (``csrc/specmask.cu``: threshold statistics, then boolean -> separable smoothing -> multiply in
one pass); ``smoothing_filter`` is kept as a buffer for API compatibility.  When the signal's STFT requires a gradient
the gate runs through ``core.grad.SpecGate`` (gradient g * (1 - amount * mask)); the noise signal is a constant of it,
as the reference's comparison makes it, and a ``denoise_amount`` that requires a gradient raises."""
import torch
from torch import nn

from ...core import AudioSignal
from ...core import STFTParams
from ...core import grad as _grad
from ...core import util


def _ramp(n: int) -> torch.Tensor:
    """0 < ... < 1 > ... > 0 triangle with n points on each flank (the reference's concatenated linspaces)."""
    up = torch.linspace(0, 1, n + 2)[:-1]
    down = torch.linspace(1, 0, n + 2)
    return torch.cat([up, down])[1:-1]


class SpectralGate(nn.Module):
    def __init__(self, n_freq: int = 3, n_time: int = 5):
        super().__init__()
        self._rf, self._rt = _ramp(n_freq), _ramp(n_time)  # the smoothing kernel is their outer product / sum: separable
        kernel = torch.outer(self._rf, self._rt)
        self.register_buffer("smoothing_filter", (kernel / kernel.sum())[None, None])

    def forward(self, audio_signal: AudioSignal, nz_signal: AudioSignal, denoise_amount: float = 1.0,
                n_std: float = 3.0, win_length: int = 2048, hop_length: int = 512):
        stft_params = STFTParams(win_length, hop_length, "sqrt_hann")
        audio_signal = audio_signal.clone()
        audio_signal.stft_data = None
        audio_signal.stft_params = stft_params
        nz_signal = nz_signal.clone()
        nz_signal.stft_params = stft_params

        from ...engine import get_engine

        _grad.refuse_param_grad("SpectralGate", "denoise_amount", denoise_amount)
        audio_signal.stft()
        with torch.no_grad():
            nz_signal.stft()
        amount = util.ensure_tensor(denoise_amount).reshape(-1)
        args = (nz_signal.stft_data, float(n_std), amount, self._rf.tolist(), self._rt.tolist())
        if _grad.wants_grad(audio_signal.stft_data):
            audio_signal.stft_data = _grad.SpecGate.apply(audio_signal.stft_data, *args)
        else:
            audio_signal.stft_data = get_engine().spec_gate(audio_signal.stft_data, *args)[0]
        audio_signal.istft()
        return audio_signal
