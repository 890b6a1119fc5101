"""ITU-R BS.1770 integrated loudness on the sm_90a engine.

``LoudnessMixin.loudness`` keeps the shell of ref:audiotools/core/loudness.py:268-320 (cache,
zero-extension to 0.5 s, clamp to -70 LUFS); the measurement itself -- K-weighting IIR, 400 ms /
75 % blocks, two-pass gating (ref :102-126, :164-247) -- is ``libb2a`` (``csrc/lufs.cu``).

Difference from the reference, on purpose: the reference switches to a 512-tap FIR
*approximation* of the K-weighting filters whenever the data is on CUDA (ref :143-146) because
torchaudio's IIR is sequential; it also folds channels into the batch there (ref :96-99).  This
engine always evaluates the exact IIR recursion (the reference's CPU semantics, the parity
target of BASELINE.json), on the GPU.  ``use_fir`` / ``zeros`` are accepted and ignored.
"""
import torch

from . import kweighting


def _engine():
    from ..engine import get_engine

    return get_engine()


class Meter(torch.nn.Module):
    """Tensorised BS.1770 meter with the constructor and ``integrated_loudness`` contract of
    ref:audiotools/core/loudness.py:11-247 (input ``[nb, nt, nch]``, output ``[nb]`` float32)."""

    def __init__(self, rate: int, filter_class: str = "K-weighting", block_size: float = 0.400,
                 zeros: int = 512, use_fir: bool = False):
        super().__init__()
        self.rate = rate
        self.filter_class = filter_class
        self.block_size = block_size
        self.use_fir = use_fir
        kweighting.design(float(rate), filter_class)  # raises for classes that are not implemented
        self.register_buffer("G", torch.from_numpy(kweighting.CHANNEL_GAINS.copy()))

    def integrated_loudness(self, data: torch.Tensor, padded_length: int = None):
        if not torch.is_tensor(data):
            data = torch.as_tensor(data)
        data = data.float()
        if data.ndim < 2:
            data = data.unsqueeze(-1)
        if data.ndim < 3:
            data = data.unsqueeze(0)
        x = data.permute(0, 2, 1).contiguous()  # -> [nb, nch, nt], the engine's layout
        return _engine().lufs(x, self.rate, self.filter_class, self.block_size, padded_length=padded_length)["lufs"]

    forward = integrated_loudness


class LoudnessMixin:
    _loudness = None
    MIN_LOUDNESS = -70
    """Minimum loudness possible."""

    def loudness(self, filter_class: str = "K-weighting", block_size: float = 0.400, **kwargs):
        """Integrated gated loudness [B] in LUFS, clamped to >= -70; cached until ``audio_data`` is reassigned."""
        if self._loudness is not None:
            return self._loudness.to(self.device)
        T = self.signal_length
        padded = T
        if self.signal_duration < 0.5:  # zero-extend to 0.5 s (ref :302-305); no copy: the kernel reads zeros
            padded = T + int((0.5 - self.signal_duration) * self.sample_rate)
        kweighting.design(float(self.sample_rate), filter_class)
        # detached: the loudness is not differentiable (nor is the reference's, ref:tests/core/test_grad.py:70)
        out = _engine().lufs(self._materialized().detach(), self.sample_rate, filter_class, block_size,
                             padded_length=padded)
        self._loudness = out["loud"]
        return self._loudness.to(self.device)
