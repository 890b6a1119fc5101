"""The BS.1770 integrated loudness as a training loss: ``LoudnessLoss`` differentiates exactly the number
``AudioSignal.loudness()`` reports (``csrc/lufs.cu``; DESIGN.md K2 and K21)."""
import numbers

import torch
from torch import nn

from ..core import AudioSignal


class LoudnessLoss(nn.Module):
    """Distance in LU between the estimates' integrated loudness and a target: ``|loud(est) - loud(ref)|`` per item,
    where ``loud`` is bit for bit what ``AudioSignal.loudness()`` returns (BS.1770 K-weighting, 0.4 s blocks, both
    gates, clamped at -70 LUFS, items under 0.5 s zero-extended), so a model trains on the number that is reported.

    Called as ``forward(estimates, references)``: the estimates FIRST, as ``STOILoss`` and the spectral losses.
    ``references`` is an ``AudioSignal`` (its ``loudness()``, a constant; references that require a gradient raise
    ``NotImplementedError``), a number, or 1 or B target LUFS values.

    Gradients reach ``estimates.audio_data``, through any deferred gain (``normalize`` / ``volume_change``).  The gate
    decisions are piecewise constant and are constants of the backward; an item clamped at -70 gets a zero gradient and
    an item with a NaN or inf sample an all-NaN one.  The estimates' loudness cache is neither read nor written.
    Without a gradient (no-grad mode, or estimates that do not require one) the loss makes exactly ``loudness()``'s
    launches.  Only ``filter_class="K-weighting"`` with 0.4 s blocks exists here.

    Parameters
    ----------
    reduction : str, optional
        'mean', 'sum' or anything else for none, by default 'mean'
    weight : float, optional
        Weight of this loss, defaults to 1.0 (stored, not applied).

    Returns (``forward``)
    ---------------------
    Tensor
        float32 on the estimates' device: the loss per item [batch] (no reduction) or its mean / sum, reduced in
        float64 before the cast.
    """

    def __init__(self, reduction: str = "mean", weight: float = 1.0):
        self.reduction = reduction
        self.weight = weight
        super().__init__()

    @staticmethod
    def _target(estimates: AudioSignal, references, device) -> torch.Tensor:
        from ..core import grad as _grad

        B = estimates.batch_size
        if isinstance(references, AudioSignal):
            if references.sample_rate != estimates.sample_rate:
                raise ValueError(f"LoudnessLoss: sample rates differ (estimates {estimates.sample_rate}, references "
                                 f"{references.sample_rate})")
            if references.batch_size != B:
                raise ValueError(f"LoudnessLoss: batch sizes differ (estimates {B}, references "
                                 f"{references.batch_size})")
            _grad.refuse_param_grad("LoudnessLoss", "references", references._materialized())
            return references.loudness()
        if isinstance(references, numbers.Number):
            return torch.full((1,), float(references), dtype=torch.float64, device=device)
        _grad.refuse_param_grad("LoudnessLoss", "references", references)
        t = torch.as_tensor(references).reshape(-1).to(device=device, dtype=torch.float64)
        if t.numel() not in (1, B):
            raise ValueError(f"LoudnessLoss: references must be an AudioSignal, a number or 1 or {B} target LUFS "
                             f"values, got {t.numel()} values")
        return t

    def forward(self, estimates: AudioSignal, references):
        from ..core import grad as _grad
        from ..core import kweighting
        from ..engine import get_engine

        est = estimates._materialized()
        target = self._target(estimates, references, est.device)
        sr = estimates.sample_rate
        if est.shape[1] > len(kweighting.CHANNEL_GAINS):
            raise ValueError(f"LoudnessLoss: loudness supports at most 5 channels, got {est.shape[1]}")
        Tp = estimates._padded_length()
        if _grad.wants_grad(est):
            loud = _grad.Loudness.apply(est, None, sr, Tp)
        else:
            loud = get_engine().lufs(est.detach(), sr, padded_length=Tp)["loud"]
        loss = (loud.double() - target.double()).abs()
        if self.reduction == "mean":
            loss = loss.mean()
        elif self.reduction == "sum":
            loss = loss.sum()
        return loss.float()
