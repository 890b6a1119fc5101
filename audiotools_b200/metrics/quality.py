"""The reference's quality metrics (ref:audiotools/metrics/quality.py).  ``stoi`` runs on ``csrc/stoi.cu`` for the
whole batch at once, and ``STOILoss`` is the same score as a differentiable training loss; ``pesq`` and ``visqol``
call an external C library / binary in the reference and are not ported.
"""
import warnings

from torch import nn

from ..core import AudioSignal


def stoi(estimates: AudioSignal, references: AudioSignal, extended: int = False):
    """Short term objective intelligibility
    Computes the STOI (See [1][2]) of a denoised signal compared to a clean signal.  The output is expected to have a
    monotonic relation with the subjective speech-intelligibility, where a higher score denotes better speech
    intelligibility.

    Both signals are mixed to mono, resampled to 10 kHz, the frames more than 40 dB below the clean signal's loudest
    are removed from both, and the third-octave envelopes of 384 ms segments are correlated -- pystoi's algorithm,
    which the reference calls per item, here in four CUDA launches for the batch.  An item with fewer than 30 frames
    left scores 1e-5, with a warning.  The extended mode leaves out the EPS-scale random noise pystoi adds before its
    normalisations, so the result is deterministic (it differs only where a band envelope is exactly constant over a
    segment, where pystoi's result is that noise).

    Parameters
    ----------
    estimates : AudioSignal
        Denoised speech
    references : AudioSignal
        Clean original speech
    extended : int, optional
        Boolean, whether to use the extended STOI described in [3], by default False

    Returns
    -------
    Tensor[float]
        Short time objective intelligibility measure between clean and denoised speech: float64 on the CPU, shape
        [batch], detached (no gradient flows, as in the reference).

    References
    ----------
    1.  C.H.Taal, R.C.Hendriks, R.Heusdens, J.Jensen 'A Short-Time
        Objective Intelligibility Measure for Time-Frequency Weighted Noisy
        Speech', ICASSP 2010, Texas, Dallas.
    2.  C.H.Taal, R.C.Hendriks, R.Heusdens, J.Jensen 'An Algorithm for
        Intelligibility Prediction of Time-Frequency Weighted Noisy Speech',
        IEEE Transactions on Audio, Speech, and Language Processing, 2011.
    3.  Jesper Jensen and Cees H. Taal, 'An Algorithm for Predicting the
        Intelligibility of Speech Masked by Modulated Noise Maskers',
        IEEE Transactions on Audio, Speech and Language Processing, 2016.
    """
    from ..engine import get_engine

    score, _, short = get_engine().stoi(estimates._materialized(), references._materialized(),
                                        references.sample_rate, bool(extended))
    score, short = score.cpu(), short.cpu()
    if bool(short.any()):
        warnings.warn("Not enough STFT frames to compute intermediate intelligibility measure after removing silent "
                      f"frames (items {short.nonzero().flatten().tolist()}). Returning 1e-5 for them. Please check "
                      "your audio", RuntimeWarning)
    return score


class STOILoss(nn.Module):
    """Negative STOI (or extended STOI) as a differentiable training loss: ``-score`` per item, where ``score`` is
    exactly what ``stoi(estimates, references, extended)`` returns (same kernels, same value), so a model trains on
    the number that is later reported.

    The arguments are in ``stoi``'s order: the estimates FIRST, then the clean references.  (``SISDRLoss`` takes the
    reference first, as in the reference.)

    Gradients reach ``estimates.audio_data`` only, through any deferred gain (``normalize`` / ``volume_change``);
    the references are constants, and references that require a gradient raise ``NotImplementedError``.  The silence
    removal depends on the references alone, so it is a constant of the backward pass; every other stage is
    differentiated exactly (CUDA backward kernels, no host synchronisation).  An item with fewer than 30 STFT frames
    left scores 1e-5, as in ``stoi``, and gets a zero gradient; unlike ``stoi`` it raises no warning.  Without a
    gradient (no-grad mode, or estimates that do not require one) the loss makes exactly ``stoi``'s launches.

    Parameters
    ----------
    extended : bool, optional
        Extended STOI [3] instead of STOI, by default False
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

    def __init__(self, extended: bool = False, reduction: str = "mean", weight: float = 1.0):
        self.extended = extended
        self.reduction = reduction
        self.weight = weight
        super().__init__()

    def forward(self, estimates: AudioSignal, references: AudioSignal):
        from ..core import grad as _grad
        from ..engine import get_engine

        est, ref = estimates._materialized(), references._materialized()
        _grad.refuse_param_grad("STOILoss", "references", ref)
        sr, ext = references.sample_rate, bool(self.extended)
        if _grad.wants_grad(est):
            score = _grad.STOI.apply(est, ref, sr, ext)
        else:
            score = get_engine().stoi(est, ref, sr, ext)[0]
        loss = -score
        if self.reduction == "mean":
            loss = loss.mean()
        elif self.reduction == "sum":
            loss = loss.sum()
        return loss.float()


def pesq(estimates: AudioSignal, references: AudioSignal, mode: str = "wb", target_sr: float = 16000):
    """PESQ (ITU-T P.862.2 MOS-LQO).  The reference calls the ``pesq`` package's C implementation of the ITU
    recommendation; it is not ported."""
    raise NotImplementedError("pesq calls the ITU P.862 C library (the pesq package): not ported")


def visqol(estimates: AudioSignal, references: AudioSignal, mode: str = "audio"):
    """ViSQOL (MOS-LQO).  The reference calls Google's ViSQOL binary through its Python bindings; it is not ported."""
    raise NotImplementedError("visqol calls the external ViSQOL binary: not ported")
