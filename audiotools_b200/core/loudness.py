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
        kweighting.design(float(self.sample_rate), filter_class)
        # detached: the loudness is not differentiable (nor is the reference's, ref:tests/core/test_grad.py:70)
        out = _engine().lufs(self._materialized().detach(), self.sample_rate, filter_class, block_size,
                             padded_length=self._padded_length())
        self._loudness = out["loud"]
        return self._loudness.to(self.device)

    def _padded_length(self) -> int:
        if self.signal_duration < 0.5:  # zero-extend to 0.5 s (ref :302-305); no copy: the kernel reads zeros
            return self.signal_length + int((0.5 - self.signal_duration) * self.sample_rate)
        return self.signal_length

    def loudness_stats(self, filter_class: str = "K-weighting", series: bool = False, true_peak: bool = False):
        """EBU R128 loudness statistics of every item, the numbers of the reference's ``r128stats``
        (ref:audiotools/core/ffmpeg.py:13-62) computed on the GPU: a dict of [B] float32 tensors

        * ``"I"``: integrated loudness, bit-identical to the engine's unclamped BS.1770 loudness (``-inf`` for silence;
          ``loudness()`` clamps it to -70);
        * ``"I Threshold"``: the relative gate of that measurement, ``-inf`` when no 400 ms block passes -70 LUFS;
        * ``"LRA"``, ``"LRA Threshold"``, ``"LRA Low"``, ``"LRA High"``: the loudness range of EBU Tech 3342.

        With ``true_peak=True`` also ``"True Peak"``, the dBTP of ``true_peak()`` (after the six, before the series).
        With ``series=True`` also ``"momentary"`` [B, n_400ms] (the loudness of every 400 ms gating block, 100 ms
        apart) and ``"short_term"`` [B, n_3s] (3 s blocks, 100 ms apart), in LUFS.

        Definitions, with s = int(0.1 * rate) samples (the gating stride), G_c the BS.1770 channel gains and the
        K-weighted energies of the strides summed in float64:

        * short-term block i covers strides i .. i + 29, S_i = -0.691 + 10 log10(sum_c G_c E_c,i / (30 s)), rounded to
          float32; there are (T - 30 s) // s + 1 of them (none below 30 s samples).  30 s is 3 s of audio at every
          common rate, but 33060 samples (2.9986 s) at 11025 Hz;
        * LRA Threshold = -0.691 + 10 log10(mean of 10^((S + 0.691) / 10) over S > -70) - 20;
        * the kept S are those > -70 and > LRA Threshold; sorted ascending (n of them), LRA Low = v[floor(0.10 (n - 1)
          + 0.5)], LRA High = v[floor(0.95 (n - 1) + 0.5)] (nearest rank, as libebur128), LRA = High - Low;
        * no S above -70 (including signals shorter than 3 s): LRA = 0 and the other three are -inf.

        These are not ffmpeg's numbers: ffmpeg's ebur128 filter quantises its gating histogram, this uses the BS.1770
        arithmetic of ``loudness()``.  The two have not been compared.  Items shorter than 0.5 s are zero-extended to
        0.5 s as in ``loudness()``.  The values are detached, and no cache (``loudness()``'s, ``stft_data``) is read or
        written.  Only ``filter_class="K-weighting"`` is implemented; R128 fixes the block at 0.4 s."""
        kweighting.design(float(self.sample_rate), filter_class)  # raises for classes that are not implemented
        x = self._materialized().detach()
        out = _engine().loudness_stats(x, self.sample_rate, padded_length=self._padded_length(), want_series=series)
        if true_peak:
            series_out = {k: out.pop(k) for k in ("momentary", "short_term") if k in out}
            out["True Peak"] = _engine().true_peak(x, self.sample_rate)["db"]
            out.update(series_out)
        return {k: v.to(self.device) for k, v in out.items()}

    def true_peak(self):
        """True-peak level of every item, [B] float32 dBTP (-inf for silence; NaN or +inf for an item with a non-finite
        sample): 20 log10 of the largest |value| over the channels of the signal oversampled by L = 4 below 96 kHz,
        2 below 192 kHz, else 1, in one pass on the GPU (``csrc/truepeak.cu``).

        The interpolator is this package's: phase 0 is the sample itself (so the true peak is never below the sample
        peak); phase p = 1 .. L-1 is y[n] = sum_{d=-6..5} h_p[d] x[n - d] with the 12 float32 taps
        h_p[d] = sinc(u) (1 + cos(pi u / 6)) / 2, u = d + p / L, designed in double (a Hann-windowed sinc over +-6
        samples, no per-phase renormalisation).  Only instants inside the item count: every phase between two
        samples, and the last sample itself.  It has the structure of ITU-R BS.1770-4 Annex 2 (a 4x polyphase FIR at
        48 kHz) but not the Annex's coefficient table, and it has not been compared with ffmpeg or libebur128.  On
        steady sines between 0.005 and 0.45 fs it reads between -0.44 and +0.11 dB of the amplitude at L = 4 (the
        largest under-read near 0.4 fs) and between -0.69 and +0.11 dB at L = 2 (near 0.25 fs).

        Read from the samples with any deferred ``normalize`` / ``volume_change`` gain applied; detached, and no
        cache is read or written."""
        return _engine().true_peak(self._materialized().detach(), self.sample_rate)["db"].to(self.device)
