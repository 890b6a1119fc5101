"""``DSPMixin``: per-item windowed-sinc low-/high-pass (ref:audiotools/core/dsp.py:153-215).

The reference loops over the batch in Python, building one ``julius.LowPassFilter`` per item;
here the per-item tap design and the filtering are one grouped launch each (``csrc/fir.cu``).
The spectral masks (SURVEY.md §8f.1, ref:audiotools/core/dsp.py:217-370) work on ``stft_data``: the two band
masks run as one store-only kernel (``csrc/specmask.cu``), the phase operations are container arithmetic on the
complex tensor.  When ``stft_data`` requires a gradient the masks run out of place through ``core/grad.py``'s
Functions (new CUDA backward kernels in specmask.cu); otherwise they make the same in-place launches as always.  The chunking helpers (``windows`` / ``collect_windows`` / ``overlap_and_add``) are container reshapes."""
import torch

from . import grad as _grad
from . import util


def _engine():
    from ..engine import get_engine

    return get_engine()


class DSPMixin:
    # ------------------------------------------------------------------ chunking helpers (ref :15-151)
    # Pure container reshapes on whatever device the samples live on (no kernel of their own): split long audio into
    # overlapping windows for chunked inference and put the processed windows back together.
    _original_batch_size = None
    _original_num_channels = None
    _padded_signal_length = None

    def _preprocess_signal_for_windowing(self, window_duration, hop_duration):
        self._original_batch_size = self.batch_size
        self._original_num_channels = self.num_channels
        window_length = int(window_duration * self.sample_rate)
        hop_length = int(hop_duration * self.sample_rate)
        if window_length % hop_length != 0:
            window_length = (window_length // hop_length) * hop_length
        self.zero_pad(hop_length, hop_length)
        self._padded_signal_length = self.signal_length
        return window_length, hop_length

    def windows(self, window_duration: float, hop_duration: float, preprocess: bool = True):
        """Generator over the windows of every (item, channel) row, each a [1, 1, window] signal (ref :31-68)."""
        if preprocess:
            window_length, hop_length = self._preprocess_signal_for_windowing(window_duration, hop_duration)
        else:
            window_length, hop_length = int(window_duration * self.sample_rate), int(hop_duration * self.sample_rate)
        self.audio_data = self.audio_data.reshape(-1, 1, self.signal_length)
        for b in range(self.batch_size):
            for start in range(0, self.signal_length - window_length + 1, hop_length):
                yield self[b, ..., start:start + window_length]

    def collect_windows(self, window_duration: float, hop_duration: float, preprocess: bool = True):
        """All windows stacked along the batch axis: [B*C*num_windows, 1, window] (ref :70-108)."""
        if preprocess:
            window_length, hop_length = self._preprocess_signal_for_windowing(window_duration, hop_duration)
        else:
            window_length, hop_length = int(window_duration * self.sample_rate), int(hop_duration * self.sample_rate)
        rows = self.audio_data.reshape(-1, self.signal_length)
        self.audio_data = rows.unfold(-1, window_length, hop_length).reshape(-1, 1, window_length).contiguous()
        return self

    def overlap_and_add(self, hop_duration: float):
        """Inverse of :meth:`collect_windows`: overlap-add the windows, divide by the number of windows covering each
        sample, drop the padding (ref :110-151)."""
        hop_length = int(hop_duration * self.sample_rate)
        window_length = self.signal_length
        nb, nch = self._original_batch_size, self._original_num_channels
        total = self._padded_signal_length
        wins = self.audio_data.reshape(nb * nch, -1, window_length)
        num = wins.shape[1]
        idx = (torch.arange(num, device=wins.device)[:, None] * hop_length
               + torch.arange(window_length, device=wins.device)[None, :]).reshape(-1)
        folded = torch.zeros(nb * nch, total, dtype=wins.dtype, device=wins.device)
        folded.index_add_(1, idx, wins.reshape(nb * nch, -1))
        norm = torch.zeros(total, dtype=wins.dtype, device=wins.device)
        norm.index_add_(0, idx, torch.ones(idx.numel(), dtype=wins.dtype, device=wins.device))
        self.audio_data = (folded / norm).reshape(nb, nch, -1)
        self.trim(hop_length, hop_length)
        return self

    def low_pass(self, cutoffs, zeros: int = 51, _bypass=None):
        """Low-pass each item at its own cutoff (Hz).  ``_bypass`` [B] (bool): items left untouched (how a transform
        applies itself to the items its mask selects without gathering / scattering the batch)."""
        cutoffs = util.ensure_tensor(util.host_view(cutoffs), 2, self.batch_size)  # host mirror first: no sync
        self.audio_data = _engine().sinc_filter(self._materialized(), cutoffs[:, 0], self.sample_rate, zeros,
                                                highpass=False, bypass=_bypass)
        self.stft_data = None
        return self

    def high_pass(self, cutoffs, zeros: int = 51, _bypass=None):
        """High-pass each item at its own cutoff (Hz): ``x - low_pass(x)``."""
        cutoffs = util.ensure_tensor(util.host_view(cutoffs), 2, self.batch_size)
        self.audio_data = _engine().sinc_filter(self._materialized(), cutoffs[:, 0], self.sample_rate, zeros,
                                                highpass=True, bypass=_bypass)
        self.stft_data = None
        return self

    def preemphasis(self, coef: float = 0.85):
        """The reference's pre-emphasis filter (ref :372-390): ``conv1d`` with the kernel ``[1, -coef, 0]`` and one
        sample of zero padding, i.e. ``y[n] = x[n-1] - coef * x[n]`` -- one launch of the direct FIR kernel."""
        x = self._materialized()
        taps = torch.tensor([[1.0, -float(coef), 0.0]], dtype=torch.float32, device=x.device)
        rows = x.shape[0] * x.shape[1]
        self.audio_data = _engine().fir_direct(x, taps, rows_per_filt=rows, left0=1, stride=1, pad_mode="constant")
        return self

    # ------------------------------------------------------------------ spectral masks (ref :217-370)
    def _band_mask(self, lo, hi, axis_vals, axis: int, val: float):
        if self.stft_data is None:
            self.stft()
        # ref :249 / :300 ``assert torch.all(lo < hi)``: checked on the host mirrors when there are some (no sync)
        h_lo, h_hi = torch.as_tensor(util.host_view(lo)).float(), torch.as_tensor(util.host_view(hi)).float()
        assert bool(torch.all(h_lo < h_hi)), "mask band must satisfy min < max"
        lo = util.ensure_tensor(lo, ndim=1).float().reshape(-1)
        hi = util.ensure_tensor(hi, ndim=1).float().reshape(-1)
        spec = self.stft_data
        if spec.dtype != torch.complex64 or not spec.is_contiguous():
            spec = spec.to(torch.complex64).contiguous()
        if _grad.wants_grad(spec):
            self.stft_data = _grad.SpecBandMask.apply(spec, axis_vals, lo, hi, axis, val)
        else:
            self.stft_data = _engine().spec_band_mask(spec, axis_vals, lo, hi, axis, val)
        return self

    def mask_frequencies(self, fmin_hz, fmax_hz, val: float = 0.0):
        """Fill the band ``fmin_hz <= f < fmax_hz`` (per item) of ``stft_data`` with ``val`` (magnitude and phase):
        SpecAugment (ref :217-264).  Cells outside the band keep their value; the reference rebuilds them as
        ``|X| exp(1j angle X)``, which differs from X by float32 rounding only."""
        if self.stft_data is None:
            self.stft()
        nbins = self.stft_data.shape[-2]
        bins_hz = torch.linspace(0, self.sample_rate / 2, nbins, device=self.device)  # the reference's own grid
        return self._band_mask(fmin_hz, fmax_hz, bins_hz, 0, val)

    def mask_timesteps(self, tmin_s, tmax_s, val: float = 0.0):
        """Fill the frames ``tmin_s <= t < tmax_s`` (per item) of ``stft_data`` with ``val`` (ref :266-306)."""
        if self.stft_data is None:
            self.stft()
        nt = self.stft_data.shape[-1]
        bins_t = torch.linspace(0, self.signal_duration, nt, device=self.device)
        return self._band_mask(tmin_s, tmax_s, bins_t, 1, val)

    def mask_low_magnitudes(self, db_cutoff, val: float = 0.0):
        """Fill magnitudes whose ``log_magnitude()`` is below ``db_cutoff`` (per item) with ``val``, keeping the phase
        (ref :308-333): one reduction pass for ``log_magnitude``'s global top_db floor, one masking pass."""
        if self.stft_data is None:
            self.stft()
        cut = util.ensure_tensor(db_cutoff, ndim=1).float().reshape(-1)
        if _grad.wants_grad(self.stft_data):
            spec = self.stft_data
            if spec.dtype != torch.complex64 or not spec.is_contiguous():
                spec = spec.to(torch.complex64).contiguous()
            self.stft_data = _grad.SpecMaskLow.apply(spec, cut, val)
        else:
            self.stft_data = _engine().spec_mask_low(self.stft_data, cut, val)
        return self

    def shift_phase(self, shift):
        """``phase += shift`` (ref :335-351), i.e. ``stft_data *= exp(1j * shift)`` in one pass.  ``shift``: a scalar,
        one value per item, or a tensor shaped like ``stft_data`` (per cell); other broadcast shapes are expanded."""
        if self.stft_data is None:
            self.stft()
        shift = util.ensure_tensor(shift, ndim=self.stft_data.ndim).float()
        B = self.stft_data.shape[0]
        if shift.numel() not in (1, B) or (shift.numel() == B and shift.shape[0] != B):
            shift = shift.to(self.device).expand(self.stft_data.shape).contiguous()
        self.stft_data = _engine().spec_rotate(self.stft_data, shift)
        return self

    def corrupt_phase(self, scale):
        """``phase += scale * N(0, 1)`` drawn on the signal's device (ref :353-369)."""
        if self.stft_data is None:
            self.stft()
        scale = util.ensure_tensor(scale, ndim=self.stft_data.ndim).float().to(self.device)
        noise = torch.randn(self.stft_data.shape, dtype=torch.float32, device=self.device)
        return self.shift_phase(scale * noise)
