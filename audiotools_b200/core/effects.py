"""``EffectMixin`` / ``ImpulseResponseMixin``: loudness normalisation, gain, mixing, mel-band
equaliser, impulse-response convolution and pitch shift with the method surface of
ref:audiotools/core/effects.py, on the sm_90a engine."""
import numpy as np
import torch

from . import grad as _grad
from . import util


def _engine():
    from ..engine import get_engine

    return get_engine()


def _on_engine(t) -> bool:
    """The kernels take this tensor: a CUDA tensor -- or, in the CPU tests, any tensor when the engine is the
    simulated build of the same kernel sources (``require_cuda=False``); plain CPU tensors otherwise keep the
    container's tensor arithmetic (host-logic tests)."""
    return t.is_cuda or not _engine().require_cuda


class EffectMixin:
    GAIN_FACTOR = np.log(10) / 20
    """Gain factor for converting between amplitude and decibels."""

    def mix(self, other, snr=10, other_eq=None):
        """Add ``other`` at the given signal-to-noise ratio (dB), optionally equalised first (ref :27-64)."""
        _grad.refuse_param_grad("mix", "snr", snr)
        snr = util.ensure_tensor(snr).to(self.device)
        other.zero_pad(0, max(0, self.signal_length - other.signal_length))
        other.truncate_samples(self.signal_length)
        if other_eq is not None:
            other = other.equalizer(other_eq)
        other = other.normalize(self.loudness() - snr)
        if _on_engine(self._audio_data):  # the noise's deferred normalisation gain and the add: one pass (csrc/effects.cu)
            g, other._pending_gain = other._pending_gain, None
            if _grad.wants_grad(self._audio_data) or _grad.wants_grad(other._audio_data):
                mixed = _grad.Mix.apply(self._materialized(), other._audio_data, g)
            else:
                mixed = _engine().mix(self._materialized(), other._audio_data, g)
            if g is not None:
                other._pending_gain = g  # `other` keeps its own (still deferred) state
            self.audio_data = mixed
        else:
            self.audio_data = self.audio_data + other.audio_data
        return self

    def convolve(self, other, start_at_max: bool = True, _bypass=None):
        """CIRCULAR convolution with ``other`` (period = signal length), the IR rolled so that its
        peak sits at t=0 and scaled by 1/max|IR| (ref :66-123).  ``_bypass`` [B]: items left untouched."""
        x = self._materialized()
        if _grad.wants_grad(x):
            _grad.refuse_param_grad("convolve", "the impulse response", other.audio_data)
            self.audio_data = _grad.CircConv.apply(x, other.audio_data, start_at_max, _bypass)
            return self
        self.audio_data = _engine().circular_convolve(x, other.audio_data, roll_to_peak=start_at_max, bypass=_bypass)
        return self

    def __matmul__(self, other):
        return self.convolve(other)

    def apply_ir(self, ir, drr=None, ir_eq=None, use_original_phase: bool = False, _bypass=None):
        """Equalise / DRR-alter the impulse response, convolve, restore the input's peak (ref :125-179).
        ``_bypass`` [B] (bool, device): items left untouched (mask-aware transforms)."""
        if ir_eq is not None:
            ir = ir.equalizer(ir_eq)
        if drr is not None:
            ir = ir.alter_drr(drr)
        return self._convolve_keeping_peak(lambda: self.convolve(ir, _bypass=_bypass), use_original_phase, _bypass)

    def apply_moving_ir(self, irs, hop: int, use_original_phase: bool = False, _bypass=None):
        """``apply_ir`` for a moving source or microphone (an extension; DESIGN.md K22): ``irs`` [B, K, C, L] (or
        [B, K, 1, L], shared by the channels) holds one impulse response per waypoint, waypoint k at sample k ``hop``.
        The output crossfades the K circular convolutions linearly between neighbouring waypoints, the last one
        holding to the end; every waypoint of an (item, channel) row is rolled and scaled by the row's first waypoint,
        so a change in delay along the path is heard.  Then each row's input peak is restored as ``apply_ir`` does.
        ``hop`` >= 1024 samples and K = (T - 1) // hop + 1, else ``ValueError``.  There is no backward: a signal or
        ``irs`` that requires a gradient raises ``NotImplementedError``.  ``_bypass`` [B]: items left untouched."""
        for name, t in (("the signal", self._materialized()), ("the impulse responses", irs)):
            if _grad.wants_grad(t):
                raise NotImplementedError(f"apply_moving_ir: {name} requires a gradient, and the moving convolution "
                                          "has no backward; call it under torch.no_grad() or on detached tensors")

        def convolve():
            self.audio_data = _engine().circular_convolve_moving(self._materialized(), irs, hop, bypass=_bypass)

        return self._convolve_keeping_peak(convolve, use_original_phase, _bypass)

    def _convolve_keeping_peak(self, convolve, use_original_phase: bool, _bypass):
        """Run ``convolve()`` on this signal, optionally put the input's phase back, and scale every (item, channel)
        row back to its input peak (ref :125-179)."""
        cuda = _on_engine(self._audio_data)
        x0 = self._materialized()
        # the peaks are values here; with a gradient, PeakScale's backward differentiates through them
        max_spk = _engine().row_absmax(x0.detach()) if cuda else \
            self.audio_data.abs().max(dim=-1, keepdims=True).values
        phase = self.phase if use_original_phase else None
        convolve()
        if use_original_phase:
            self.stft()
            self.stft_data = self.magnitude * torch.exp(1j * phase)
            self.istft()

        def restore(y):
            max_transformed = _engine().row_absmax(y.detach()) if cuda else y.abs().max(dim=-1, keepdims=True).values
            scale = max_spk.clamp(1e-8) / max_transformed.clamp(1e-8)
            if _bypass is not None:
                byp = torch.as_tensor(_bypass).to(scale.device).bool().reshape(-1, 1, 1)
                scale = torch.where(byp, torch.ones_like(scale), scale)
            if cuda:  # per-row scale: the gain kernel with one "item" per (batch, channel) row
                return _engine().gain(y.reshape(-1, 1, y.shape[-1]), scale.reshape(-1)).reshape(y.shape)
            return y * scale

        y = self._materialized() if cuda else self.audio_data
        if cuda and _grad.wants_grad(y):
            self.audio_data = _grad.PeakScale.apply(y, x0, 1.0, _bypass, restore)
        else:
            self.audio_data = restore(y)
        return self

    def ensure_max_of_audio(self, max: float = 1.0):
        """Scale every (item, channel) row whose peak exceeds ``max`` down to it (ref :181-198): a peak pass and a
        scale pass of csrc/effects.cu."""
        if _on_engine(self._audio_data):
            x = self._materialized()
            if _grad.wants_grad(x):
                self.audio_data = _grad.PeakScale.apply(x, None, float(max), None,
                                                        lambda y: _engine().limit_peak(y, float(max)))
            else:
                self.audio_data = _engine().limit_peak(x, float(max))
            return self
        peak = self.audio_data.abs().max(dim=-1, keepdims=True)[0]
        peak_gain = torch.where(peak > max, max / peak, torch.ones_like(peak))  # no boolean-mask host sync
        self.audio_data = self.audio_data * peak_gain
        return self

    def normalize(self, db=-24.0, _bypass=None, *, true_peak_limit=None):
        """Scale every item to ``db`` LUFS (scalar or [B]) (ref :200-220).  The per-item gain comes
        out of the loudness kernel; the multiply is deferred and fused into the next kernel that
        reads the samples (``stft`` / ``mel_spectrogram``) or materialised on first access.

        ``true_peak_limit`` (dBTP, scalar or [B]; an extension): an item whose true peak (``true_peak()``, measured
        before the gain) would exceed the limit after normalisation gets the smaller gain that puts it at the limit,
        ``min(gain, 10^((limit - true_peak) / 20))``, so it ends below ``db`` LUFS.  Other items keep the gain they
        get without a limit, bit for bit.  The gain stays a constant of the backward pass.  To keep the loudness and
        still meet a ceiling, follow ``normalize(db)`` with :meth:`limit`, which reshapes the waveform around the overs."""
        db = util.ensure_tensor(db).to(self.device).float().reshape(-1)
        if self._loudness is None and self._pending_gain is None:
            T = self.signal_length
            padded = T
            if self.signal_duration < 0.5:
                padded = T + int((0.5 - self.signal_duration) * self.sample_rate)
            # the gain is a constant: gradients reach audio_data through the gain op, not the loudness
            out = _engine().lufs(self._audio_data.detach(), self.sample_rate, padded_length=padded, target_db=db)
            gain = out["gain"]
            measured = out["loud"]
        else:
            measured = self.loudness()
            gain = torch.exp((db - measured) * float(np.float32(self.GAIN_FACTOR)))
        if true_peak_limit is not None:
            limit = float(true_peak_limit) if isinstance(true_peak_limit, (int, float)) else \
                util.ensure_tensor(true_peak_limit).to(gain.device).float().reshape(-1)  # a number needs no copy
            peak = _engine().true_peak(self._audio_data.detach(), self.sample_rate)["db"]
            cap = torch.exp((limit - peak) * float(np.float32(self.GAIN_FACTOR)))
            if self._pending_gain is not None:  # still deferred (a cached loudness was used): it scales the peak too
                cap = cap / self._pending_gain
            gain = torch.minimum(gain, cap)
        if _bypass is not None:  # items the transform's mask does not select keep their samples (gain exactly 1)
            gain = torch.where(torch.as_tensor(_bypass).to(gain.device).bool().reshape(-1), torch.ones_like(gain), gain)
        self._defer_gain(gain)
        self._measured_loudness = measured  # extension: the LUFS the gain was derived from (logging / statistics)
        return self

    def limit(self, ceiling_db=-1.0, lookahead: float = 0.0015, release: float = 0.05):
        """Look-ahead true-peak limiter (an extension; DESIGN.md K18): every item is multiplied by one gain series,
        shared by its channels, that dips around each instant where the true-peak envelope (``true_peak()``'s
        interpolator) passes ``ceiling_db`` (dBTP, scalar or [B]) and is exactly 1 elsewhere, so
        ``normalize(-16).limit(-1)`` keeps the loudness that a whole-item cap would give up.  ``lookahead`` (s) is the
        hold before an over and the length of the box attack, ``release`` (s) the time constant of the recovery; the
        windows are centred, so nothing is delayed.  Samples away from every over, and items that never pass the
        ceiling, come back bit for bit.  A gain deferred by ``normalize`` / ``volume_change`` is applied inside the
        limiter's own passes.  No backward: a signal that requires a gradient raises ``NotImplementedError``."""
        if not isinstance(ceiling_db, (int, float)):  # a number needs no copy to the device
            ceiling_db = util.ensure_tensor(ceiling_db).to(self.device).float().reshape(-1)
        # the setter drops the consumed gain and the loudness cache
        self.audio_data = _engine().limit(self._audio_data, self.sample_rate, ceiling_db, lookahead, release,
                                          gain=self._pending_gain)
        self.stft_data = None
        return self

    def sos_filter(self, sos, zero_phase: bool = False, _bypass=None):
        """Filter every item with a cascade of second-order sections (an extension; DESIGN.md K19):
        ``scipy.signal.sosfilt(sos, x)`` with zero initial state, run exactly (no warm-up, no FIR approximation) on
        the GPU.  ``sos`` is [S, 6] for the whole batch or [B, S, 6] per item (1 <= S <= 8), rows
        ``b0 b1 b2 a0 a1 a2``; each row is divided by its a0 and rounded to float32 once.  All channels of an item use
        its sections.  An item with a section whose poles are not strictly inside the unit circle comes back all NaN;
        a NaN or inf sample makes its row non-finite from that sample on.  ``zero_phase=True`` runs
        ``scipy.signal.sosfiltfilt(sos, x)`` with scipy's defaults instead (odd extension, each item's default
        padlen; the signal must be longer than 3 (2S + 1) samples): forwards and backwards, so no sample moves, and a
        NaN or inf sample makes its whole row non-finite.  A gain deferred by ``normalize`` / ``volume_change`` is
        applied inside the filter's own passes.  Differentiable with respect to ``audio_data``; ``sos`` is a constant.
        ``_bypass`` [B]: items given identity sections, which return their samples unchanged."""
        _grad.refuse_param_grad("sos_filter", "sos", sos)
        x = self._audio_data
        eng = _engine()
        sos = eng.sos_coefficients(sos, self.batch_size, x.device)
        if _bypass is not None:
            ident = (torch.arange(6, device=sos.device) % 3 == 0).to(sos.dtype)  # 1 0 0 1 0 0, built without a copy
            byp = torch.as_tensor(_bypass).to(sos.device).bool().reshape(-1, 1, 1)
            sos = torch.where(byp, ident, sos.expand(self.batch_size, -1, -1)).contiguous()
        gain = self._pending_gain
        if zero_phase:
            if _grad.wants_grad(x):
                y = _grad.SOSFiltFilt.apply(x, sos, gain, "odd", None)
            else:
                y = eng.sos_filtfilt(x, sos, gain=gain)
        elif _grad.wants_grad(x):
            y = _grad.SOSFilter.apply(x, sos, gain)
        else:
            y = eng.sos_filter(x, sos, gain=gain)
        self.audio_data = y  # the setter drops the consumed gain and the loudness cache
        self.stft_data = None
        return self

    def parametric_eq(self, kind, freq, gain_db=0.0, q=0.7071, _bypass=None):
        """Parametric equaliser (an extension): one RBJ Audio EQ Cookbook biquad per band and per item
        (``core/biquad.py``), run as one :meth:`sos_filter` cascade.  ``kind``: one of ``peaking``, ``low_shelf``,
        ``high_shelf``, ``low_pass``, ``high_pass``, ``band_pass``, ``notch``, ``all_pass``, or a list of n_bands of
        them.  ``freq`` (Hz, in (0, sr/2)), ``gain_db`` (peaking and shelves) and ``q`` (> 0): numbers, [n_bands] or
        [B, n_bands]; they are checked on host values, so a transform's parameter table costs no synchronisation.
        Gradients reach ``audio_data`` only: a parameter that requires one raises ``NotImplementedError``."""
        from . import biquad

        for name, v in (("freq", freq), ("gain_db", gain_db), ("q", q)):
            _grad.refuse_param_grad("parametric_eq", name, v)
        kinds = [kind] if isinstance(kind, str) else list(kind)
        biquad.check(kinds, freq, q, self.sample_rate)
        sos = biquad.design(kinds, freq, gain_db, q, self.sample_rate, self.batch_size, self.device)
        return self.sos_filter(sos, _bypass=_bypass)

    def volume_change(self, db, _bypass=None):
        """Multiply every item by ``10**(db/20)`` (ref :222-238)."""
        db = util.ensure_tensor(db, ndim=1).to(self.device).float()
        gain = torch.exp(db * float(np.float32(self.GAIN_FACTOR)))
        if _bypass is not None:
            gain = torch.where(torch.as_tensor(_bypass).to(gain.device).bool().reshape(-1), torch.ones_like(gain), gain)
        self._defer_gain(util.ensure_tensor(gain, 1, self.batch_size))
        return self

    def pitch_shift(self, n_semitones, quick: bool = True):
        """Shift the pitch of every item by ``n_semitones`` keeping the length (ref :247-277, SoX there).  Extension:
        ``n_semitones`` may also hold one shift per item (list / tensor of batch_size values, read on the host)."""
        shifts = util.host_view(n_semitones) if torch.is_tensor(n_semitones) else n_semitones
        if not torch.is_tensor(shifts) and np.ndim(shifts) == 0:
            shifts = float(shifts)
        self.audio_data = _engine().pitch_shift(self._materialized(), self.sample_rate, shifts, quick=quick)
        return self

    def time_stretch(self, factor: float, quick: bool = True):
        """Change the speed by ``factor`` (duration / factor) keeping the pitch (ref :279-309, SoX ``tempo`` there):
        the WSOLA search + overlap-add stages of :meth:`pitch_shift`.  Like SoX's output it is pinned by properties
        only (duration, pitch, batch == single)."""
        self.audio_data = _engine().time_stretch(self._materialized(), self.sample_rate, float(factor))
        return self

    def apply_codec(self, *args, **kwargs):
        raise NotImplementedError("apply_codec calls external lossy codecs: out of scope (SURVEY.md §2 row 3)")

    def mel_filterbank(self, n_bands: int):
        """Split into ``n_bands`` mel-spaced bands -> [B, C, T, n_bands] (ref :386-403)."""
        return _engine().mel_filterbank(self._materialized(), self.sample_rate, n_bands)

    def equalizer(self, db, _bypass=None):
        """Mel-spaced band equaliser; band weights are ``10**db`` exactly as in the reference (ref :405-433).
        The band split and the weighted sum collapse into ONE FIR per item.  ``_bypass`` [B]: items left untouched."""
        db = util.ensure_tensor(db)
        if db.ndim == 2:
            if db.shape[0] != 1:
                assert db.shape[0] == self.batch_size
        else:
            db = db.unsqueeze(0)
        x = self._materialized()
        if _grad.wants_grad(x):
            _grad.refuse_param_grad("equalizer", "db", db)
            self.audio_data = _grad.Equalizer.apply(x, self.sample_rate, db.to(self.device), _bypass)
            return self
        self.audio_data = _engine().equalizer(x, self.sample_rate, db.to(self.device), bypass=_bypass)
        return self

    def clip_distortion(self, clip_percentile):
        """Clip at the ``clip_percentile / 2`` and ``1 - clip_percentile / 2`` quantiles (ref :435-461).  The reference
        indexes ``torch.quantile``'s [Q, B, C] result as [:, :nc, :], i.e. item i is clipped at the quantiles q_i of
        ROW 0 of the batch (and the call only broadcasts for mono signals); reproduced as is: radix-selected order
        statistics of row 0 + one clamp pass (csrc/effects.cu), no sort."""
        clip_percentile = util.ensure_tensor(clip_percentile, ndim=1)
        if _on_engine(self._audio_data) and self.num_channels == 1:
            x = self._materialized()
            q = clip_percentile.to(x.device).float().reshape(-1)
            if q.numel() == 1:
                q = q.expand(self.batch_size)
            assert q.numel() == self.batch_size
            thr = _engine().quantile(x[0, 0], torch.cat([q / 2, 1 - (q / 2)]))
            self.audio_data = _engine().clamp_items(x, thr[: self.batch_size], thr[self.batch_size:])
            return self
        min_thresh = torch.quantile(self.audio_data, clip_percentile / 2, dim=-1)
        max_thresh = torch.quantile(self.audio_data, 1 - (clip_percentile / 2), dim=-1)
        nc = self.audio_data.shape[1]
        self.audio_data = self.audio_data.clamp(min_thresh[:, :nc, :], max_thresh[:, :nc, :])
        return self

    def quantization(self, quantization_channels):
        if _on_engine(self._audio_data):
            q = util.ensure_tensor(quantization_channels, ndim=1)
            self.audio_data = self._straight_through(lambda x: _engine().quantize(x, q))
            return self
        q = util.ensure_tensor(quantization_channels, ndim=3).to(self.device)
        x = self.audio_data
        x = (x + 1) / 2
        x = (x * q).floor() / q
        self.audio_data = 2 * x - 1
        return self

    def _straight_through(self, fwd):
        """``fwd`` of the samples; with a gradient, the identity backward of the reference's x - (x - q).detach()."""
        x = self._materialized()
        return _grad.StraightThrough.apply(x, fwd) if _grad.wants_grad(x) else fwd(x)

    def mulaw_quantization(self, quantization_channels):
        if _on_engine(self._audio_data):
            q = util.ensure_tensor(quantization_channels, ndim=1)
            self.audio_data = self._straight_through(lambda x: _engine().quantize(x, q, mulaw=True))
            return self
        mu = util.ensure_tensor(quantization_channels, ndim=3).to(self.device) - 1.0
        x = self.audio_data
        x = torch.sign(x) * torch.log1p(mu * torch.abs(x)) / torch.log1p(mu)
        x = ((x + 1) / 2 * mu + 0.5).to(torch.int64)
        x = (x / mu) * 2 - 1.0
        self.audio_data = torch.sign(x) * (torch.exp(torch.abs(x) * torch.log1p(mu)) - 1.0) / mu
        return self


class ImpulseResponseMixin:
    """Impulse-response augmentation of Bryan (ICASSP 2020): early/late split around the direct
    path, DRR measurement and alteration (ref :529-647)."""

    def decompose_ir(self):
        x = self.audio_data
        td = torch.argmax(x, dim=-1, keepdim=True)
        t0 = int(self.sample_rate * 0.0025)
        idx = torch.arange(x.shape[-1], device=self.device)[None, None, :].expand(self.batch_size, -1, -1)
        early_idx = (idx >= td - t0) * (idx <= td + t0)
        early = torch.where(early_idx, x, torch.zeros_like(x))
        late = torch.where(early_idx, torch.zeros_like(x), x)
        # ref :569-573 fills window[b, ..., widx] with get_window("hann", widx.shape[-1]) where widx =
        # early_idx[b, 0].nonzero() has shape [n, 1]: the window length is always 1 (scipy's hann(1) == [1.0])
        # and channel 0's early region is used for every channel.  Same values without the per-item loop, its
        # nonzero() host synchronisations and the per-item host->device window copies:
        window = early_idx[:, :1].to(x.dtype).expand_as(x)
        return early, late, window

    def measure_drr(self):
        early, late, _ = self.decompose_ir()
        return 10 * torch.log10((early ** 2).sum(dim=-1) / (late ** 2).sum(dim=-1))

    @staticmethod
    def solve_alpha(early_response, late_field, wd, target_drr):
        e_sq = early_response ** 2
        a = ((wd ** 2) * e_sq).sum(dim=-1)
        b = (2 * (1 - wd) * wd * e_sq).sum(dim=-1)
        c = (((1 - wd) ** 2) * e_sq).sum(dim=-1) - torch.pow(10, target_drr / 10) * (late_field ** 2).sum(dim=-1)
        expr = ((b ** 2) - 4 * a * c).sqrt()
        return torch.maximum((-b - expr) / (2 * a), (-b + expr) / (2 * a))

    def alter_drr(self, drr):
        if _on_engine(self._audio_data):  # one fused launch (csrc/effects.cu) instead of ~25 tensor passes
            self.audio_data = _engine().alter_drr(self._materialized(), self.sample_rate,
                                                  util.ensure_tensor(drr, 2, self.batch_size))
            return self
        drr = util.ensure_tensor(drr, 2, self.batch_size).to(self.device)
        early, late, window = self.decompose_ir()
        alpha = self.solve_alpha(early, late, window, drr)
        if _on_engine(self._audio_data):
            min_alpha = (_engine().row_absmax(late) / _engine().row_absmax(early))[..., 0]
        else:
            min_alpha = late.abs().max(dim=-1)[0] / early.abs().max(dim=-1)[0]
        alpha = torch.maximum(alpha, min_alpha)[..., None]
        self.audio_data = alpha * window * early + ((1 - window) * early) + late
        self.ensure_max_of_audio()
        return self
