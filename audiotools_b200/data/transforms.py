"""Batched, seed-reproducible transforms with the API of ref:audiotools/data/transforms.py.

A transform has two halves.  ``instantiate(state, signal)`` draws its parameters on the host from
distribution tuples with a ``numpy.random.RandomState`` (so a seed reproduces them) and returns a
nested dict keyed by the transform's name; ``transform(signal, **kwargs)`` applies it to a whole
batch on the device, gated per item by the boolean ``mask`` drawn with probability ``prob``.
``Compose`` names its children ``"{position}.{Name}"`` and threads the same nested dict through
them; ``Choose`` turns the children's masks into a one-hot choice.

Every concrete transform is one ``AudioSignal`` method, i.e. one or two launches of ``libb2a``.
Transforms of the reference that need file-backed loaders (``BackgroundNoise``, ``CrossTalk``,
file-based ``RoomImpulseResponse``) take in-memory ``AudioSignal`` pools here instead: decoding
audio files is outside the accelerated hot path (SURVEY.md §2 row 7).
"""
import copy
from contextlib import contextmanager
from inspect import signature
from typing import List

import numpy as np
import torch
from numpy.random import RandomState

from ..core import AudioSignal
from ..core import util
from ..core.audio_signal import _on_engine

tt = torch.tensor
"""Shorthand for converting things to torch.tensor."""


# ------------------------------------------------------------------------------------------
# Parameter tables.  A transform draws its parameters as PLAIN host values (python / numpy scalars, small arrays,
# AudioSignals) -- the RNG calls and their order are the reference's, so a seed reproduces them -- and they only become
# tensors once per batch: ``batch_instantiate`` stacks the B draws of every parameter into ONE tensor per key
# (the reference builds B x n_keys zero-dim tensors and collates them), ``instantiate`` tensorises a single draw.  ``util.prepare_batch`` then uploads each
# table once and keeps its host mirror, so mask / cutoff / shift decisions never synchronise with the device.
# ------------------------------------------------------------------------------------------
def _tensorize(value):
    """One draw -> the reference's ``instantiate`` output: every leaf a tensor (``torch.tensor(v)``)."""
    if isinstance(value, dict):
        return {k: _tensorize(v) for k, v in value.items()}
    if isinstance(value, (list, tuple)):
        return [_tensorize(v) for v in value]
    if isinstance(value, (AudioSignal, torch.Tensor)):
        return value
    return tt(value)


def _stack_leaf(vals: list):
    """B draws of one parameter -> one [B, ...] tensor with the dtype ``default_collate([torch.tensor(v) ...])`` gives."""
    v0 = vals[0]
    if isinstance(v0, AudioSignal):
        return AudioSignal.batch(list(vals), pad_signals=True)
    if isinstance(v0, torch.Tensor):
        return torch.stack(list(vals))
    if isinstance(v0, (list, tuple)):  # e.g. Choose's one_hot: a list of per-child flags -> a list of [B] tensors
        return [_stack_leaf([v[i] for v in vals]) for i in range(len(v0))]
    dtype = tt(v0).dtype  # python float -> float32, python int -> int64, bool -> bool, numpy scalars / arrays keep theirs
    arr = np.asarray(vals)
    return torch.as_tensor(arr).to(dtype) if arr.dtype != object else torch.stack([tt(v) for v in vals])


def _host_values(v, dtype=np.float64) -> np.ndarray:
    """A drawn parameter (host values, or a tensor read through its host mirror: no device sync) as a numpy array."""
    if torch.is_tensor(v):
        v = util.host_view(v).detach().cpu().numpy()
    return np.asarray(v, dtype=dtype)


def _collate_draws(draws: list):
    flats = [util.flatten(d) for d in draws]
    return util.unflatten({k: _stack_leaf([f[k] for f in flats]) for k in flats[0]})


class BaseTransform:
    def __init__(self, keys: list = [], name: str = None, prob: float = 1.0):
        # parameter names come from the _transform signature (everything but signal / kwargs)
        params = signature(self._transform).parameters
        tfm_keys = [k for k in params.keys() if k not in ("signal", "kwargs", "_bypass")]
        self.keys = keys + tfm_keys + ["mask"]
        # mask-aware: ``_transform(signal, ..., _bypass=[B] bool)`` runs on the WHOLE batch and leaves the flagged items
        # untouched inside the kernels (csrc: bypass flags / unit gains / zero shifts): no gather, no scatter
        # ... where that pays: `_bypass_pays = False` marks the FFT-convolution transforms, whose forward block FFTs run
        # for every row of the launch, flagged or not, so those keep the gather (at prob 0.5: half the rows, two cheap
        # copies)
        self._mask_aware = "_bypass" in params and getattr(self, "_bypass_pays", True)
        self.prob = prob
        self.name = self.__class__.__name__ if name is None else name
        self._needs_signal = "signal" in signature(self._instantiate).parameters  # inspected once, not per item

    def _prepare(self, batch: dict):
        sub_batch = batch[self.name]
        for k in self.keys:
            assert k in sub_batch.keys(), f"{k} not in batch"
        return sub_batch

    def _transform(self, signal):
        return signal

    def _instantiate(self, state: RandomState, signal: AudioSignal = None):
        return {}

    @staticmethod
    def apply_mask(batch: dict, mask: torch.Tensor):
        return util.unflatten({k: v[mask] for k, v in util.flatten(batch).items()})

    def transform(self, signal: AudioSignal, **kwargs):
        """``signal[mask] = self._transform(signal[mask], **kwargs[mask])`` (ref :133-166).  When every item is
        selected the gather / scatter copies of the whole batch are skipped and the transform runs on ``signal``
        itself, leaving the same state the masked round trip leaves (samples replaced; a loudness / STFT cache is
        only overwritten when both sides hold one, :1658-1679).  The mask is read from its host mirror
        (``util.prepare_batch``) when there is one: no device synchronisation."""
        tfm_kwargs = self._prepare(kwargs)
        mask = tfm_kwargs["mask"]
        host_mask = util.host_view(mask)
        n_sel = int(host_mask.sum())
        if n_sel == 0:
            return signal
        if host_mask.ndim == 1 and n_sel == host_mask.numel() == signal.batch_size:
            tfm_kwargs = {k: v for k, v in tfm_kwargs.items() if k != "mask"}
            pre_loud, pre_stft = signal._loudness, signal.stft_data
            out = self._transform(signal, **tfm_kwargs)
            if out is signal:
                new_loud, new_stft = signal._loudness, signal.stft_data
                signal._loudness = new_loud if (pre_loud is not None and new_loud is not None) else pre_loud
                signal.stft_data = new_stft if (pre_stft is not None and new_stft is not None) else pre_stft
                return signal
            signal[mask] = out
            return signal
        if self._mask_aware and host_mask.ndim == 1 and host_mask.numel() == signal.batch_size and \
                _on_engine(signal._audio_data) and self._bypass_ok(signal, tfm_kwargs):
            # the reference gathers signal[mask], transforms the copy and scatters it back (:133-166): two extra passes
            # over the selected items.  Here the kernels take the complement of the mask as per-item bypass flags.
            args = {k: v for k, v in tfm_kwargs.items() if k != "mask"}
            pre_loud, pre_stft = signal._loudness, signal.stft_data
            bypass = ~mask.to(signal.device).bool()
            if bypass.is_cuda:  # host mirror (the mask's own): host-side decisions on the flags need no sync
                bypass._b2a_host = (~host_mask.bool(), bypass._version)
            out = self._transform(signal, **args, _bypass=bypass)
            if out is signal:
                # state of `signal[mask] = out` (:1658-1679): caches are overwritten only where both sides hold one,
                # and only for the selected items
                new_loud, new_stft = signal._loudness, signal.stft_data
                sel = mask.to(signal.device).bool()
                if pre_loud is not None and new_loud is not None:
                    signal._loudness = torch.where(sel, new_loud, pre_loud)
                else:
                    signal._loudness = pre_loud
                if pre_stft is not None and new_stft is not None and pre_stft.shape == new_stft.shape:
                    signal.stft_data = torch.where(sel.reshape(-1, 1, 1, 1), new_stft, pre_stft)
                else:
                    signal.stft_data = pre_stft
                return signal
            signal[mask] = out[mask]
            return signal
        tfm_kwargs = self.apply_mask(tfm_kwargs, mask)
        tfm_kwargs = {k: v for k, v in tfm_kwargs.items() if k != "mask"}
        signal[mask] = self._transform(signal[mask], **tfm_kwargs)
        return signal

    def _bypass_ok(self, signal, tfm_kwargs) -> bool:
        """Per-call veto of the bypass-flag path (e.g. a filter long enough to go through the FFT engine)."""
        return True

    def __call__(self, *args, **kwargs):
        return self.transform(*args, **kwargs)

    def _draw(self, state: RandomState, signal: AudioSignal = None) -> dict:
        """One item's parameters as plain host values, keyed by the transform's name (mask last, as in the reference:
        ``state.rand() <= prob`` is drawn AFTER the parameters, ref :228-240)."""
        params = self._instantiate(state, signal) if self._needs_signal else self._instantiate(state)
        params["mask"] = bool(state.rand() <= self.prob)
        return {self.name: params}

    def instantiate(self, state: RandomState = None, signal: AudioSignal = None):
        return _tensorize(self._draw(util.random_state(state), signal))

    def batch_instantiate(self, states: list = None, signal: AudioSignal = None):
        """Parameters for a batch, one seed / state per item (ref :242-265): B draws, ONE tensor per parameter."""
        return _collate_draws([self._draw(util.random_state(state), signal) for state in states])


class Identity(BaseTransform):
    pass


class SpectralTransform(BaseTransform):
    """stft -> transform -> istft."""

    def transform(self, signal, **kwargs):
        signal.stft()
        super().transform(signal, **kwargs)
        signal.istft()
        return signal


class Compose(BaseTransform):
    def __init__(self, *transforms: list, name: str = None, prob: float = 1.0):
        if isinstance(transforms[0], list):
            transforms = transforms[0]
        for i, tfm in enumerate(transforms):
            tfm.name = f"{i}.{tfm.name}"
        keys = [tfm.name for tfm in transforms]
        super().__init__(keys=keys, name=name, prob=prob)
        self.transforms = transforms
        self.transforms_to_apply = keys

    @contextmanager
    def filter(self, *names: list):
        old = self.transforms_to_apply
        self.transforms_to_apply = names
        yield
        self.transforms_to_apply = old

    def _transform(self, signal, **kwargs):
        for transform in self.transforms:
            if any([x in transform.name for x in self.transforms_to_apply]):
                signal = transform(signal, **kwargs)
        return signal

    def _instantiate(self, state: RandomState, signal: AudioSignal = None):
        parameters = {}
        for transform in self.transforms:
            parameters.update(transform._draw(state, signal))
        return parameters

    def __getitem__(self, idx):
        return self.transforms[idx]

    def __len__(self):
        return len(self.transforms)

    def __iter__(self):
        for transform in self.transforms:
            yield transform


class Choose(Compose):
    def __init__(self, *transforms: list, weights: list = None, name: str = None, prob: float = 1.0):
        super().__init__(*transforms, name=name, prob=prob)
        if weights is None:
            n = len(self.transforms)
            weights = [1 / n for _ in range(n)]
        self.weights = np.array(weights)

    def _instantiate(self, state: RandomState, signal: AudioSignal = None):
        kwargs = super()._instantiate(state, signal)
        tfm_idx = state.choice(list(range(len(self.transforms))), p=self.weights)
        one_hot = []
        for i, t in enumerate(self.transforms):
            if kwargs[t.name]["mask"]:
                kwargs[t.name]["mask"] = bool(i == tfm_idx)
            one_hot.append(kwargs[t.name]["mask"])
        kwargs["one_hot"] = one_hot
        return kwargs


class Repeat(Compose):
    def __init__(self, transform, n_repeat: int = 1, name: str = None, prob: float = 1.0):
        super().__init__([copy.copy(transform) for _ in range(n_repeat)], name=name, prob=prob)
        self.n_repeat = n_repeat


class RepeatUpTo(Choose):
    def __init__(self, transform, max_repeat: int = 5, weights: list = None, name: str = None, prob: float = 1.0):
        transforms = [Repeat(transform, n_repeat=n) for n in range(1, max_repeat)]
        super().__init__(transforms, name=name, prob=prob, weights=weights)
        self.max_repeat = max_repeat


# ------------------------------------------------------------------------------------------
# concrete transforms (one AudioSignal method each)
# ------------------------------------------------------------------------------------------
class VolumeChange(BaseTransform):
    """``signal.volume_change(db)`` (ref :941-970)."""

    def __init__(self, db: tuple = ("uniform", -12.0, 0.0), name: str = None, prob: float = 1.0):
        super().__init__(name=name, prob=prob)
        self.db = db

    def _instantiate(self, state: RandomState):
        return {"db": util.sample_from_dist(self.db, state)}

    def _transform(self, signal, db, _bypass=None):
        return signal.volume_change(db, _bypass=_bypass)


class VolumeNorm(BaseTransform):
    """``signal.normalize(db)`` -- LUFS normalisation (ref :973-1003).  ``true_peak_limit`` (dBTP, an extension):
    passed to ``normalize``, which lowers the gain of items whose true peak would exceed it.  It is not drawn."""

    def __init__(self, db: tuple = ("const", -24), name: str = None, prob: float = 1.0, true_peak_limit: float = None):
        super().__init__(name=name, prob=prob)
        self.db = db
        self.true_peak_limit = true_peak_limit

    def _instantiate(self, state: RandomState):
        return {"db": util.sample_from_dist(self.db, state)}

    def _transform(self, signal, db, _bypass=None):
        return signal.normalize(db, _bypass=_bypass, true_peak_limit=self.true_peak_limit)


class Limiter(BaseTransform):
    """``signal.limit(ceiling)`` -- look-ahead true-peak limiter (an extension; the reference has none).  ``ceiling``
    (dBTP) is drawn per item; ``lookahead`` and ``release`` (seconds) are not drawn."""

    def __init__(self, ceiling: tuple = ("const", -1.0), lookahead: float = 0.0015, release: float = 0.05,
                 name: str = None, prob: float = 1.0):
        super().__init__(name=name, prob=prob)
        self.ceiling = ceiling
        self.lookahead = lookahead
        self.release = release

    def _instantiate(self, state: RandomState):
        return {"ceiling": util.sample_from_dist(self.ceiling, state)}

    def _transform(self, signal, ceiling):
        return signal.limit(ceiling, lookahead=self.lookahead, release=self.release)


class ParametricEQ(BaseTransform):
    """``signal.parametric_eq(kinds, freq, gain_db, q)`` -- a random parametric equaliser (an extension; the reference
    has none).  Each band is ``(kind, freq, gain_db, q)``: a cookbook kind (``core/biquad.py``) and three distribution
    tuples, drawn per item and per band.  Frequencies are drawn in Hz and kept below 0.45 of the signal's rate.  Items
    the mask does not select get identity sections and come back unchanged."""

    DEFAULT_BANDS = (("low_shelf", ("uniform", 40.0, 300.0), ("uniform", -12.0, 12.0), ("const", 0.7071)),
                     ("peaking", ("uniform", 200.0, 2000.0), ("uniform", -12.0, 12.0), ("uniform", 0.5, 4.0)),
                     ("peaking", ("uniform", 1000.0, 8000.0), ("uniform", -12.0, 12.0), ("uniform", 0.5, 4.0)),
                     ("high_shelf", ("uniform", 4000.0, 12000.0), ("uniform", -12.0, 12.0), ("const", 0.7071)))

    def __init__(self, bands: tuple = DEFAULT_BANDS, name: str = None, prob: float = 1.0):
        super().__init__(name=name, prob=prob)
        self.bands = tuple(bands)

    def _instantiate(self, state: RandomState, signal: AudioSignal):
        top = 0.45 * signal.sample_rate
        freq = [min(float(util.sample_from_dist(b[1], state)), top) for b in self.bands]
        gain_db = [float(util.sample_from_dist(b[2], state)) for b in self.bands]
        q = [float(util.sample_from_dist(b[3], state)) for b in self.bands]
        return {"freq": np.array(freq), "gain_db": np.array(gain_db), "q": np.array(q)}

    def _transform(self, signal, freq, gain_db, q, _bypass=None):
        return signal.parametric_eq([b[0] for b in self.bands], freq, gain_db, q, _bypass=_bypass)


class GlobalVolumeNorm(BaseTransform):
    """Normalise using the loudness of the whole source file, read from
    ``signal.metadata["loudness"]`` (ref :1006-1050)."""

    def __init__(self, db: tuple = ("const", -24), name: str = None, prob: float = 1.0):
        super().__init__(name=name, prob=prob)
        self.db = db

    def _instantiate(self, state: RandomState, signal: AudioSignal):
        if "loudness" not in signal.metadata:
            db_change = 0.0
        elif float(signal.metadata["loudness"]) == float("-inf"):
            db_change = 0.0
        else:
            db_change = util.sample_from_dist(self.db, state) - float(signal.metadata["loudness"])
        return {"db": db_change}

    def _transform(self, signal, db):
        return signal.volume_change(db)


class Equalizer(BaseTransform):
    """``signal.equalizer(eq)`` with ``eq = -eq_amount * rand(n_bands)`` (ref :564-600)."""
    _bypass_pays = False  # 641 taps: FFT convolution

    def __init__(self, eq_amount: tuple = ("const", 1.0), n_bands: int = 6, name: str = None, prob: float = 1.0):
        super().__init__(name=name, prob=prob)
        self.eq_amount = eq_amount
        self.n_bands = n_bands

    def _instantiate(self, state: RandomState):
        eq_amount = util.sample_from_dist(self.eq_amount, state)
        return {"eq": -eq_amount * state.rand(self.n_bands)}

    def _transform(self, signal, eq, _bypass=None):
        return signal.equalizer(eq, _bypass=_bypass)


class LowPass(BaseTransform):
    """``signal.low_pass(cutoff, zeros)`` (ref :1095-1131)."""

    def __init__(self, cutoff: tuple = ("choice", [4000, 8000, 16000]), zeros: int = 51, name: str = None,
                 prob: float = 1):
        super().__init__(name=name, prob=prob)
        self.cutoff = cutoff
        self.zeros = zeros

    def _instantiate(self, state: RandomState):
        return {"cutoff": util.sample_from_dist(self.cutoff, state)}

    def _transform(self, signal, cutoff, _bypass=None):
        return signal.low_pass(cutoff, zeros=self.zeros, _bypass=_bypass)

    def _bypass_ok(self, signal, tfm_kwargs) -> bool:
        # flags pay when the time-domain kernel serves the call (a flagged row is a plain copy); a bank long enough for
        # the FFT engine (> 320 taps) would spend its forward FFTs on the unselected rows as well: gather instead
        cut = util.host_view(tfm_kwargs["cutoff"]).reshape(-1).float()
        sel = util.host_view(tfm_kwargs["mask"]).reshape(-1).bool()
        if not bool(sel.any()) or float(cut[sel].min()) <= 0:
            return False
        return 2 * int(self.zeros / (float(cut[sel].min()) / signal.sample_rate) / 2) + 1 <= 320


class HighPass(BaseTransform):
    """``signal.high_pass(cutoff, zeros)`` (ref :1134-1170)."""

    def __init__(self, cutoff: tuple = ("choice", [50, 100, 250, 500, 1000]), zeros: int = 51, name: str = None,
                 prob: float = 1):
        super().__init__(name=name, prob=prob)
        self.cutoff = cutoff
        self.zeros = zeros

    def _instantiate(self, state: RandomState):
        return {"cutoff": util.sample_from_dist(self.cutoff, state)}

    def _transform(self, signal, cutoff, _bypass=None):
        return signal.high_pass(cutoff, zeros=self.zeros, _bypass=_bypass)

    def _bypass_ok(self, signal, tfm_kwargs) -> bool:
        # flags pay when the time-domain kernel serves the call (a flagged row is a plain copy); a bank long enough for
        # the FFT engine (> 320 taps) would spend its forward FFTs on the unselected rows as well: gather instead
        cut = util.host_view(tfm_kwargs["cutoff"]).reshape(-1).float()
        sel = util.host_view(tfm_kwargs["mask"]).reshape(-1).bool()
        if not bool(sel.any()) or float(cut[sel].min()) <= 0:
            return False
        return 2 * int(self.zeros / (float(cut[sel].min()) / signal.sample_rate) / 2) + 1 <= 320


class _PoolTransform(BaseTransform):
    """Shared by the transforms that draw another signal: ``sources`` is an in-memory pool -- a list of ``AudioSignal``
    (any lengths, resampled to the target rate on the device if needed) or a callable ``(state, signal) ->
    AudioSignal`` -- instead of the reference's csv lists of audio files (file decoding is outside the hot path)."""

    def _init_pool(self, sources, weights):
        self.sources = sources
        self.weights = weights

    def _draw_excerpt(self, state: RandomState, signal: AudioSignal):
        """One pool item, cut / zero-padded to the duration of ``signal`` at a random offset, with its channels."""
        if callable(self.sources):
            return self.sources(state, signal)
        if not self.sources:
            raise ValueError(f"{type(self).__name__} needs `sources`: a list of AudioSignal or a callable")
        src = self.sources[state.choice(len(self.sources), p=self.weights)].clone()
        if src.sample_rate != signal.sample_rate:
            raise ValueError(f"pool item at {src.sample_rate} Hz, signal at {signal.sample_rate} Hz: resample the pool")
        n = signal.signal_length
        if src.signal_length > n:
            off = int(state.randint(0, src.signal_length - n + 1))
            src.audio_data = src.audio_data[..., off:off + n]
        else:
            src.zero_pad_to(n)
        if src.num_channels != signal.num_channels:  # mono pool item -> every channel (ref loader: num_channels=...)
            src.audio_data = src.audio_data[:, :1].expand(-1, signal.num_channels, -1).contiguous()
        return src


class NoiseFloor(BaseTransform):
    """Adds Gaussian noise at ``db`` LUFS (ref :669-704).  The reference normalises the noise on the CPU while
    instantiating; here the (seeded, host-drawn) noise is normalised by the LUFS kernel when the transform runs."""

    def __init__(self, db: tuple = ("const", -50.0), name: str = None, prob: float = 1.0):
        super().__init__(name=name, prob=prob)
        self.db = db

    def _instantiate(self, state: RandomState, signal: AudioSignal):
        db = util.sample_from_dist(self.db, state)
        audio_data = state.randn(signal.num_channels, signal.signal_length)
        return {"nz_signal": AudioSignal(torch.from_numpy(audio_data).float()[None], signal.sample_rate), "db": db}

    def _transform(self, signal, nz_signal, db):
        return signal + nz_signal.clone().normalize(db)


class BackgroundNoise(_PoolTransform):
    """``signal.mix(bg_signal, snr, eq)`` (ref :707-792) with an in-memory pool of noise signals."""

    def __init__(self, snr: tuple = ("uniform", 10.0, 30.0), sources: List[AudioSignal] = None,
                 weights: List[float] = None, eq_amount: tuple = ("const", 1.0), n_bands: int = 3, name: str = None,
                 prob: float = 1.0):
        super().__init__(name=name, prob=prob)
        self.snr = snr
        self.eq_amount = eq_amount
        self.n_bands = n_bands
        self._init_pool(sources, weights)

    def _instantiate(self, state: RandomState, signal: AudioSignal):
        eq_amount = util.sample_from_dist(self.eq_amount, state)
        eq = -eq_amount * state.rand(self.n_bands)
        snr = util.sample_from_dist(self.snr, state)
        return {"eq": eq, "bg_signal": self._draw_excerpt(state, signal), "snr": snr}

    def _transform(self, signal, bg_signal, snr, eq):
        return signal.mix(bg_signal.clone(), snr, eq)


class CrossTalk(_PoolTransform):
    """Mixes another talker in at ``snr`` and restores the original loudness (ref :795-854)."""

    def __init__(self, snr: tuple = ("uniform", 0.0, 10.0), sources: List[AudioSignal] = None,
                 weights: List[float] = None, name: str = None, prob: float = 1.0):
        super().__init__(name=name, prob=prob)
        self.snr = snr
        self._init_pool(sources, weights)

    def _instantiate(self, state: RandomState, signal: AudioSignal):
        snr = util.sample_from_dist(self.snr, state)
        return {"crosstalk_signal": self._draw_excerpt(state, signal), "snr": snr}

    def _transform(self, signal, crosstalk_signal, snr):
        loudness = signal.loudness()
        mix = signal.mix(crosstalk_signal.clone(), snr)
        mix.normalize(loudness)
        return mix


class RoomImpulseResponse(BaseTransform):
    """``signal.apply_ir(ir, drr, eq)`` (ref :857-938).  ``sources`` is an in-memory pool: a list of
    single-item ``AudioSignal`` impulse responses (or a callable ``(state, signal) -> AudioSignal``);
    one is drawn per item with ``state.choice`` and zero-padded to one second like the reference."""
    _bypass_pays = False  # FFT convolution

    def __init__(self, drr: tuple = ("uniform", 0.0, 30.0), sources: List[AudioSignal] = None,
                 weights: List[float] = None, eq_amount: tuple = ("const", 1.0), n_bands: int = 6,
                 name: str = None, prob: float = 1.0, use_original_phase: bool = False):
        super().__init__(name=name, prob=prob)
        self.drr = drr
        self.eq_amount = eq_amount
        self.n_bands = n_bands
        self.use_original_phase = use_original_phase
        self.sources = sources
        self.weights = weights

    def _draw_ir(self, state, signal):
        if callable(self.sources):
            return self.sources(state, signal)
        if not self.sources:
            raise ValueError("RoomImpulseResponse needs `sources`: a list of AudioSignal impulse responses")
        idx = state.choice(len(self.sources), p=self.weights)
        return self.sources[idx].clone()

    def _instantiate(self, state: RandomState, signal: AudioSignal = None):
        eq_amount = util.sample_from_dist(self.eq_amount, state)
        eq = -eq_amount * state.rand(self.n_bands)
        drr = util.sample_from_dist(self.drr, state)
        ir_signal = self._draw_ir(state, signal)
        ir_signal.zero_pad_to(signal.sample_rate)
        return {"eq": eq, "ir_signal": ir_signal, "drr": drr}

    def _transform(self, signal, ir_signal, drr, eq, _bypass=None):
        return signal.apply_ir(ir_signal.clone(), drr, eq, use_original_phase=self.use_original_phase, _bypass=_bypass)


class SyntheticRoomImpulseResponse(BaseTransform):
    """``signal.apply_ir(ir)`` with one simulated shoebox room per item (an extension; ``core.room.image_source_ir``):
    no impulse-response collection is needed.  The signal's C channels are C microphones on a horizontal line.

    Per item, in this order: the room's x, y and z (``room``, three distribution tuples, metres); ``rt60`` (seconds),
    raised to 1.01 times the room's smallest feasible RT60 (``core.room.min_rt60``); the source, one
    ``state.uniform`` call for x, y, z inside the room shrunk by ``margin`` on every side; the microphone spacing
    (``mic_spacing``, metres); the array's azimuth, ``uniform(0, 2 pi)``; the array's centre, one ``state.uniform``
    call inside the room shrunk by ``margin`` plus half the array's extent along x and y.  A room too small for the
    margin or the array raises ``ValueError``.  The IR is ``duration`` seconds long when given, else the batch's
    longest RT60, and never longer than the signal.  All walls absorb alike (Sabine); ``max_order`` and ``high_pass``
    are passed to ``image_source_ir``.

    ``diffuse_after`` (seconds: a float or a distribution tuple) makes hybrid responses, images before it and a diffuse
    tail after it (``image_source_ir(..., diffuse_after=, seed=)``), much cheaper for long RT60s.  Only then two more
    draws follow the ones above: the time (when it is a tuple), then the tail's seed, ``state.randint(0, 2**31 - 1)``.
    It needs ``max_order = -1``.

    ``bands=K`` makes the rooms frequency-dependent over K octave bands (``image_source_ir(..., bands=)``):
    ``band_rt60`` is K distribution tuples, each band's RT60 as a ratio to the item's ``rt60`` (None: 1 for every band),
    each raised like ``rt60`` to 1.01 times the room's smallest feasible RT60; ``air_absorption`` is K constants in
    dB/m (None: no air absorption).  Only then K more draws follow all the ones above, one per band in order, and the
    IR is as long as the longest band RT60 when no ``duration`` is given.

    ``source_speed`` (a distribution tuple, m/s) makes the source move (``AudioSignal.apply_moving_ir``, DESIGN.md
    K22): the drawn source is the start of a straight path that it follows at the drawn speed toward an end point, and
    where it stops.  Only then two more draws follow all the ones above: the end point (``end``), one
    ``state.uniform`` call inside the same margin box as the source, so the whole path stays in the box; then the speed
    (``speed``), which must be >= 0 (a negative draw raises ``ValueError``).  One response is computed every
    ``max(1024, round(waypoint_hop * sample_rate))`` samples at the source's position at that time (1024 is the
    convolution's smallest hop, so below 20.48 kHz the default 0.05 s becomes 1024 samples), and the signal is
    convolved with the path, crossfading between neighbouring waypoints.  With ``diffuse_after`` all waypoints of an item share its seed, so their tails are the same noise under
    slightly different envelopes and a crossfade loses no tail power.  A smaller ``waypoint_hop`` reduces the comb
    filtering a crossfade makes when the delay changes by more than a sample between waypoints.

    ``mic_pattern`` and ``source_pattern`` (a name of ``core.room.PATTERNS`` or p in [0, 1]) make the microphones and
    the sources directional (``image_source_ir(..., mic_pattern=, source_pattern=)``, DESIGN.md K20 "Directivity").
    Only then more draws follow all the ones above: with ``mic_pattern`` the azimuth of the microphones
    (``mic_azimuth``, radians, default ``uniform(0, 2 pi)``), all of them pointing horizontally that way
    (``mic_orientation``); then with ``source_pattern`` the source's yaw (``source_yaw``, radians, default
    ``uniform(-pi/2, pi/2)``), the source pointing horizontally toward the array's centre turned by the yaw
    (``source_orientation``).  A moving source keeps its orientation along its path."""
    _bypass_pays = False  # FFT convolution

    DEFAULT_ROOM = (("uniform", 3.0, 10.0), ("uniform", 3.0, 8.0), ("uniform", 2.4, 4.0))

    def __init__(self, room: tuple = DEFAULT_ROOM, rt60: tuple = ("uniform", 0.2, 0.8), margin: float = 0.5,
                 mic_spacing: tuple = ("uniform", 0.05, 0.2), max_order: int = -1, duration: float = None,
                 high_pass: bool = True, name: str = None, prob: float = 1.0, use_original_phase: bool = False,
                 diffuse_after=None, bands: int = None, band_rt60=None, air_absorption=None, source_speed=None,
                 waypoint_hop: float = 0.05, mic_pattern=None, source_pattern=None,
                 mic_azimuth: tuple = ("uniform", 0.0, 2.0 * np.pi),
                 source_yaw: tuple = ("uniform", -0.5 * np.pi, 0.5 * np.pi)):
        super().__init__(name=name, prob=prob)
        from ..core.room import PATTERNS

        for end, pat in (("mic", mic_pattern), ("source", source_pattern)):
            if pat is None:  # omnidirectional: no draw is made, so no key is expected
                self.keys = [k for k in self.keys if k != f"{end}_orientation"]
            elif isinstance(pat, str) and pat not in PATTERNS:
                raise ValueError(f"SyntheticRoomImpulseResponse: {end}_pattern = {pat!r}; one of "
                                 f"{', '.join(PATTERNS)} or a value in [0, 1]")
            elif not isinstance(pat, str) and not (np.ndim(pat) == 0 and 0.0 <= float(pat) <= 1.0):
                raise ValueError(f"SyntheticRoomImpulseResponse: {end}_pattern = {pat!r}; a name or one value in "
                                 "[0, 1], shared by every item")
        self.mic_pattern, self.source_pattern = mic_pattern, source_pattern
        self.mic_azimuth, self.source_yaw = mic_azimuth, source_yaw
        if source_speed is None:  # a static source: neither draw is made, so neither key is expected
            self.keys = [k for k in self.keys if k not in ("end", "speed")]
        if diffuse_after is None:  # no tail: neither draw is made, so neither key is expected
            self.keys = [k for k in self.keys if k not in ("diffuse_after", "seed")]
        if bands is None:
            if band_rt60 is not None or air_absorption is not None:
                raise ValueError("SyntheticRoomImpulseResponse: band_rt60 and air_absorption need bands")
            self.keys = [k for k in self.keys if k != "band_rt60"]
        else:
            from ..core.room import MAX_BANDS

            if isinstance(bands, bool) or not isinstance(bands, (int, np.integer)) or not 1 <= bands <= MAX_BANDS:
                raise ValueError(f"SyntheticRoomImpulseResponse: bands = {bands!r}; an int in 1 .. {MAX_BANDS}")
            band_rt60 = tuple(band_rt60) if band_rt60 is not None else (("const", 1.0),) * bands
            if len(band_rt60) != bands:
                raise ValueError(f"SyntheticRoomImpulseResponse: band_rt60 has {len(band_rt60)} entries for {bands} "
                                 "bands")
            if air_absorption is not None:
                air_absorption = np.asarray(air_absorption, dtype=np.float64)
                if air_absorption.shape != (bands,):
                    raise ValueError(f"SyntheticRoomImpulseResponse: air_absorption must be {bands} values (dB/m), "
                                     f"got shape {air_absorption.shape}")
        self.bands = None if bands is None else int(bands)
        self.band_rt60 = band_rt60
        self.air_absorption = air_absorption
        self.room = tuple(room)
        self.diffuse_after = diffuse_after
        self.rt60 = rt60
        self.margin = float(margin)
        self.mic_spacing = mic_spacing
        self.max_order = int(max_order)
        self.duration = duration
        self.high_pass = high_pass
        self.use_original_phase = use_original_phase
        self.source_speed = source_speed
        self.waypoint_hop = float(waypoint_hop)
        if not (np.isfinite(self.waypoint_hop) and self.waypoint_hop > 0):
            raise ValueError(f"SyntheticRoomImpulseResponse: waypoint_hop = {waypoint_hop!r}; seconds > 0")

    def _instantiate(self, state: RandomState, signal: AudioSignal):
        from ..core import room as _room

        dims = np.array([float(util.sample_from_dist(d, state)) for d in self.room])
        rt60 = float(util.sample_from_dist(self.rt60, state))
        lo, hi = np.full(3, self.margin), dims - self.margin
        if np.any(lo >= hi):
            raise ValueError(f"SyntheticRoomImpulseResponse: room {dims} m is too small for a {self.margin} m margin")
        source = state.uniform(lo, hi)
        spacing = float(util.sample_from_dist(self.mic_spacing, state))
        azimuth = state.uniform(0.0, 2.0 * np.pi)
        C = signal.num_channels
        axis = np.array([np.cos(azimuth), np.sin(azimuth), 0.0])
        ext = 0.5 * (C - 1) * spacing * np.abs(axis)
        if np.any(lo + ext > hi - ext):
            raise ValueError(f"SyntheticRoomImpulseResponse: room {dims} m is too small for {C} microphones "
                             f"{spacing} m apart and a {self.margin} m margin")
        centre = state.uniform(lo + ext, hi - ext)
        mics = centre + (np.arange(C) - 0.5 * (C - 1))[:, None] * spacing * axis
        rt60 = max(rt60, 1.01 * float(_room.min_rt60(dims)))
        out = {"room": dims, "rt60": np.float64(rt60), "source": source, "mics": mics}
        if self.diffuse_after is not None:
            td = self.diffuse_after
            out["diffuse_after"] = np.float64(util.sample_from_dist(td, state) if isinstance(td, tuple) else td)
            out["seed"] = np.int64(state.randint(0, 2 ** 31 - 1))
        if self.bands is not None:
            floor = 1.01 * float(_room.min_rt60(dims))
            out["band_rt60"] = np.array([max(float(util.sample_from_dist(r, state)) * rt60, floor)
                                         for r in self.band_rt60])
        if self.source_speed is not None:
            out["end"] = state.uniform(lo, hi)
            speed = float(util.sample_from_dist(self.source_speed, state))
            if not (np.isfinite(speed) and speed >= 0):
                raise ValueError(f"SyntheticRoomImpulseResponse: source_speed drew {speed} m/s; speeds must be "
                                 "finite and >= 0")
            out["speed"] = np.float64(speed)
        if self.mic_pattern is not None:
            az = float(util.sample_from_dist(self.mic_azimuth, state))
            out["mic_orientation"] = np.array([np.cos(az), np.sin(az), 0.0])
        if self.source_pattern is not None:
            yaw = float(util.sample_from_dist(self.source_yaw, state))
            to = mics.mean(axis=0) - source
            ang = np.arctan2(to[1], to[0]) + yaw
            out["source_orientation"] = np.array([np.cos(ang), np.sin(ang), 0.0])
        return out

    def _transform(self, signal, room, rt60, source, mics, diffuse_after=None, seed=None, band_rt60=None, end=None,
                   speed=None, mic_orientation=None, source_orientation=None, _bypass=None):
        from ..core.room import image_source_ir

        sr, T = signal.sample_rate, signal.signal_length
        walls = rt60 if band_rt60 is None else band_rt60
        seconds = self.duration if self.duration is not None else float(util.host_view(walls).max())
        length = max(1, min(T, int(np.ceil(seconds * sr))))
        bands = {} if self.bands is None else dict(bands=self.bands, air_absorption=self.air_absorption)
        B, C = signal.batch_size, signal.num_channels
        if mic_orientation is not None:  # one azimuth per item, shared by its microphones: [B, C, 3]
            mic_orientation = np.broadcast_to(_host_values(mic_orientation).reshape(-1, 1, 3), (B, C, 3))
        if source_orientation is not None:
            source_orientation = _host_values(source_orientation).reshape(-1, 3)
        if end is None:
            ir = image_source_ir(room, source, mics, sr, length, rt60=walls, max_order=self.max_order,
                                 high_pass=self.high_pass, diffuse_after=diffuse_after, seed=seed,
                                 device=signal.device, mic_pattern=self.mic_pattern, mic_orientation=mic_orientation,
                                 source_pattern=self.source_pattern, source_orientation=source_orientation, **bands)
            return signal.apply_ir(ir, use_original_phase=self.use_original_phase, _bypass=_bypass)
        from ..engine import Engine

        hop = max(Engine.MOVING_IR_MIN_HOP, int(round(self.waypoint_hop * sr)))
        K = (T - 1) // hop + 1
        path = self.path(source, end, speed, K, hop / sr)  # [B, K, 3]

        def per_waypoint(v, nd: int, dtype=np.float64):  # each item's value [..nd dims], repeated for its waypoints
            if v is None:
                return None
            v = _host_values(v, dtype)
            return np.repeat(np.broadcast_to(v, (B,) + v.shape[v.ndim - nd:]), K, axis=0)

        from ..core.room import MAX_ROWS

        room_k, mics_k = per_waypoint(room, 1), per_waypoint(mics, 2)
        walls_k = per_waypoint(walls, 0 if band_rt60 is None else 1)
        td_k, seed_k = per_waypoint(diffuse_after, 0), per_waypoint(seed, 0, np.int64)
        mo_k, so_k = per_waypoint(mic_orientation, 2), per_waypoint(source_orientation, 1)
        step = max(1, MAX_ROWS // (C * (self.bands or 1)))  # items per call: items x microphones x bands <= MAX_ROWS
        irs = []
        for i in range(0, B * K, step):
            s = slice(i, i + step)
            irs.append(image_source_ir(room_k[s], path.reshape(-1, 3)[s], mics_k[s], sr, length, rt60=walls_k[s],
                                       max_order=self.max_order, high_pass=self.high_pass,
                                       diffuse_after=None if td_k is None else td_k[s],
                                       seed=None if seed_k is None else seed_k[s], device=signal.device,
                                       mic_pattern=self.mic_pattern,
                                       mic_orientation=None if mo_k is None else mo_k[s],
                                       source_pattern=self.source_pattern,
                                       source_orientation=None if so_k is None else so_k[s], **bands).audio_data)
        irs = torch.cat(irs).reshape(B, K, C, length)
        return signal.apply_moving_ir(irs, hop, use_original_phase=self.use_original_phase, _bypass=_bypass)

    @staticmethod
    def path(source, end, speed, K: int, dt: float) -> np.ndarray:
        """[B, K, 3] positions of sources moving from ``source`` [B, 3] toward ``end`` [B, 3] at ``speed`` [B] m/s,
        stopping there, sampled every ``dt`` seconds from 0."""
        source, end = _host_values(source).reshape(-1, 3), _host_values(end).reshape(-1, 3)
        speed = _host_values(speed).reshape(-1, 1)
        span = end - source
        dist = np.linalg.norm(span, axis=-1, keepdims=True)
        frac = speed * dt * np.arange(K)[None, :] / np.maximum(dist, 1e-300)  # [B, K]
        return np.where(frac[..., None] >= 1.0, end[:, None], source[:, None] + frac[..., None] * span[:, None])


class PitchShift(BaseTransform):
    """``signal.pitch_shift(n_semitones)``.  NEW: the reference has no PitchShift transform (only the
    ``AudioSignal.pitch_shift`` method, ref:audiotools/core/effects.py:247-277, which takes ONE shift
    for the whole batch); BASELINE.json config 4 needs it.  Items are grouped by their drawn shift inside the
    engine (one set of launches for the whole batch)."""

    def __init__(self, n_semitones: tuple = ("choice", [-2, -1, 0, 1, 2]), quick: bool = True, name: str = None,
                 prob: float = 1.0):
        super().__init__(name=name, prob=prob)
        self.n_semitones = n_semitones
        self.quick = quick

    def _instantiate(self, state: RandomState):
        return {"n_semitones": util.sample_from_dist(self.n_semitones, state)}

    def _transform(self, signal, n_semitones, _bypass=None):
        # the grouping by shift is a host decision (host mirror: no sync); all groups share the kernel launches
        shifts = util.ensure_tensor(util.host_view(n_semitones), 1, signal.batch_size).reshape(-1)
        if _bypass is not None:  # shift 0 = the kernels copy the row through
            shifts = torch.where(util.host_view(_bypass).cpu().bool().reshape(-1), torch.zeros_like(shifts), shifts)
        return signal.pitch_shift(shifts, quick=self.quick)


class ClippingDistortion(BaseTransform):
    def __init__(self, perc: tuple = ("uniform", 0.0, 0.1), name: str = None, prob: float = 1.0):
        super().__init__(name=name, prob=prob)
        self.perc = perc

    def _instantiate(self, state: RandomState):
        return {"perc": util.sample_from_dist(self.perc, state)}

    def _transform(self, signal, perc):
        return signal.clip_distortion(perc)


class Quantization(BaseTransform):
    def __init__(self, channels: tuple = ("choice", [8, 32, 128, 256, 1024]), name: str = None, prob: float = 1.0):
        super().__init__(name=name, prob=prob)
        self.channels = channels

    def _instantiate(self, state: RandomState):
        return {"channels": util.sample_from_dist(self.channels, state)}

    def _transform(self, signal, channels):
        return signal.quantization(channels)


class MuLawQuantization(BaseTransform):
    def __init__(self, channels: tuple = ("choice", [8, 32, 128, 256, 1024]), name: str = None, prob: float = 1.0):
        super().__init__(name=name, prob=prob)
        self.channels = channels

    def _instantiate(self, state: RandomState):
        return {"channels": util.sample_from_dist(self.channels, state)}

    def _transform(self, signal, channels):
        return signal.mulaw_quantization(channels)


class RescaleAudio(BaseTransform):
    def __init__(self, val: float = 1.0, name: str = None, prob: float = 1):
        super().__init__(name=name, prob=prob)
        self.val = val

    def _transform(self, signal):
        return signal.ensure_max_of_audio(self.val)


class ShiftPhase(SpectralTransform):
    """stft -> ``phase += shift`` -> istft (ref :1200-1229)."""

    def __init__(self, shift: tuple = ("uniform", -np.pi, np.pi), name: str = None, prob: float = 1):
        super().__init__(name=name, prob=prob)
        self.shift = shift

    def _instantiate(self, state: RandomState):
        return {"shift": util.sample_from_dist(self.shift, state)}

    def _transform(self, signal, shift):
        return signal.shift_phase(shift)


class InvertPhase(ShiftPhase):
    """Phase shift by pi (ref :1232-1247)."""

    def __init__(self, name: str = None, prob: float = 1):
        super().__init__(shift=("const", np.pi), name=name, prob=prob)


class CorruptPhase(SpectralTransform):
    """Adds host-drawn (seeded) Gaussian noise to the phase (ref :1250-1278)."""

    def __init__(self, scale: tuple = ("uniform", 0, np.pi), name: str = None, prob: float = 1):
        super().__init__(name=name, prob=prob)
        self.scale = scale

    def _instantiate(self, state: RandomState, signal: AudioSignal = None):
        scale = util.sample_from_dist(self.scale, state)
        # the shape of one item's phase, without touching the device: [C, F, N]
        wl, hop, _, match_stride, _ = signal._resolve_stft(None, None, None, None, None)
        right_pad, pad = signal.compute_stft_padding(wl, hop, match_stride)
        if signal.stft_data is not None:
            n_frames = signal.stft_data.shape[-1]
        else:
            from ..engine import get_engine

            n_frames = get_engine().num_frames(signal.signal_length, wl, hop, pad, right_pad, 2 if match_stride else 0)
        shape = (signal.num_channels, wl // 2 + 1, n_frames)
        corruption = state.normal(scale=scale, size=shape)
        return {"corruption": corruption.astype("float32")}

    def _transform(self, signal, corruption):
        return signal.shift_phase(shift=corruption)


class FrequencyMask(SpectralTransform):
    """Zeroes a frequency band around a drawn centre (SpecAugment; ref :1281-1324)."""

    def __init__(self, f_center: tuple = ("uniform", 0.0, 1.0), f_width: tuple = ("const", 0.1), name: str = None,
                 prob: float = 1):
        super().__init__(name=name, prob=prob)
        self.f_center = f_center
        self.f_width = f_width

    def _instantiate(self, state: RandomState, signal: AudioSignal):
        f_center = util.sample_from_dist(self.f_center, state)
        f_width = util.sample_from_dist(self.f_width, state)
        fmin = max(f_center - (f_width / 2), 0.0)
        fmax = min(f_center + (f_width / 2), 1.0)
        return {"fmin_hz": (signal.sample_rate / 2) * fmin, "fmax_hz": (signal.sample_rate / 2) * fmax}

    def _transform(self, signal, fmin_hz: float, fmax_hz: float):
        return signal.mask_frequencies(fmin_hz=fmin_hz, fmax_hz=fmax_hz)


class TimeMask(SpectralTransform):
    """Zeroes a span of frames around a drawn centre (SpecAugment; ref :1327-1369)."""

    def __init__(self, t_center: tuple = ("uniform", 0.0, 1.0), t_width: tuple = ("const", 0.025), name: str = None,
                 prob: float = 1):
        super().__init__(name=name, prob=prob)
        self.t_center = t_center
        self.t_width = t_width

    def _instantiate(self, state: RandomState, signal: AudioSignal):
        t_center = util.sample_from_dist(self.t_center, state)
        t_width = util.sample_from_dist(self.t_width, state)
        tmin = max(t_center - (t_width / 2), 0.0)
        tmax = min(t_center + (t_width / 2), 1.0)
        return {"tmin_s": signal.signal_duration * tmin, "tmax_s": signal.signal_duration * tmax}

    def _transform(self, signal, tmin_s: float, tmax_s: float):
        return signal.mask_timesteps(tmin_s=tmin_s, tmax_s=tmax_s)


class MaskLowMagnitudes(SpectralTransform):
    """Zeroes STFT cells below a drawn dB threshold (ref :1372-1402)."""

    def __init__(self, db_cutoff: tuple = ("uniform", -10, 10), name: str = None, prob: float = 1):
        super().__init__(name=name, prob=prob)
        self.db_cutoff = db_cutoff

    def _instantiate(self, state: RandomState, signal: AudioSignal = None):
        return {"db_cutoff": util.sample_from_dist(self.db_cutoff, state)}

    def _transform(self, signal, db_cutoff: float):
        return signal.mask_low_magnitudes(db_cutoff)


class Smoothing(BaseTransform):
    """Convolves the signal with a drawn window and restores its peak (ref :1405-1453)."""

    def __init__(self, window_type: tuple = ("const", "average"),
                 window_length: tuple = ("choice", [8, 16, 32, 64, 128, 256, 512]), name: str = None, prob: float = 1):
        super().__init__(name=name, prob=prob)
        self.window_type = window_type
        self.window_length = window_length

    def _instantiate(self, state: RandomState, signal: AudioSignal = None):
        window_type = util.sample_from_dist(self.window_type, state)
        window_length = util.sample_from_dist(self.window_length, state)
        window = signal.get_window(window_type=window_type, window_length=window_length, device="cpu")
        return {"window": AudioSignal(window.clone(), signal.sample_rate)}

    def _transform(self, signal, window):
        sscale = signal.audio_data.abs().max(dim=-1, keepdim=True).values
        sscale = torch.where(sscale == 0.0, torch.ones_like(sscale), sscale)
        out = signal.convolve(window)
        oscale = out.audio_data.abs().max(dim=-1, keepdim=True).values
        oscale = torch.where(oscale == 0.0, torch.ones_like(oscale), oscale)
        return out * (sscale / oscale)


def _refill_masked_cells(signal):
    """Replace the cells a band mask zeroed (|X| == 0 and angle == 0) by N(0,1) magnitude / phase noise drawn on
    the device (ref :1485-1495 / :1526-1536)."""
    mag, phase = signal.magnitude, signal.phase
    mag_r, phase_r = torch.randn_like(mag), torch.randn_like(phase)
    mask = (mag == 0.0) & (phase == 0.0)
    # the reference assigns `signal.magnitude = mag` and then `signal.phase = phase`; the second setter re-reads
    # |stft_data|, so a refilled cell ends up as |mag_r| exp(1j phase_r)
    signal.stft_data = torch.where(mask, mag_r.abs(), mag) * torch.exp(1j * torch.where(mask, phase_r, phase))
    return signal


class TimeNoise(TimeMask):
    """TimeMask, then the masked frames are filled with noise (ref :1456-1495)."""

    def _transform(self, signal, tmin_s: float, tmax_s: float):
        return _refill_masked_cells(signal.mask_timesteps(tmin_s=tmin_s, tmax_s=tmax_s, val=0.0))


class FrequencyNoise(FrequencyMask):
    """FrequencyMask, then the masked band is filled with noise (ref :1498-1536)."""

    def _transform(self, signal, fmin_hz: float, fmax_hz: float):
        return _refill_masked_cells(signal.mask_frequencies(fmin_hz=fmin_hz, fmax_hz=fmax_hz))


class Silence(BaseTransform):
    """Replace the item by silence while KEEPING its cached loudness (ref :1053-1092)."""

    def __init__(self, name: str = None, prob: float = 0.1):
        super().__init__(name=name, prob=prob)

    def _transform(self, signal):
        _loudness = signal._loudness
        signal = AudioSignal(torch.zeros_like(signal.audio_data), sample_rate=signal.sample_rate,
                             stft_params=signal.stft_params)
        signal._loudness = _loudness  # so that the target still can be normalised relative to it
        return signal


class SpectralDenoising(Equalizer):
    """Spectral gating against a host-drawn (seeded) white-noise excerpt, normalised and equalised on the device
    (ref :1539-1592; ``ml.layers.SpectralGate``)."""

    def __init__(self, eq_amount: tuple = ("const", 1.0), denoise_amount: tuple = ("uniform", 0.8, 1.0),
                 nz_volume: float = -40, n_bands: int = 6, n_freq: int = 3, n_time: int = 5, name: str = None,
                 prob: float = 1):
        super().__init__(eq_amount=eq_amount, n_bands=n_bands, name=name, prob=prob)
        from ..ml.layers import SpectralGate

        self.nz_volume = nz_volume
        self.denoise_amount = denoise_amount
        self.spectral_gate = SpectralGate(n_freq, n_time)

    def _transform(self, signal, nz, eq, denoise_amount):
        nz = nz.normalize(self.nz_volume).equalizer(eq)
        self.spectral_gate = self.spectral_gate.to(signal.device)
        return self.spectral_gate(signal, nz, denoise_amount)

    def _instantiate(self, state: RandomState):
        kwargs = super()._instantiate(state)
        kwargs["denoise_amount"] = util.sample_from_dist(self.denoise_amount, state)
        kwargs["nz"] = AudioSignal(torch.from_numpy(state.randn(22050)).float(), 44100)
        return kwargs
