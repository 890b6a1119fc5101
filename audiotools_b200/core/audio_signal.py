"""``AudioSignal``: the batched waveform container of the hot path, with the reference's
method surface (ref:audiotools/core/audio_signal.py) on top of the sm_90a engine.

State: ``audio_data`` [B, C, T] float32, ``stft_data`` [B, C, F, N] complex64 (cache of the
last ``stft()``), ``_loudness`` [B] (cache, cleared by the ``audio_data`` setter, kept by
``__setitem__``), ``sample_rate``, ``stft_params``, ``metadata``.  Methods mutate ``self`` and
return ``self`` except ``stft / mel_spectrogram / mfcc / loudness`` which return tensors.

All DSP runs in ``libb2a`` (``audiotools_b200.engine``) on CUDA tensors; a CPU-resident signal
is only a container (construction, batching, indexing, arithmetic) -- calling a DSP method on it
raises, there is no CPU implementation.  File IO (``load_from_file``, ``write``, ``excerpt``,
``salient_excerpt``, ``hash``) is out of scope (SURVEY.md §2 row 1).
"""
import copy
import functools
import math
import warnings
from collections import namedtuple

import numpy as np
import torch

from . import grad as _grad
from . import mel as _mel
from . import util
from .dsp import DSPMixin
from .effects import EffectMixin, ImpulseResponseMixin
from .loudness import LoudnessMixin

STFTParams = namedtuple(
    "STFTParams", ["window_length", "hop_length", "window_type", "match_stride", "padding_type"])
STFTParams.__new__.__defaults__ = (None, None, None, None, None)


def _engine():
    from ..engine import get_engine

    return get_engine()


def _on_engine(t) -> bool:
    """CUDA tensor, or any tensor when the engine is the CPU-simulated build of the kernels (tests)."""
    return t.is_cuda or not _engine().require_cuda


@functools.lru_cache(None)
def _cached_window(window_type: str, window_length: int, device: str) -> torch.Tensor:
    from scipy import signal

    if window_type == "average":
        w = np.ones(window_length) / window_length
    elif window_type == "sqrt_hann":
        w = np.sqrt(signal.get_window("hann", window_length))
    else:
        w = signal.get_window(window_type, window_length)
    return torch.from_numpy(w).to(device).float()


class AudioSignal(EffectMixin, LoudnessMixin, ImpulseResponseMixin, DSPMixin):
    def __init__(self, audio_path_or_array, sample_rate: int = None, stft_params: STFTParams = None,
                 offset: float = 0, duration: float = None, device: str = None):
        if isinstance(audio_path_or_array, (str, bytes)) or hasattr(audio_path_or_array, "__fspath__"):
            raise NotImplementedError(
                "audiotools_b200.AudioSignal is built from arrays/tensors; decoding audio files is "
                "outside the accelerated hot path (decode with your loader, then pass the samples)")
        if not (isinstance(audio_path_or_array, np.ndarray) or torch.is_tensor(audio_path_or_array)):
            raise ValueError("audio_path_or_array must be either a Path, string, numpy array, or torch Tensor!")
        self.path_to_file = None
        self._audio_data = None
        self._pending_gain = None
        self._measured_loudness = None  # set by normalize(): the LUFS its gain was derived from
        self._stft_data = None
        self._loudness = None
        self.sources = None
        assert sample_rate is not None, "Must set sample rate!"
        self.load_from_array(audio_path_or_array, sample_rate, device=device)
        self.window = None
        self.stft_params = stft_params
        self.metadata = {"offset": offset, "duration": duration}

    # ------------------------------------------------------------------ construction
    def load_from_array(self, audio_array, sample_rate: int, device: str = None):
        data = util.ensure_tensor(audio_array)
        if data.dtype == torch.double:
            data = data.float()
        while data.ndim < 3:
            data = data.unsqueeze(0)
        self.audio_data = data
        self.original_signal_length = self.signal_length
        self.sample_rate = sample_rate
        return self.to(device) if device is not None else self

    @classmethod
    def zeros(cls, duration: float, sample_rate: int, num_channels: int = 1, batch_size: int = 1, **kwargs):
        n = int(duration * sample_rate)
        return cls(torch.zeros(batch_size, num_channels, n), sample_rate, **kwargs)

    @classmethod
    def wave(cls, frequency: float, duration: float, sample_rate: int, num_channels: int = 1,
             shape: str = "sine", **kwargs):
        from scipy import signal as sps

        t = torch.linspace(0, duration, int(duration * sample_rate))
        arg = 2 * np.pi * frequency * t
        if shape == "sawtooth":
            w = torch.from_numpy(sps.sawtooth(arg.numpy(), 0.5))
        elif shape == "square":
            w = torch.from_numpy(sps.square(arg.numpy()))
        elif shape == "sine":
            w = torch.sin(arg)
        elif shape == "triangle":
            w = torch.from_numpy(sps.sawtooth(arg.numpy(), 0.5))
        else:
            raise ValueError(f"Invalid shape {shape}")
        return cls(w.float().unsqueeze(0).unsqueeze(0).repeat(1, num_channels, 1), sample_rate, **kwargs)

    @classmethod
    def excerpt(cls, source, offset: float = None, duration: float = None, state=None, **kwargs):
        """Randomly draw an excerpt of ``duration`` seconds between ``offset`` seconds and the end of ``source``
        (ref:audiotools/core/audio_signal.py:178-225).  ``source`` is an in-memory ``AudioSignal`` (batch size 1):
        decoding files is outside the hot path (SURVEY.md 2), so the reference's ``audio_path`` is not accepted.
        The window starts at sample ``int(offset * sample_rate)`` and has ``int(duration * sample_rate)`` samples
        (zero-padded past the end, like a short read)."""
        if not isinstance(source, AudioSignal):
            raise NotImplementedError("excerpt / salient_excerpt take an in-memory AudioSignal (file decoding is out "
                                      "of scope: SURVEY.md 2)")
        assert source.batch_size == 1, "excerpt: the source must hold one item"
        state = util.random_state(state)
        lower = 0 if offset is None else offset
        upper = max(source.signal_duration - duration, 0)
        off = state.uniform(lower, upper)
        n = int(duration * source.sample_rate)
        start = int(off * source.sample_rate)
        x = source.audio_data
        if _on_engine(x):
            data = _engine().pack_rows([x], n, offsets=[start])
        else:
            data = torch.zeros(1, x.shape[1], n, dtype=x.dtype)
            seg = x[..., start:start + n]
            data[..., : seg.shape[-1]] = seg
        sig = cls(data, source.sample_rate, **kwargs)
        sig.metadata["offset"], sig.metadata["duration"] = off, duration
        return sig

    @classmethod
    def salient_excerpt(cls, source, loudness_cutoff: float = None, num_tries: int = 8, state=None, **kwargs):
        """``excerpt`` that only accepts windows louder than ``loudness_cutoff`` dB LUFS, giving up after
        ``num_tries`` draws (ref:audiotools/core/audio_signal.py:227-286).  On the device the candidates are screened
        as a BATCH (SURVEY.md 8f.4): all pending offsets are drawn from a copy of ``state``, gathered with one launch
        of csrc/collate.cu, measured with one call of the loudness kernels, and the first one above the cutoff wins;
        ``state`` is then advanced by exactly the number of draws the reference's loop would have made."""
        state = util.random_state(state)
        if loudness_cutoff is None:
            return cls.excerpt(source, state=state, **kwargs)
        if not isinstance(source, AudioSignal):
            raise NotImplementedError("excerpt / salient_excerpt take an in-memory AudioSignal (file decoding is out "
                                      "of scope: SURVEY.md 2)")
        assert source.batch_size == 1, "salient_excerpt: the source must hold one item"
        offset, duration = kwargs.pop("offset", None), kwargs.pop("duration", None)
        lower = 0 if offset is None else offset
        upper = max(source.signal_duration - duration, 0)
        n = int(duration * source.sample_rate)
        x = source.audio_data
        tried = 0
        while True:
            chunk = 8 if num_tries is None else min(8, num_tries - tried)
            probe = np.random.RandomState()
            probe.set_state(state.get_state())
            offs = [probe.uniform(lower, upper) for _ in range(chunk)]
            starts = [int(o * source.sample_rate) for o in offs]
            if _on_engine(x):
                cand = _engine().pack_rows([x] * chunk, n, offsets=starts)
            else:
                cand = torch.zeros(chunk, x.shape[1], n, dtype=x.dtype)
                for i, st in enumerate(starts):
                    seg = x[0, :, st:st + n]
                    cand[i, :, : seg.shape[-1]] = seg
            loud = cls(cand, source.sample_rate).loudness().cpu().numpy()
            above = np.nonzero(loud > loudness_cutoff)[0]
            last = tried + chunk >= num_tries if num_tries is not None else False
            if len(above) or last:
                k = int(above[0]) if len(above) else chunk - 1
                for _ in range(k + 1):  # the draws the reference's sequential loop makes
                    state.uniform(lower, upper)
                sig = cls(cand[k:k + 1].clone(), source.sample_rate, **kwargs)
                sig.metadata["offset"], sig.metadata["duration"] = offs[k], duration
                return sig
            for _ in range(chunk):
                state.uniform(lower, upper)
            tried += chunk

    @classmethod
    def batch(cls, audio_signals: list, pad_signals: bool = False, truncate_signals: bool = False,
              resample: bool = False, dim: int = 0):
        lengths = [s.signal_length for s in audio_signals]
        rates = [s.sample_rate for s in audio_signals]
        if len(set(rates)) != 1:
            if not resample:
                raise RuntimeError(
                    f"Not all signals had the same sample rate! Got {rates}. "
                    f"All signals must have the same sample rate, or resample must be True. ")
            for s in audio_signals:
                s.resample(rates[0])
        if len(set(lengths)) != 1:
            if not (pad_signals or truncate_signals):
                raise RuntimeError(
                    f"Not all signals had the same length! Got {lengths}. "
                    f"All signals must be the same length, or pad_signals/truncate_signals must be True. ")
            target = max(lengths) if pad_signals else min(lengths)
            datas = [s.audio_data for s in audio_signals]
            if (dim == 0 and all(_on_engine(d) and d.device == datas[0].device for d in datas)
                    and len({d.shape[1] for d in datas}) == 1):
                # device collate (SURVEY.md 8f.4): ONE gather launch writes the padded / truncated batch; the inputs
                # become views of it, which is the state the reference's in-place zero_pad / truncate_samples leaves
                packed = _engine().pack_rows(datas, target)
                i = 0
                for s in audio_signals:
                    b = s.batch_size
                    s.audio_data = packed[i:i + b]
                    i += b
                out = cls(packed, sample_rate=audio_signals[0].sample_rate)
                out.path_to_file = [s.path_to_file for s in audio_signals]
                return out
            for s in audio_signals:
                if pad_signals:
                    s.zero_pad(0, target - s.signal_length)
                else:
                    s.truncate_samples(target)
        out = cls(torch.cat([s.audio_data for s in audio_signals], dim=dim), sample_rate=audio_signals[0].sample_rate)
        out.path_to_file = [s.path_to_file for s in audio_signals]
        return out

    # ------------------------------------------------------------------ copies / devices
    def deepcopy(self):
        return copy.deepcopy(self)

    def copy(self):
        return copy.copy(self)

    def clone(self):
        c = type(self)(self.audio_data.clone(), self.sample_rate, stft_params=self.stft_params)
        if self.stft_data is not None:
            c.stft_data = self.stft_data.clone()
        if self._loudness is not None:
            c._loudness = self._loudness.clone()
        c.path_to_file = copy.deepcopy(self.path_to_file)
        c.metadata = copy.deepcopy(self.metadata)
        return c

    def detach(self):
        if self._loudness is not None:
            self._loudness = self._loudness.detach()
        if self.stft_data is not None:
            self.stft_data = self.stft_data.detach()
        self.audio_data = self.audio_data.detach()
        return self

    def to(self, device):
        if self.stft_data is not None:
            self.stft_data = self.stft_data.to(device)
        if self.audio_data is not None:
            # through the setter on purpose: like the reference (ref :739-759) a move drops the
            # loudness cache, so a parent batch never carries a cache that a later masked
            # ``signal[mask] = ...`` could leave stale
            self.audio_data = self.audio_data.to(device)
        return self

    def float(self):
        self.audio_data = self.audio_data.float()
        return self

    def cpu(self):
        return self.to("cpu")

    def cuda(self):
        return self.to("cuda")

    def numpy(self):
        return self.audio_data.detach().cpu().numpy()

    # ------------------------------------------------------------------ length ops
    def to_mono(self):
        self.audio_data = self.audio_data.mean(1, keepdim=True)
        return self

    def zero_pad(self, before: int, after: int):
        self.audio_data = torch.nn.functional.pad(self.audio_data, (before, after))
        return self

    def zero_pad_to(self, length: int, mode: str = "after"):
        if mode == "before":
            self.zero_pad(max(length - self.signal_length, 0), 0)
        elif mode == "after":
            self.zero_pad(0, max(length - self.signal_length, 0))
        return self

    def trim(self, before: int, after: int):
        self.audio_data = self.audio_data[..., before:] if after == 0 else self.audio_data[..., before:-after]
        return self

    def truncate_samples(self, length_in_samples: int):
        self.audio_data = self.audio_data[..., :length_in_samples]
        return self

    def resample(self, sample_rate: int):
        """Windowed-sinc polyphase resampling (ref :716-736 -> julius.resample_frac)."""
        if sample_rate == self.sample_rate:
            return self
        x = self.audio_data
        if _grad.wants_grad(x):
            self.audio_data = _grad.Resample.apply(x, int(self.sample_rate), int(sample_rate))
        else:
            self.audio_data = _engine().resample(x, int(self.sample_rate), int(sample_rate))
        self.sample_rate = sample_rate
        return self

    # ------------------------------------------------------------------ properties
    @property
    def device(self):
        if self._audio_data is not None:
            return self._audio_data.device
        if self.stft_data is not None:
            return self.stft_data.device

    @property
    def audio_data(self):
        """[B, C, T] samples.  A gain deferred by ``normalize`` / ``volume_change`` is applied here
        on first access (one pass of the gain kernel) unless a spectral kernel consumed it first."""
        if self._pending_gain is not None:
            self._materialized()
        return self._audio_data

    @audio_data.setter
    def audio_data(self, data):
        if data is not None:
            assert torch.is_tensor(data), "audio_data should be torch.Tensor"
            assert data.ndim == 3, "audio_data should be 3-dim (B, C, T)"
        self._audio_data = data
        self._pending_gain = None
        self._loudness = None  # any new waveform invalidates the cached loudness
        return

    def _defer_gain(self, gain: torch.Tensor):
        """``audio_data = audio_data * gain[:, None, None]`` with the multiply postponed so that it
        can ride along the next kernel that reads the samples (ref:audiotools/core/effects.py:219,237).
        Same observable state as the reference's assignment: the loudness cache is dropped."""
        gain = gain.reshape(-1).float()
        if _grad.wants_grad(gain):
            raise NotImplementedError("normalize / volume_change: db requires a gradient; gradients reach audio_data "
                                      "only (the gain is a constant, as the reference's loudness is not differentiable)")
        if _grad.wants_grad(self._audio_data) and _on_engine(self._audio_data):
            # a signal that carries a gradient is scaled at once, by the differentiable gain op (after any gain that
            # was deferred while grad mode was off)
            self.audio_data = _grad.Gain.apply(self._materialized(), gain)
            return
        if not self._audio_data.is_cuda:  # plain container arithmetic, like ``signal * x``
            self.audio_data = self._audio_data * gain.to(self._audio_data.device)[:, None, None]
            return
        self._pending_gain = gain if self._pending_gain is None else self._pending_gain * gain
        self._loudness = None

    def _materialized(self) -> torch.Tensor:
        """The sample tensor with any deferred gain applied."""
        if self._pending_gain is not None:
            g, self._pending_gain = self._pending_gain, None
            if _grad.wants_grad(self._audio_data):
                self._audio_data = _grad.Gain.apply(self._audio_data, g)
            else:
                self._audio_data = _engine().gain(self._audio_data, g)
        return self._audio_data

    samples = audio_data

    @property
    def stft_data(self):
        return self._stft_data

    @stft_data.setter
    def stft_data(self, data):
        if data is not None:
            assert torch.is_tensor(data) and torch.is_complex(data)
            if self.stft_data is not None and self.stft_data.shape != data.shape:
                warnings.warn("stft_data changed shape")
        self._stft_data = data
        return

    @property
    def batch_size(self):
        return self._audio_data.shape[0]

    @property
    def signal_length(self):
        return self._audio_data.shape[-1]

    length = signal_length

    @property
    def shape(self):
        return self._audio_data.shape

    @property
    def signal_duration(self):
        return self.signal_length / self.sample_rate

    duration = signal_duration

    @property
    def num_channels(self):
        return self._audio_data.shape[1]

    # ------------------------------------------------------------------ STFT
    @staticmethod
    @functools.lru_cache(None)
    def get_window(window_type: str, window_length: int, device: str):
        """scipy window (periodic), float64 -> float32; ``sqrt_hann`` and ``average`` specials (ref :1009-1039).
        Cached per (type, length, device): the reference rebuilds and re-uploads it on every stft/istft call."""
        return _cached_window(str(window_type), int(window_length), str(device))

    @property
    def stft_params(self):
        return self._stft_params

    @stft_params.setter
    def stft_params(self, value: STFTParams):
        win = int(2 ** (np.ceil(np.log2(0.032 * self.sample_rate))))
        defaults = STFTParams(window_length=win, hop_length=win // 4, window_type="hann",
                              match_stride=False, padding_type="reflect")._asdict()
        value = value._asdict() if value else defaults
        for k in defaults:
            if value[k] is None:
                value[k] = defaults[k]
        self._stft_params = STFTParams(**value)
        self.stft_data = None

    def compute_stft_padding(self, window_length: int, hop_length: int, match_stride: bool):
        """-> (right_pad, pad)  (ref :1089-1121)."""
        length = self.signal_length
        if match_stride:
            assert hop_length == window_length // 4, "For match_stride, hop must equal n_fft // 4"
            return math.ceil(length / hop_length) * hop_length - length, (window_length - hop_length) // 2
        return 0, 0

    def _resolve_stft(self, window_length, hop_length, window_type, match_stride, padding_type):
        sp = self.stft_params
        return (sp.window_length if window_length is None else int(window_length),
                sp.hop_length if hop_length is None else int(hop_length),
                sp.window_type if window_type is None else window_type,
                sp.match_stride if match_stride is None else match_stride,
                sp.padding_type if padding_type is None else padding_type)

    def _spectral(self, stft_args, method="stft", **engine_kwargs):
        window_length, hop_length, window_type, match_stride, padding_type = self._resolve_stft(*stft_args)
        window = self.get_window(window_type, window_length, self._audio_data.device)
        right_pad, pad = self.compute_stft_padding(window_length, hop_length, match_stride)
        if _grad.wants_grad(self._audio_data):
            fb = engine_kwargs.get("mel_fb")
            _grad.check_supported(method, window_length, hop_length, self.batch_size * self.num_channels,
                                  0 if fb is None else fb.shape[0])
            mel = None
            if engine_kwargs.get("mel_fb") is not None:
                mel = (engine_kwargs["mel_fb"], engine_kwargs["mel_lo"], engine_kwargs["mel_hi"],
                       engine_kwargs.get("post", 0), engine_kwargs.get("post_eps", 0.0),
                       engine_kwargs.get("post_power", 1.0))
            x = self._materialized()  # a gain deferred while grad mode was off is applied first, differentiably
            stft, mel_out = _grad.Spectral.apply(x, window_length, hop_length, window, pad, right_pad, padding_type,
                                                 2 if match_stride else 0, mel, engine_kwargs.get("want_stft", True))
            return {"stft": stft, "mel": mel_out, "scaled": None}
        gain = self._pending_gain
        if gain is not None and (pad or right_pad or match_stride):
            gain = None
            self._materialized()
        out = _engine().spectral(self._audio_data, window_length, hop_length, window, pad=pad, right_pad=right_pad,
                                 pad_mode=padding_type, drop_edge=2 if match_stride else 0, gain=gain,
                                 want_scaled=gain is not None, **engine_kwargs)
        if gain is not None:  # the deferred gain rode along: the scaled waveform came out of the same pass
            self._audio_data, self._pending_gain = out["scaled"], None
        return out

    def stft(self, window_length: int = None, hop_length: int = None, window_type: str = None,
             match_stride: bool = None, padding_type: str = None):
        """Centre-reflect-padded, one-sided, un-normalised STFT -> complex64 [B, C, F, N]; cached in
        ``stft_data`` (ref :1123-1212)."""
        out = self._spectral((window_length, hop_length, window_type, match_stride, padding_type), want_stft=True)
        self.stft_data = out["stft"]
        return self.stft_data

    def istft(self, window_length: int = None, hop_length: int = None, window_type: str = None,
              match_stride: bool = None, length: int = None):
        """Inverse STFT of ``stft_data`` into ``audio_data`` (ref :1214-1296): one fused kernel (inverse real FFT,
        window, overlap-add, envelope division; ``csrc/istft.cu``) for power-of-two windows in [64, 2048]; powers of two
        in [4096, 32768] run a per-frame inverse FFT (``csrc/fft_large.cu``) and every other window length a dense
        inverse DFT (``csrc/dft.cu``), both followed by the overlap-add fold of dft.cu.  No ``torch.istft`` on the path."""
        if self.stft_data is None:
            raise RuntimeError("Cannot do inverse STFT without self.stft_data!")
        window_length, hop_length, window_type, match_stride, _ = self._resolve_stft(
            window_length, hop_length, window_type, match_stride, None)
        window = self.get_window(window_type, window_length, self.stft_data.device)
        right_pad, pad = self.compute_stft_padding(window_length, hop_length, match_stride)
        if length is None:
            length = self.original_signal_length + 2 * pad + right_pad
        eng = _engine()  # (the engine refuses CPU tensors)
        if _grad.wants_grad(self.stft_data):
            _grad.check_supported("istft", window_length, hop_length, self.stft_data.shape[0] * self.stft_data.shape[1])
            pad_frames, trim, out_len = (2, pad, length - 2 * pad - right_pad) if match_stride else (0, 0, length)
            self.audio_data = _grad.ISTFT.apply(self.stft_data, window_length, hop_length, window, out_len, pad_frames,
                                                trim)
            return self
        if match_stride:
            # the reference pads 2 zero frames on either side, inverts to `length`, then keeps
            # [pad : length - (pad + right_pad)] (:1276-1292)
            audio = eng.istft(self.stft_data, window_length, hop_length, window,
                              length=length - 2 * pad - right_pad, pad_frames=2, trim=pad)
        else:
            audio = eng.istft(self.stft_data, window_length, hop_length, window, length=length)
        self.audio_data = audio
        return self

    @staticmethod
    def get_mel_filters(sr: int, n_fft: int, n_mels: int, fmin: float = 0.0, fmax: float = None):
        return _mel.mel_filters(sr, n_fft, n_mels, fmin, fmax)

    @staticmethod
    @functools.lru_cache(None)
    def _mel_tables(sr, n_fft, n_mels, fmin, fmax, device):
        fb = _mel.mel_filters(sr, n_fft, n_mels, fmin, fmax)
        lo, hi = _mel.band_table(fb)
        return (torch.from_numpy(np.array(fb)).to(device), torch.from_numpy(lo).to(device),
                torch.from_numpy(hi).to(device))

    def mel_spectrogram(self, n_mels: int = 80, mel_fmin: float = 0.0, mel_fmax: float = None,
                        log: bool = False, clamp_eps: float = 1e-5, pow: float = 2.0, **kwargs):
        """|STFT| x Slaney mel filterbank -> [B, C, n_mels, N] (ref :1333-1369).  One fused kernel;
        ``stft_data`` is NOT materialised.  ``log=True`` additionally fuses the reference's log-mel
        ``mel.clamp(clamp_eps).pow(pow).log10()`` (ref:audiotools/metrics/spectral.py:187-190)."""
        args = tuple(kwargs.pop(k, None) for k in
                     ("window_length", "hop_length", "window_type", "match_stride", "padding_type"))
        if kwargs:
            raise TypeError(f"unexpected stft arguments {sorted(kwargs)}")
        n_fft = self._resolve_stft(*args)[0]
        fb, lo, hi = self._mel_tables(self.sample_rate, n_fft, n_mels, mel_fmin, mel_fmax, self._audio_data.device)
        from .. import _lib

        out = self._spectral(args, method="mel_spectrogram", want_stft=False, mel_fb=fb, mel_lo=lo, mel_hi=hi,
                             post=_lib.POST_LOG10 if log else _lib.POST_NONE, post_eps=clamp_eps, post_power=pow)
        return out["mel"]

    @staticmethod
    @functools.lru_cache(None)
    def get_dct(n_mfcc: int, n_mels: int, norm: str = "ortho", device: str = None):
        """DCT-II matrix [n_mels, n_mfcc] (what ``torchaudio.functional.create_dct`` returns)."""
        n = torch.arange(float(n_mels))
        k = torch.arange(float(n_mfcc)).unsqueeze(1)
        dct = torch.cos(math.pi / float(n_mels) * (n + 0.5) * k)
        if norm is None:
            dct *= 2.0
        else:
            assert norm == "ortho"
            dct[0] *= 1.0 / math.sqrt(2.0)
            dct *= math.sqrt(2.0 / float(n_mels))
        return dct.t().to(device)

    def mfcc(self, n_mfcc: int = 40, n_mels: int = 80, log_offset: float = 1e-6, **kwargs):
        """log(mel + log_offset) @ DCT (ref :1398-1426); the log is fused behind the mel kernel."""
        args = tuple(kwargs.pop(k, None) for k in
                     ("window_length", "hop_length", "window_type", "match_stride", "padding_type"))
        mel_fmin, mel_fmax = kwargs.pop("mel_fmin", 0.0), kwargs.pop("mel_fmax", None)
        n_fft = self._resolve_stft(*args)[0]
        fb, lo, hi = self._mel_tables(self.sample_rate, n_fft, n_mels, mel_fmin, mel_fmax, self._audio_data.device)
        from .. import _lib

        logmel = self._spectral(args, method="mfcc", want_stft=False, mel_fb=fb, mel_lo=lo, mel_hi=hi,
                                post=_lib.POST_LN, post_eps=log_offset)["mel"]
        dct = self.get_dct(n_mfcc, n_mels, "ortho", self.device)
        if _grad.wants_grad(logmel):
            return _grad.MelDCT.apply(logmel, dct)
        return _engine().mel_dct(logmel, dct)

    @property
    def magnitude(self):
        if self.stft_data is None:
            self.stft()
        return torch.abs(self.stft_data)

    @magnitude.setter
    def magnitude(self, value):
        self.stft_data = value * torch.exp(1j * self.phase)

    def log_magnitude(self, ref_value: float = 1.0, amin: float = 1e-5, top_db: float = 80.0):
        magnitude = self.magnitude
        amin = amin ** 2
        log_spec = 10.0 * torch.log10(magnitude.pow(2).clamp(min=amin))
        log_spec -= 10.0 * np.log10(np.maximum(amin, ref_value))
        if top_db is not None:
            log_spec = torch.maximum(log_spec, log_spec.max() - top_db)
        return log_spec

    @property
    def phase(self):
        if self.stft_data is None:
            self.stft()
        return torch.angle(self.stft_data)

    @phase.setter
    def phase(self, value):
        self.stft_data = self.magnitude * torch.exp(1j * value)

    # ------------------------------------------------------------------ arithmetic
    def __add__(self, other):
        new = self.clone()
        new.audio_data += util._get_value(other)
        return new

    def __iadd__(self, other):
        self.audio_data += util._get_value(other)
        return self

    def __radd__(self, other):
        return self + other

    def __sub__(self, other):
        new = self.clone()
        new.audio_data -= util._get_value(other)
        return new

    def __isub__(self, other):
        self.audio_data -= util._get_value(other)
        return self

    def __mul__(self, other):
        new = self.clone()
        new.audio_data *= util._get_value(other)
        return new

    def __imul__(self, other):
        self.audio_data *= util._get_value(other)
        return self

    def __rmul__(self, other):
        return self * other

    # ------------------------------------------------------------------ repr / compare
    def _info(self):
        dur = f"{self.signal_duration:0.3f}" if self.signal_duration else "[unknown]"
        return {
            "duration": f"{dur} seconds",
            "batch_size": self.batch_size,
            "path": self.path_to_file if self.path_to_file else "path unknown",
            "sample_rate": self.sample_rate,
            "num_channels": self.num_channels if self.num_channels else "[unknown]",
            "audio_data.shape": self.audio_data.shape,
            "stft_params": self.stft_params,
            "device": self.device,
        }

    def markdown(self):
        rows = "".join(f"| {k} | {v} |\n" for k, v in self._info().items())
        return "| Key | Value \n|---|--- \n" + rows

    def __str__(self):
        return "".join(f"{k}: {v}\n" for k, v in self._info().items())

    def __eq__(self, other):
        self._materialized()
        other._materialized()
        for k, v in list(self.__dict__.items()):
            if torch.is_tensor(v):
                if not torch.is_tensor(other.__dict__.get(k)):
                    return False
                if not torch.allclose(v, other.__dict__[k], atol=1e-6):
                    print(f"Max abs error for {k}: {(v - other.__dict__[k]).abs().max()}")
                    return False
        return True

    def __ne__(self, other):
        return not self == other

    __hash__ = object.__hash__

    # ------------------------------------------------------------------ batch-dim indexing
    @staticmethod
    def _is_whole_item_key(key):
        return torch.is_tensor(key) and key.ndim == 0 and key.item() is True

    @staticmethod
    def _is_batch_key(key):
        return isinstance(key, (bool, int, list, slice, tuple)) or (torch.is_tensor(key) and key.ndim <= 1)

    def __getitem__(self, key):
        if self._is_whole_item_key(key):
            assert self.batch_size == 1
            audio, loud, stft = self.audio_data, self._loudness, self.stft_data
        elif self._is_batch_key(key):
            audio = self.audio_data[key]
            loud = self._loudness[key] if self._loudness is not None else None
            stft = self.stft_data[key] if self.stft_data is not None else None
        else:
            raise TypeError(f"unsupported AudioSignal index {key!r}")
        out = type(self)(audio, self.sample_rate, stft_params=self.stft_params)
        out._loudness = loud
        out._stft_data = stft
        out.sources = None
        return out

    def __setitem__(self, key, value):
        if not isinstance(value, type(self)):
            self.audio_data[key] = value
            return
        if self._is_whole_item_key(key):
            assert self.batch_size == 1
            self.audio_data = value.audio_data
            self._loudness = value._loudness
            self.stft_data = value.stft_data
            return
        if self._is_batch_key(key):
            # index_put into the existing tensors: does not go through the audio_data setter, so the
            # loudness cache of untouched items survives (ref :1658-1679; Silence relies on it)
            if self.audio_data is not None and value.audio_data is not None:
                self.audio_data[key] = value.audio_data
            if self._loudness is not None and value._loudness is not None:
                self._loudness[key] = value._loudness
            if self.stft_data is not None and value.stft_data is not None:
                self.stft_data[key] = value.stft_data
