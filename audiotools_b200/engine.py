"""Tensor-level entry points over the C ABI of ``libb2a`` (``include/b2a.h``).

One ``Engine`` wraps one loaded library.  Inputs are float32 CUDA tensors; every
call is enqueued on torch's current stream of the tensor's device and returns
torch tensors that torch allocated (the library owns no buffers).  There is no
CPU path: a non-CUDA tensor raises.  (``require_cuda=False`` exists only so that
tests can drive the *same marshalling code* against ``tests/cusim``'s CPU build of
the kernels; the module-level engine is always built with ``require_cuda=True``.)
"""
import ctypes
import math
import sys
from typing import Optional

import numpy as np
import torch

from . import _lib
from .core import kweighting
from .core import room as _room


def _dptr(t: Optional[torch.Tensor]):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


class Engine:
    def __init__(self, lib: _lib.B2ALibrary, require_cuda: bool = True):
        self.lib = lib
        self.require_cuda = require_cuda
        self.launches = 0  # kernels of libb2a launched through this engine (bench.py reports it)
        self._packed_cache = {}
        self._routes = {}
        self._crossovers = {}  # octave_crossovers: (rate, bands, device) -> (taps, half)

    # ------------------------------------------------------------------ helpers
    DIFFERENTIABLE = ("AudioSignal.stft", "istft", "mel_spectrogram", "mfcc", "normalize", "volume_change",
                      "and magnitude / phase / log_magnitude through stft_data; resample, equalizer, convolve, apply_ir, "
                      "ensure_max_of_audio, mix, quantization, mulaw_quantization, sos_filter, parametric_eq, core.iir.sosfiltfilt (gradients to "
                      "audio_data); "
                      "mask_frequencies, mask_timesteps, mask_low_magnitudes, ml.layers.SpectralGate (gradients to "
                      "stft_data / the gated signal); metrics.STOILoss, metrics.LoudnessLoss (gradients to the "
                      "estimates)")

    @classmethod
    def _refuse_grad(cls, t: torch.Tensor, name: str):
        """A tensor that requires a gradient while grad mode is on reaches a kernel without a backward: raise instead
        of returning a silently detached result.  The message names the engine method that was called: the innermost
        caller whose name does not start with an underscore, so private helpers (``_prep``, ``_per_item``,
        ``_band_args``, ...) and dunder callers (a transform's ``__call__``) are skipped."""
        if t.requires_grad and torch.is_grad_enabled():
            frame = sys._getframe(1)
            while frame.f_code.co_name.startswith("_") and frame.f_back is not None:
                frame = frame.f_back
            raise NotImplementedError(
                f"{frame.f_code.co_name}: {name} requires a gradient, and this method has no backward.  "
                f"Differentiable: {', '.join(cls.DIFFERENTIABLE)}.  Call it under torch.no_grad() or on a detached "
                "signal.")

    def _prep(self, t: torch.Tensor, name: str, dtype=torch.float32) -> torch.Tensor:
        if not torch.is_tensor(t):
            raise TypeError(f"{name} must be a torch.Tensor")
        self._refuse_grad(t, name)
        if self.require_cuda and not t.is_cuda:
            raise RuntimeError(
                f"{name} is on {t.device}: audiotools_b200 runs on CUDA (sm_90a) only and has no CPU fallback")
        if t.dtype != dtype:
            t = t.to(dtype)
        return t.contiguous()

    def _per_item(self, v, n: int, name: str, device) -> torch.Tensor:
        """``v`` (a tensor, number or sequence of 1 or ``n`` values) as a contiguous float32 [n] tensor on ``device``:
        one value is broadcast to all ``n`` items."""
        v = torch.as_tensor(v).reshape(-1).to(device=device, dtype=torch.float32)
        assert v.numel() in (1, n), f"{name} must have 1 or {n} entries, got {v.numel()}"
        self._refuse_grad(v, name)
        return v.expand(n).contiguous()

    def _stream(self, t: torch.Tensor):
        """The stream the call is issued on.  Every entry point of the library launches on the CURRENT device, so a
        tensor that lives on another GPU of the process (``AudioSignal(..., device="cuda:1")``) makes its device
        current first -- the attribute / occupancy queries and the launch then all refer to the tensor's device."""
        if t.is_cuda:
            if torch.cuda.current_device() != t.device.index:
                torch.cuda.set_device(t.device)
            return ctypes.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)
        return None

    def _call(self, fn, *args):
        """Every call of an entry point that launches kernels goes through here: raise on its error code, and count
        the kernels it launched in ``launches``."""
        self.launches += self.lib.call(fn, *args)

    # ------------------------------------------------------------------ inverse STFT
    @staticmethod
    def _envelope_min(window: torch.Tensor, n_fft: int, hop: int, n_frames: int, start: int, end: int) -> float:
        """min over [start, end) of sum_n w^2[t - n*hop] (host, float64): the quantity torch.istft checks.  The
        envelope is hop-periodic away from the first / last n_fft samples, so edges + one period suffice."""
        w2 = window.detach().double().cpu().numpy() ** 2
        total = (n_frames - 1) * hop + n_fft
        end = min(end, total)
        if end <= start:
            return float("inf")

        def env_at(ts):
            ts = np.asarray(ts, dtype=np.int64)
            out = np.zeros(len(ts))
            n_hi = np.minimum(ts // hop, n_frames - 1)
            for d in range((n_fft + hop - 1) // hop + 1):
                n = n_hi - d
                off = ts - n * hop
                ok = (n >= 0) & (off >= 0) & (off < n_fft)
                out[ok] += w2[off[ok]]
            return out

        edge = 2 * n_fft + hop
        if end - start <= 2 * edge + hop:
            ts = np.arange(start, end)
        else:
            ts = np.concatenate([np.arange(start, start + edge), np.arange(end - edge, end)])
        return float(env_at(ts).min())

    def istft(self, spec: torch.Tensor, n_fft: int, hop: int, window: torch.Tensor, length: int,
              pad_frames: int = 0, trim: int = 0) -> torch.Tensor:
        """``torch.istft(spec, n_fft, hop, window=window, length=..., center=True)`` for spec [B, C, F, N] complex64
        (ref:audiotools/core/audio_signal.py:1214-1296) -> [B, C, length].  ``pad_frames`` zero frames are put back
        on either side and ``trim`` extra leading samples are dropped (the reference's match_stride handling)."""
        spec = self._spec_ok(spec, "istft")
        B, C, F, N = spec.shape
        assert F == n_fft // 2 + 1, (F, n_fft)
        route = self.route(n_fft, hop, 1)
        if route == _lib.ROUTE_NONE:
            raise self.route_error(n_fft, hop, 1)
        window = self._prep(window, "window")
        assert window.numel() == n_fft
        start = n_fft // 2 + int(trim)
        # torch.istft's "window overlap add min" check, evaluated on the host once per (window, geometry): the key
        # holds the window tensor itself (the caller caches its windows), so a re-used window costs no sync
        key = ("istft_env", window.data_ptr(), int(window._version), n_fft, hop, N + 2 * pad_frames, start, int(length))
        if key not in self._packed_cache:
            stale = [k for k in self._packed_cache if k[0] == "istft_env"]
            if len(stale) >= 64:  # bounded: one entry per distinct (window, geometry, length)
                for k in stale[:32]:
                    del self._packed_cache[k]
            self._packed_cache[key] = (window, self._envelope_min(window, n_fft, hop, N + 2 * pad_frames, start,
                                                                  start + int(length)))
        if self._packed_cache[key][1] < 1e-11:
            raise RuntimeError("istft: window overlap add min: 1 (the window envelope vanishes inside the output)")
        out = torch.empty(B, C, int(length), dtype=torch.float32, device=spec.device)
        imat = self.dft_matrix(window, int(n_fft), inverse=1) if route == _lib.ROUTE_DENSE else None
        nbytes = int(self.lib.b2a_istft_workspace_bytes(B * C, N, int(n_fft), int(hop)))
        ws = torch.empty((nbytes + 3) // 4, dtype=torch.float32, device=spec.device) if nbytes else None
        self._call(self.lib.b2a_istft_f32, _dptr(spec), B * C, N, int(n_fft), int(hop), _dptr(window), _dptr(imat),
                   int(pad_frames), start, int(length), _dptr(out), _dptr(ws), nbytes, self._stream(spec))
        return out

    # ------------------------------------------------------------------ backward passes (csrc/grad.cu)
    def backward_supported(self, n_fft: int, hop: int) -> bool:
        return self.route(n_fft, hop, 1) != _lib.ROUTE_NONE

    def stft_backward(self, grad_spec: torch.Tensor, T: int, n_fft: int, hop: int, window: torch.Tensor, pad: int = 0,
                      right_pad: int = 0, pad_mode: str = "reflect", drop_edge: int = 0) -> torch.Tensor:
        """Gradient wrt x [B, C, T] of ``spectral``'s STFT from grad_spec [B, C, F, N] (complex, torch's convention)."""
        grad_spec = self._complex64(grad_spec)
        B, C, F, N = grad_spec.shape
        window = self._prep(window, "window")
        nbytes = int(self.lib.b2a_stft_backward_workspace_bytes(B * C, int(T), int(n_fft), int(hop), int(pad),
                                                                int(right_pad), int(drop_edge)))
        if nbytes == 0:
            raise NotImplementedError(f"stft backward: window_length {n_fft} hop {hop}")
        route = self.route(n_fft, hop, 1)
        amat = self.dft_matrix(window, int(n_fft), inverse=2) if route == _lib.ROUTE_DENSE else None
        ws = torch.empty((nbytes + 3) // 4, dtype=torch.float32, device=grad_spec.device)
        gx = torch.empty(B, C, int(T), dtype=torch.float32, device=grad_spec.device)
        self._call(self.lib.b2a_stft_backward_f32, _dptr(grad_spec), B * C, int(T), int(n_fft), int(hop), _dptr(window),
                   _dptr(amat), int(pad), int(right_pad), _lib.PAD_MODES[pad_mode], int(drop_edge), _dptr(gx), _dptr(ws),
                   nbytes, self._stream(grad_spec))
        return gx

    def istft_backward(self, grad_out: torch.Tensor, n_frames: int, n_fft: int, hop: int, window: torch.Tensor,
                       pad_frames: int = 0, trim: int = 0) -> torch.Tensor:
        """Gradient wrt spec [B, C, F, n_frames] (complex64) of ``istft`` from grad_out [B, C, length]."""
        grad_out = grad_out.to(torch.float32).contiguous()
        B, C, L = grad_out.shape
        window = self._prep(window, "window")
        mat = self.dft_matrix(window, int(n_fft), inverse=0) if self.route(n_fft, hop, 1) == _lib.ROUTE_DENSE else None
        nbytes = int(self.lib.b2a_istft_backward_workspace_bytes(B * C, L))
        ws = torch.empty((nbytes + 3) // 4, dtype=torch.float32, device=grad_out.device)
        gs = torch.empty(B, C, n_fft // 2 + 1, int(n_frames), dtype=torch.complex64, device=grad_out.device)
        self._call(self.lib.b2a_istft_backward_f32, _dptr(grad_out), B * C, int(n_frames), int(n_fft), int(hop),
                   _dptr(window), _dptr(mat), int(pad_frames), n_fft // 2 + int(trim), L, _dptr(gs), _dptr(ws), nbytes,
                   self._stream(grad_out))
        return gs

    def _bin_table(self, mel_lo: torch.Tensor, mel_hi: torch.Tensor, F: int):
        """[F] int32 (bin_lo, bin_hi): the filters whose band may hold bin k lie in [bin_lo[k], bin_hi[k]) -- the
        transposed band table of the mel backward, built on the host once per filterbank (the entry keeps both alive)."""
        key = ("bins", mel_lo.data_ptr(), mel_hi.data_ptr(), mel_lo.numel(), int(F))
        if key not in self._packed_cache:
            lo, hi = mel_lo.cpu().numpy().astype("int64"), mel_hi.cpu().numpy().astype("int64")
            blo = np.full(F, len(lo), dtype=np.int32)
            bhi = np.zeros(F, dtype=np.int32)
            for m in range(len(lo)):
                if hi[m] > lo[m]:
                    blo[lo[m]:hi[m]] = np.minimum(blo[lo[m]:hi[m]], m)
                    bhi[lo[m]:hi[m]] = np.maximum(bhi[lo[m]:hi[m]], m + 1)
            blo = np.minimum(blo, bhi)
            dev = mel_lo.device
            self._packed_cache[key] = (torch.from_numpy(blo).to(dev), torch.from_numpy(bhi).to(dev), mel_lo, mel_hi)
        return self._packed_cache[key][:2]

    def mel_backward(self, stft: torch.Tensor, grad_mel: torch.Tensor, mel_fb: torch.Tensor, mel_lo: torch.Tensor,
                     mel_hi: torch.Tensor, post: int = _lib.POST_NONE, post_eps: float = 0.0,
                     post_power: float = 1.0) -> torch.Tensor:
        """Gradient wrt the complex STFT [B, C, F, N] of ``spectral``'s mel output from grad_mel [B, C, n_mels, N]."""
        stft = self._complex64(stft)
        B, C, F, N = stft.shape
        grad_mel = grad_mel.to(torch.float32).contiguous()
        mel_fb = self._prep(mel_fb, "mel_fb")
        mel_lo = self._prep(mel_lo, "mel_lo", torch.int32)
        mel_hi = self._prep(mel_hi, "mel_hi", torch.int32)
        bin_lo, bin_hi = self._bin_table(mel_lo, mel_hi, F)
        out = torch.empty_like(stft)
        self._call(self.lib.b2a_mel_backward_f32, _dptr(stft), B * C, F, N, _dptr(mel_fb), _dptr(mel_lo), _dptr(mel_hi),
                   mel_fb.shape[0], _dptr(bin_lo), _dptr(bin_hi), int(post), float(post_eps), float(post_power),
                   _dptr(grad_mel), _dptr(out), self._stream(stft))
        return out

    # ------------------------------------------------------------------ spectral L1 losses (csrc/loss.cu)
    def spectral_loss_supported(self, n_fft: int, hop: int, n_mels: int = 0) -> bool:
        return bool(self.lib.b2a_spectral_loss_supported(int(n_fft), int(hop), int(n_mels)))

    def spectral_loss(self, x: torch.Tensor, y: torch.Tensor, n_fft: int, hop: int, window: torch.Tensor, pad: int = 0,
                      right_pad: int = 0, pad_mode: str = "reflect", drop_edge: int = 0, mel=None,
                      clamp_eps: float = 1e-5, pow: float = 2.0, log_weight: float = 1.0, mag_weight: float = 1.0,
                      want_grad_x: bool = False, want_grad_y: bool = False):
        """One scale of the reference's L1 spectral losses (MultiScaleSTFTLoss, or MelSpectrogramLoss with
        ``mel=(fb, lo, hi)``) between x and y [B, C, T] -> (loss, dL/dX, dL/dY): a 0-dim float32 tensor and, when asked
        for, the gradients wrt the two STFTs [B, C, F, N] complex64 (``stft_backward`` takes them to the waveforms)."""
        x = self._prep(x, "x")
        y = self._prep(y, "y")
        assert x.ndim == 3 and x.shape == y.shape, (x.shape, y.shape)
        B, C, T = x.shape
        if pad_mode not in _lib.PAD_MODES:
            raise NotImplementedError(f"padding_type {pad_mode!r} (supported: {sorted(_lib.PAD_MODES)})")
        window = self._prep(window, "window")
        assert window.numel() == n_fft
        N = self.num_frames(T, n_fft, hop, pad, right_pad, drop_edge)
        F = n_fft // 2 + 1
        fb = lo = hi = blo = bhi = None
        n_mels = 0
        if mel is not None:
            fb, lo, hi = mel
            fb = self._prep(fb, "mel_fb")
            assert fb.shape[1] == F, (fb.shape, F)
            n_mels = fb.shape[0]
            lo = self._prep(lo, "mel_lo", torch.int32)
            hi = self._prep(hi, "mel_hi", torch.int32)
            blo, bhi = self._bin_table(lo, hi, F)
        nbytes = int(self.lib.b2a_spectral_loss_workspace_bytes(int(n_fft), int(hop), n_mels))
        if nbytes == 0:
            raise NotImplementedError(f"spectral_loss: window_length {n_fft} hop {hop} n_mels {n_mels}")
        dev = x.device
        ws = torch.empty((nbytes + 7) // 8, dtype=torch.float64, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        gx = torch.empty(B, C, F, max(N, 1), dtype=torch.complex64, device=dev) if want_grad_x else None
        gy = torch.empty(B, C, F, max(N, 1), dtype=torch.complex64, device=dev) if want_grad_y else None
        self._call(self.lib.b2a_spectral_loss_f32, _dptr(x), _dptr(y), B * C, T, int(n_fft), int(hop), _dptr(window),
                   int(pad), int(right_pad), _lib.PAD_MODES[pad_mode], int(drop_edge), _dptr(fb), _dptr(lo), _dptr(hi),
                   _dptr(blo), _dptr(bhi), n_mels, float(clamp_eps), float(pow), float(log_weight), float(mag_weight),
                   _dptr(loss), _dptr(gx), _dptr(gy), _dptr(ws), nbytes, self._stream(x))
        return loss, gx, gy

    # ------------------------------------------------------------------ STFT routes, dense DFT (any window length)
    def route(self, n_fft: int, hop: int, inverse: int) -> int:
        """``b2a_stft_route``: the kernel family (``_lib.ROUTE_*``) that runs the STFT (inverse 0) or the inverse STFT
        and both backward passes (inverse 1) of this geometry.  Memoised: ``stft()`` is launch-latency bound at
        batch=4 x 1 s, where a foreign-function call per call is measurable."""
        key = (n_fft, hop, inverse)
        r = self._routes.get(key)
        if r is None:
            r = self._routes[key] = int(self.lib.b2a_stft_route(int(n_fft), int(hop), int(inverse)))
        return r

    @staticmethod
    def route_error(n_fft: int, hop: int, inverse: int, backward_of: Optional[str] = None) -> NotImplementedError:
        """The error for a geometry whose route is ``ROUTE_NONE``: of the STFT (inverse 0), the inverse STFT (inverse 1),
        or, when ``backward_of`` names the differentiable method, of its backward."""
        if backward_of is not None:
            return NotImplementedError(
                f"{backward_of}: no backward for window_length {n_fft} hop {hop}: gradients through the STFT need "
                "hop <= window_length and a window of any length up to 8192 or a power of two up to 32768")
        msg = (f"istft: n_fft={n_fft} hop={hop}" if inverse else
               f"stft: window_length {n_fft} hop {hop}: the dense DFT path covers 2..8192")
        if n_fft > 32768 and (n_fft & (n_fft - 1)) == 0:
            msg += ": power-of-two windows run on the FFT kernels up to 32768"
        return NotImplementedError(msg)

    def dft_matrix(self, window: torch.Tensor, n_fft: int, inverse: int = 0) -> torch.Tensor:
        """The windowed DFT matrix of csrc/dft.cu for (n_fft, window), built on the device once and cached (the cache
        entry holds the window tensor, so its address / version identify it).  ``inverse``: 0 forward, 1 inverse
        (c_k / n_fft weights), 2 the STFT's adjoint (the inverse layout, weight 1)."""
        key = ("dft", window.data_ptr(), int(window._version), int(n_fft), int(inverse))
        hit = self._packed_cache.get(key)
        if hit is None:
            n = int(self.lib.b2a_dft_matrix_floats(int(n_fft), int(inverse)))
            if n == 0:
                raise NotImplementedError(f"window_length {n_fft}: the dense DFT path covers 2..8192")
            mat = torch.empty(n, dtype=torch.float32, device=window.device)
            self._call(self.lib.b2a_dft_matrix_f32, _dptr(window), int(n_fft), int(inverse), _dptr(mat),
                       self._stream(window))
            hit = self._packed_cache[key] = (mat, window)
        return hit[0]

    # ------------------------------------------------------------------ spectral masks
    def spec_band_mask(self, spec: torch.Tensor, axis_vals: torch.Tensor, lo: torch.Tensor, hi: torch.Tensor,
                       axis: int, val: float = 0.0) -> torch.Tensor:
        """In place: ``spec[b, c, f, n] = val * exp(1j * val)`` where ``lo[b] <= axis_vals[f or n] < hi[b]``
        (ref:audiotools/core/dsp.py:217-306).  spec [B, C, F, N] complex64, contiguous; returns it."""
        spec = self._spec_ok(spec, "spec_band_mask")
        B, C, F, N = spec.shape
        axis_vals, lo, hi = self._band_args(spec, axis_vals, lo, hi, axis)
        fill = self._band_fill(val)
        self._call(self.lib.b2a_spec_band_mask_f32, _dptr(spec), B * C, F, N, _dptr(axis_vals), _dptr(lo), _dptr(hi), C,
                   int(axis), float(fill.real), float(fill.imag), self._stream(spec))
        return spec

    def _band_args(self, spec, axis_vals, lo, hi, axis):
        B, _, F, N = spec.shape
        axis_vals = self._prep(axis_vals.to(spec.device), "axis_vals")
        assert axis_vals.numel() == (F if axis == 0 else N)
        return axis_vals, self._per_item(lo, B, "lo", spec.device), self._per_item(hi, B, "hi", spec.device)

    @staticmethod
    def _band_fill(val):
        v = torch.tensor(float(val), dtype=torch.float32)
        return v * torch.exp(1j * v)  # the reference's own arithmetic for a filled cell (complex64)

    def spec_band_mask_out(self, spec: torch.Tensor, axis_vals: torch.Tensor, lo: torch.Tensor, hi: torch.Tensor,
                           axis: int, val: float = 0.0) -> torch.Tensor:
        """``spec_band_mask`` into a new tensor (the forward of the gradient path: ``spec`` may be saved by autograd)."""
        spec = self._spec_ok(spec, "spec_band_mask_out")
        B, C, F, N = spec.shape
        axis_vals, lo, hi = self._band_args(spec, axis_vals, lo, hi, axis)
        fill = self._band_fill(val)
        out = torch.empty_like(spec)
        self._call(self.lib.b2a_spec_band_mask_out_f32, _dptr(spec), _dptr(out), B * C, F, N, _dptr(axis_vals),
                   _dptr(lo), _dptr(hi), C, int(axis), float(fill.real), float(fill.imag), self._stream(spec))
        return out

    def spec_band_mask_backward(self, grad: torch.Tensor, spec: torch.Tensor, axis_vals: torch.Tensor,
                                lo: torch.Tensor, hi: torch.Tensor, axis: int) -> torch.Tensor:
        """dL/dspec of ``spec_band_mask``: 0 in the band and where spec == 0, ``grad`` elsewhere (the reference's
        |X| exp(1j angle X) round trip, differentiated by torch)."""
        spec = self._spec_ok(spec, "spec_band_mask_backward")
        grad = self._spec_ok(grad, "spec_band_mask_backward")
        B, C, F, N = spec.shape
        assert grad.shape == spec.shape, (grad.shape, spec.shape)
        axis_vals, lo, hi = self._band_args(spec, axis_vals, lo, hi, axis)
        gs = torch.empty_like(spec)
        self._call(self.lib.b2a_spec_band_mask_backward_f32, _dptr(grad), _dptr(spec), B * C, F, N, _dptr(axis_vals),
                   _dptr(lo), _dptr(hi), C, int(axis), _dptr(gs), self._stream(spec))
        return gs

    def _spec_ok(self, spec: torch.Tensor, what: str) -> torch.Tensor:
        if not torch.is_complex(spec):
            raise TypeError(f"{what}: spec must be complex")
        self._refuse_grad(spec, "spec")
        if self.require_cuda and not spec.is_cuda:
            raise RuntimeError(f"stft_data is on {spec.device}: audiotools_b200 runs on CUDA (sm_90a) only and has "
                               "no CPU fallback")
        return self._complex64(spec)

    @staticmethod
    def _complex64(t: torch.Tensor) -> torch.Tensor:
        """``t`` as a contiguous complex64 tensor whose memory holds its values.  A lazy conjugate or negative view
        (``X.conj()``, which autograd hands to a backward when the loss used it) shares its buffer with ``X``, and the
        kernels read the buffer as it lies: such a view is resolved into a copy first."""
        return t.resolve_conj().resolve_neg().to(torch.complex64).contiguous()

    def spec_rotate(self, spec: torch.Tensor, shift: torch.Tensor) -> torch.Tensor:
        """``spec * exp(1j * shift)`` in place on a contiguous complex64 [B, ...] tensor (a copy otherwise);
        ``shift`` has B entries (one per item) or one per cell (ref:audiotools/core/dsp.py:335-351)."""
        spec = self._spec_ok(spec, "spec_rotate")
        B = spec.shape[0]
        cells = spec.numel() // B
        shift = self._prep(shift.to(spec.device), "shift").reshape(-1)
        per_cell = shift.numel() == spec.numel() and cells > 1
        if not per_cell:
            shift = self._per_item(shift, B, "shift", spec.device)
        self._call(self.lib.b2a_spec_rotate_f32, _dptr(spec), B, cells, _dptr(shift), int(per_cell), self._stream(spec))
        return spec

    def spec_mask_low(self, spec: torch.Tensor, db_cutoff: torch.Tensor, val: float = 0.0, amin: float = 1e-5,
                      top_db: float = 80.0) -> torch.Tensor:
        """``mask_low_magnitudes`` (ref:audiotools/core/dsp.py:308-333) in place: two passes (global max, mask)."""
        spec = self._spec_ok(spec, "spec_mask_low")
        B = spec.shape[0]
        cells = spec.numel() // B
        db_cutoff = self._per_item(db_cutoff, B, "db_cutoff", spec.device)
        ws = torch.empty(1, dtype=torch.int32, device=spec.device)
        self._call(self.lib.b2a_spec_mask_low_f32, _dptr(spec), B, cells, _dptr(db_cutoff), float(amin ** 2),
                   float(top_db), float(val), _dptr(ws), self._stream(spec))
        return spec

    def spec_mask_low_out(self, spec: torch.Tensor, db_cutoff: torch.Tensor, val: float = 0.0, amin: float = 1e-5,
                          top_db: float = 80.0):
        """``spec_mask_low`` into a new tensor (the forward of the gradient path) -> (out, ws): ws holds the maximum
        |X|^2 the top_db floor came from, for ``spec_mask_low_backward``."""
        spec = self._spec_ok(spec, "spec_mask_low_out")
        B = spec.shape[0]
        db_cutoff = self._per_item(db_cutoff, B, "db_cutoff", spec.device)
        out = torch.empty_like(spec)
        ws = torch.empty(1, dtype=torch.int32, device=spec.device)
        self._call(self.lib.b2a_spec_mask_low_out_f32, _dptr(spec), _dptr(out), B, spec.numel() // B, _dptr(db_cutoff),
                   float(amin ** 2), float(top_db), float(val), _dptr(ws), self._stream(spec))
        return out, ws

    def spec_mask_low_backward(self, grad: torch.Tensor, spec: torch.Tensor, db_cutoff: torch.Tensor, val: float,
                               ws: torch.Tensor, amin: float = 1e-5, top_db: float = 80.0) -> torch.Tensor:
        """dL/dspec of ``mask_low_magnitudes`` with the mask recomputed from ``spec`` and the forward's ``ws``: unmasked
        cells pass ``grad``; masked cells (magnitude := val, phase kept) follow the phase, val (g - Re(g conj u) u) / |X|;
        0 where spec == 0."""
        spec = self._spec_ok(spec, "spec_mask_low_backward")
        grad = self._spec_ok(grad, "spec_mask_low_backward")
        assert grad.shape == spec.shape, (grad.shape, spec.shape)
        B = spec.shape[0]
        db_cutoff = self._per_item(db_cutoff, B, "db_cutoff", spec.device)
        gs = torch.empty_like(spec)
        self._call(self.lib.b2a_spec_mask_low_backward_f32, _dptr(grad), _dptr(spec), B, spec.numel() // B,
                   _dptr(db_cutoff), float(amin ** 2), float(top_db), float(val), _dptr(ws), _dptr(gs),
                   self._stream(spec))
        return gs

    def alter_drr(self, ir: torch.Tensor, sample_rate: int, drr: torch.Tensor) -> torch.Tensor:
        """``ImpulseResponseMixin.alter_drr`` (ref:audiotools/core/effects.py:540-647) for ir [B, C, T] and drr [B]:
        early / late split at the direct path, alpha from the DRR quadratic, re-weighting and the peak limit in one
        launch (csrc/effects.cu)."""
        ir = self._prep(ir, "ir")
        B, C, T = ir.shape
        drr = self._per_item(drr, B, "drr", ir.device)
        out = torch.empty_like(ir)
        self._call(self.lib.b2a_alter_drr_f32, _dptr(ir), _dptr(out), B * C, T, C, int(sample_rate * 0.0025), _dptr(drr),
                   1.0, self._stream(ir))
        return out

    def spec_gate(self, spec: torch.Tensor, nz_spec: torch.Tensor, n_std: float, amount: torch.Tensor,
                  smooth_f, smooth_t):
        """The spectral noise gate's mask algebra (ref:audiotools/ml/layers/spectral_gate.py:97-124) as two launches:
        per-bin threshold from the noise STFT's dB statistics, then boolean -> separable 2-D smoothing ->
        ``spec * (1 - amount * mask)`` in one pass.  spec [B, C, F, N], nz_spec [1 or B, 1 or C, F, Nz] complex64;
        amount: scalar or [B]; smooth_f / smooth_t: the two 1-D factors of the smoothing kernel.  Returns (a new
        tensor, the thresholds [nz rows, F] that ``spec_gate_backward`` takes)."""
        spec = self._spec_ok(spec, "spec_gate")
        B, C, F, N = spec.shape
        nz_spec = self._spec_ok(nz_spec, "spec_gate")
        if nz_spec.shape[:2] != (1, 1):
            nz_spec = nz_spec.expand(B, C, -1, -1).contiguous()
        assert nz_spec.shape[2] == F, (nz_spec.shape, F)
        nz_rows = nz_spec.shape[0] * nz_spec.shape[1]
        amount = self._per_item(amount, B, "amount", spec.device)
        sf, st = self._gate_smoothing(smooth_f, smooth_t)
        out = torch.empty_like(spec)
        ws = torch.empty(nz_rows * F, dtype=torch.float32, device=spec.device)
        self._call(self.lib.b2a_spec_gate_f32, _dptr(spec), B * C, F, N, _dptr(nz_spec), nz_rows, nz_spec.shape[-1],
                   float(n_std), _dptr(amount), C, sf, len(smooth_f), st, len(smooth_t), _dptr(out), _dptr(ws),
                   self._stream(spec))
        return out, ws.reshape(nz_rows, F)

    @staticmethod
    def _gate_smoothing(smooth_f, smooth_t):
        return ((ctypes.c_float * len(smooth_f))(*[float(v) for v in smooth_f]),
                (ctypes.c_float * len(smooth_t))(*[float(v) for v in smooth_t]))

    def spec_gate_backward(self, grad: torch.Tensor, spec: torch.Tensor, thresh: torch.Tensor, amount: torch.Tensor,
                           smooth_f, smooth_t) -> torch.Tensor:
        """dL/dspec of ``spec_gate``: ``grad * (1 - amount * mask)``, the smoothed mask recomputed from ``spec`` and the
        forward's thresholds (the mask comes from a comparison: a constant of the gradient, as in the reference)."""
        spec = self._spec_ok(spec, "spec_gate_backward")
        grad = self._spec_ok(grad, "spec_gate_backward")
        assert grad.shape == spec.shape, (grad.shape, spec.shape)
        B, C, F, N = spec.shape
        amount = self._per_item(amount, B, "amount", spec.device)
        sf, st = self._gate_smoothing(smooth_f, smooth_t)
        gs = torch.empty_like(spec)
        self._call(self.lib.b2a_spec_gate_backward_f32, _dptr(grad), _dptr(spec), B * C, F, N, _dptr(thresh),
                   thresh.shape[0], _dptr(amount), C, sf, len(smooth_f), st, len(smooth_t), _dptr(gs),
                   self._stream(spec))
        return gs

    # ------------------------------------------------------------------ loudness
    def lufs(self, x: torch.Tensor, sample_rate: float, filter_class: str = "K-weighting",
             block_size: float = 0.400, padded_length: Optional[int] = None,
             target_db: Optional[torch.Tensor] = None, want_blocks: bool = False):
        """Integrated loudness of ``x`` [B, C, T] (ref:audiotools/core/loudness.py:176-247, IIR path).

        Returns a dict: ``lufs`` [B] (unclamped), ``loud`` [B] (= max(lufs, -70)), and, when
        ``target_db`` (1 or B values) is given, ``gain`` [B] = exp((target_db - loud) ln10/20);
        ``blocks`` [B, C, nblk] when ``want_blocks``.
        """
        x = self._prep(x, "x")
        assert x.ndim == 3, "x must be [B, C, T]"
        B, C, T = x.shape
        Tp = T if padded_length is None else int(padded_length)
        sos, sgain = kweighting.design(float(sample_rate), filter_class)
        G = np.ascontiguousarray(kweighting.CHANNEL_GAINS[:C], dtype=np.float64)
        if C > len(kweighting.CHANNEL_GAINS):
            raise ValueError(f"loudness supports at most 5 channels, got {C}")
        L = self.lib
        nblk = L.b2a_lufs_num_blocks(Tp, float(sample_rate), float(block_size))
        ws_bytes = L.b2a_lufs_workspace_bytes(B, C, Tp, float(sample_rate), float(block_size))
        if nblk < 1 or ws_bytes == 0:
            raise _lib.B2AError(f"lufs: unsupported geometry (T={Tp}, rate={sample_rate}, block={block_size})")
        dev = x.device
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        lufs = torch.empty(B, dtype=torch.float32, device=dev)
        loud = torch.empty(B, dtype=torch.float32, device=dev)
        blocks = torch.empty(B, C, nblk, dtype=torch.float32, device=dev) if want_blocks else None
        gain = None
        n_target = 0
        if target_db is not None:
            target_db = self._prep(torch.as_tensor(target_db, device=dev).reshape(-1), "target_db")
            n_target = target_db.numel()
            if n_target not in (1, B):
                raise ValueError(f"target_db must have 1 or {B} entries, got {n_target}")
            gain = torch.empty(B, dtype=torch.float32, device=dev)
        dp = ctypes.POINTER(ctypes.c_double)
        self._call(L.b2a_lufs_f32, _dptr(x), B, C, T, Tp, float(sample_rate), sos.ctypes.data_as(dp),
                   sgain.ctypes.data_as(dp), sos.shape[0], float(block_size), G.ctypes.data_as(dp), _dptr(blocks),
                   _dptr(lufs), _dptr(loud), _dptr(target_db), n_target, _dptr(gain), _dptr(ws), ws_bytes,
                   self._stream(x))
        return {"lufs": lufs, "loud": loud, "gain": gain, "blocks": blocks}

    def lufs_backward(self, grad_loud: torch.Tensor, x: torch.Tensor, sample_rate: float, blocks: torch.Tensor,
                      lufs: torch.Tensor, padded_length: Optional[int] = None, gain: Optional[torch.Tensor] = None,
                      block_size: float = 0.400) -> torch.Tensor:
        """dL/dx [B, C, T] float32 of ``loud`` = max(lufs, -70) that :meth:`lufs` returned for ``x`` (times ``gain``
        [B] when given: the forward measured float32(gain x)), from that call's ``blocks`` and ``lufs`` and dL/dloud
        ``grad_loud`` [B] (``b2a_lufs_backward_f32``, DESIGN.md K21).  The gate decisions are the forward's.  Items
        clamped at -70 get zeros, items with a NaN or inf sample NaN.  K-weighting only; seven launches, no host
        sync."""
        x = self._prep(x, "x")
        assert x.ndim == 3, "x must be [B, C, T]"
        B, C, T = x.shape
        if C > len(kweighting.CHANNEL_GAINS):
            raise ValueError(f"loudness supports at most 5 channels, got {C}")
        Tp = T if padded_length is None else int(padded_length)
        g = self._prep(grad_loud.reshape(-1), "grad_loud")
        assert g.numel() == B, (g.numel(), B)
        if gain is not None:
            gain = self._prep(gain.reshape(-1), "gain")
            assert gain.numel() == B
        blocks, lufs = self._prep(blocks, "blocks"), self._prep(lufs.reshape(-1), "lufs")
        sos, sgain = kweighting.design(float(sample_rate))
        G = np.ascontiguousarray(kweighting.CHANNEL_GAINS[:C], dtype=np.float64)
        L = self.lib
        nblk = L.b2a_lufs_num_blocks(Tp, float(sample_rate), float(block_size))
        assert blocks.shape == (B, C, nblk) and lufs.numel() == B, (tuple(blocks.shape), (B, C, nblk))
        ws_bytes = int(L.b2a_lufs_backward_workspace_bytes(B, C, Tp, float(sample_rate), float(block_size)))
        if ws_bytes == 0:
            raise _lib.B2AError(f"lufs_backward: unsupported geometry (T={Tp}, rate={sample_rate}, block={block_size})")
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
        gx = torch.empty_like(x)
        dp = ctypes.POINTER(ctypes.c_double)
        self._call(L.b2a_lufs_backward_f32, _dptr(g), _dptr(x), _dptr(gain), B, C, T, Tp, float(sample_rate),
                   sos.ctypes.data_as(dp), sgain.ctypes.data_as(dp), sos.shape[0], float(block_size),
                   G.ctypes.data_as(dp), _dptr(blocks), _dptr(lufs), _dptr(gx), _dptr(ws), ws_bytes, self._stream(x))
        return gx

    LOUDNESS_STATS = ("I", "I Threshold", "LRA", "LRA Threshold", "LRA Low", "LRA High")

    def loudness_stats(self, x: torch.Tensor, sample_rate: float, padded_length: Optional[int] = None,
                       want_series: bool = False):
        """EBU R128 statistics of ``x`` [B, C, T] with the K-weighting and 0.4 s blocks of ``lufs``
        (``b2a_loudness_stats_f32``): a dict of [B] float32 tensors under the keys of ``LOUDNESS_STATS``, plus
        ``momentary`` [B, nblk] and ``short_term`` [B, n_st] (LUFS) when ``want_series``."""
        x = self._prep(x, "x")
        assert x.ndim == 3, "x must be [B, C, T]"
        B, C, T = x.shape
        Tp = T if padded_length is None else int(padded_length)
        if C > len(kweighting.CHANNEL_GAINS):
            raise ValueError(f"loudness supports at most 5 channels, got {C}")
        sos, sgain = kweighting.design(float(sample_rate))
        G = np.ascontiguousarray(kweighting.CHANNEL_GAINS[:C], dtype=np.float64)
        L = self.lib
        nblk = L.b2a_lufs_num_blocks(Tp, float(sample_rate), 0.4)
        n_st = L.b2a_loudness_stats_num_short_term(Tp, float(sample_rate))
        ws_bytes = L.b2a_loudness_stats_workspace_bytes(B, C, Tp, float(sample_rate))
        if nblk < 1 or n_st < 0 or ws_bytes == 0:
            raise _lib.B2AError(f"loudness_stats: unsupported geometry (T={Tp}, rate={sample_rate})")
        dev = x.device
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        stats = torch.empty(B, 6, dtype=torch.float32, device=dev)
        mom = torch.empty(B, nblk, dtype=torch.float32, device=dev) if want_series else None
        st = torch.empty(B, n_st, dtype=torch.float32, device=dev) if want_series else None
        dp = ctypes.POINTER(ctypes.c_double)
        self._call(L.b2a_loudness_stats_f32, _dptr(x), B, C, T, Tp, float(sample_rate), sos.ctypes.data_as(dp),
                   sgain.ctypes.data_as(dp), sos.shape[0], G.ctypes.data_as(dp), _dptr(stats), _dptr(mom), _dptr(st),
                   _dptr(ws), ws_bytes, self._stream(x))
        out = dict(zip(self.LOUDNESS_STATS, stats.unbind(1)))
        if want_series:
            out["momentary"], out["short_term"] = mom, st
        return out

    def _true_peak_factor(self, sample_rate: float) -> int:
        """The oversampling factor of ``true_peak`` at this rate (``b2a_true_peak_factor``); raises for a bad rate."""
        L = self.lib.b2a_true_peak_factor(float(sample_rate))
        self.lib.check(min(L, 0))
        return L

    def true_peak_taps(self, sample_rate: float) -> np.ndarray:
        """The float32 taps ``true_peak`` interpolates with at this rate: [L - 1, 12] (phase p = 1 .. L-1, tap
        d = -6 .. 5), empty for L = 1 (``b2a_true_peak_taps``)."""
        L = self._true_peak_factor(sample_rate)
        taps = np.zeros((L - 1, 12), dtype=np.float32)
        self.lib.check(self.lib.b2a_true_peak_taps(L, taps.ctypes.data_as(ctypes.c_void_p)))
        return taps

    def true_peak(self, x: torch.Tensor, sample_rate: float):
        """True-peak level of ``x`` [B, C, T] (``b2a_true_peak_f32``): ``rows`` [B, C], the linear peak of every row
        oversampled by 4 (below 96 kHz), 2 (below 192 kHz) or 1, and ``db`` [B], 20 log10 of each item's channel
        maximum in dBTP (-inf for silence).  float32 on x's device."""
        x = self._prep(x, "x")
        assert x.ndim == 3, "x must be [B, C, T]"
        B, C, T = x.shape
        L = self._true_peak_factor(sample_rate)
        rows = torch.empty(B, C, dtype=torch.float32, device=x.device)
        db = torch.empty(B, dtype=torch.float32, device=x.device)
        self._call(self.lib.b2a_true_peak_f32, _dptr(x), B, C, T, L, _dptr(rows), _dptr(db), self._stream(x))
        return {"rows": rows, "db": db}

    LIMITER_MAX_LOOKAHEAD = 1024  # samples (csrc/limiter.cu)

    def limiter_params(self, sample_rate: float, ceiling_db, lookahead: float, release: float, B: int, device):
        """What ``limit`` hands to ``b2a_limiter_f32``: the oversampling factor, the linear ceiling [B] (float32 on
        ``device``; a Python number is filled in without a host copy), the look-ahead in samples and the float32
        release coefficient exp(-1 / (release * rate))."""
        L = self._true_peak_factor(sample_rate)
        A = int(round(float(lookahead) * float(sample_rate)))
        if not 0 <= A <= self.LIMITER_MAX_LOOKAHEAD:
            raise ValueError(f"limit: a lookahead of {lookahead} s is {A} samples at {sample_rate} Hz; "
                             f"0 .. {self.LIMITER_MAX_LOOKAHEAD} are supported")
        if not float(release) > 0:
            raise ValueError(f"limit: release must be positive, got {release}")
        a = float(np.float32(np.exp(-1.0 / (float(release) * float(sample_rate)))))
        if isinstance(ceiling_db, (int, float)):
            ceiling = torch.full((B,), float(np.float32(10.0 ** (float(ceiling_db) / 20.0))), dtype=torch.float32,
                                 device=device)
        else:
            db = self._per_item(ceiling_db, B, "ceiling_db", device)
            ceiling = torch.exp(db * float(np.float32(np.log(10) / 20)))
        return L, ceiling, A, a

    def limit(self, x: torch.Tensor, sample_rate: float, ceiling_db, lookahead: float = 0.0015, release: float = 0.05,
              gain: Optional[torch.Tensor] = None, want_reduction: bool = False, out: Optional[torch.Tensor] = None):
        """Look-ahead true-peak limiter of ``x`` [B, C, T] (``b2a_limiter_f32``, DESIGN.md K18): every item is
        multiplied by one gain series ``1 - r[n]`` that keeps the true-peak envelope of ``true_peak``'s interpolator
        at or under ``ceiling_db`` (dBTP, a number or 1 / B values) and is exactly 1 away from the overs.
        ``lookahead`` (s) is both the hold and the length of the box attack, ``release`` (s) the time constant of the
        exponential release.  ``gain`` [B]: the item is ``float32(gain * x)`` (a deferred normalisation gain needs no
        pass of its own).  ``out`` may be ``x``.  Returns the limited signal, or ``(signal, r [B, T])`` with
        ``want_reduction``."""
        x = self._prep(x, "x")
        assert x.ndim == 3, "x must be [B, C, T]"
        B, C, T = x.shape
        L, ceiling, A, a = self.limiter_params(sample_rate, ceiling_db, lookahead, release, B, x.device)
        if gain is not None:
            gain = self._prep(gain.reshape(-1), "gain")
            assert gain.numel() == B
        if out is None:
            out = torch.empty_like(x)
        assert out.shape == x.shape and out.dtype == torch.float32 and out.is_contiguous() and out.device == x.device
        ws_bytes = int(self.lib.b2a_limiter_workspace_bytes(B, C, T))
        if ws_bytes == 0:
            raise _lib.B2AError(f"limit: unsupported shape {tuple(x.shape)}")
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
        red = torch.empty(B, T, dtype=torch.float32, device=x.device) if want_reduction else None
        self._call(self.lib.b2a_limiter_f32, _dptr(x), _dptr(gain), B, C, T, L, _dptr(ceiling), A, a, _dptr(out),
                   _dptr(red), _dptr(ws), self._stream(x))
        return (out, red) if want_reduction else out

    SOS_MAX_SECTIONS = 8  # csrc/iir.cu

    def sos_coefficients(self, sos, B: int, device) -> torch.Tensor:
        """``sos`` ([S, 6] or [1 or B, S, 6], rows b0 b1 b2 a0 a1 a2) as the kernels take it: every row divided by
        its a0 in float64 and rounded to float32 once, [1 or B, S, 6] contiguous on ``device``."""
        sos = torch.as_tensor(sos)
        self._refuse_grad(sos, "sos")
        if sos.ndim == 2:
            sos = sos.unsqueeze(0)
        if sos.ndim != 3 or sos.shape[-1] != 6 or sos.shape[0] not in (1, B):
            raise ValueError(f"sos_filter: sos must be [S, 6] or [1 or {B}, S, 6], got {tuple(sos.shape)}")
        if not 1 <= sos.shape[1] <= self.SOS_MAX_SECTIONS:
            raise ValueError(f"sos_filter: {sos.shape[1]} sections; 1 .. {self.SOS_MAX_SECTIONS} are supported")
        sos = sos.to(device=device, dtype=torch.float64, non_blocking=True)
        return (sos / sos[..., 3:4]).to(torch.float32).contiguous()

    def sos_filter(self, x: torch.Tensor, sos, gain: Optional[torch.Tensor] = None, reverse: bool = False,
                   out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``scipy.signal.sosfilt(sos, x)`` with zero initial state for x [B, C, T] (``b2a_sos_filter_f32``, DESIGN.md
        K19): ``sos`` [S, 6] for the whole batch or [B, S, 6] per item, 1 <= S <= 8, normalised by a0 and rounded to
        float32 (``sos_coefficients``).  ``gain`` [B]: the item is ``float32(gain * x)``.  ``reverse`` runs every row
        back to front (the adjoint).  An item with a section whose poles are not strictly inside the unit circle comes
        back all NaN.  ``out`` may be ``x``.  Three launches."""
        x = self._prep(x, "x")
        assert x.ndim == 3, "x must be [B, C, T]"
        B, C, T = x.shape
        sos = self.sos_coefficients(sos, B, x.device)
        if gain is not None:
            gain = self._prep(gain.reshape(-1), "gain")
            assert gain.numel() == B
        if out is None:
            out = torch.empty_like(x)
        assert out.shape == x.shape and out.dtype == torch.float32 and out.is_contiguous() and out.device == x.device
        S = sos.shape[1]
        ws_bytes = int(self.lib.b2a_sos_filter_workspace_bytes(B, C, T, S))
        if ws_bytes == 0:
            raise _lib.B2AError(f"sos_filter: unsupported shape {tuple(x.shape)}")
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
        self._call(self.lib.b2a_sos_filter_f32, _dptr(x), _dptr(gain), B, C, T, _dptr(sos), sos.shape[0], S,
                   int(bool(reverse)), _dptr(out), _dptr(ws), self._stream(x))
        return out

    def _sos_args(self, x, sos, gain, out, name):
        """The shared marshalling of the stateful and zero-phase cascades: x [B, C, T], sos as the kernels take it,
        the gain [B] or None, out."""
        x = self._prep(x, name)
        if x.ndim != 3:
            raise ValueError(f"{name}: x must be [B, C, T], got {tuple(x.shape)}")
        B = x.shape[0]
        sos = self.sos_coefficients(sos, B, x.device)
        if gain is not None:
            gain = self._prep(gain.reshape(-1), "gain")
            assert gain.numel() == B
        if out is None:
            out = torch.empty_like(x)
        assert out.shape == x.shape and out.dtype == torch.float32 and out.is_contiguous() and out.device == x.device
        return x, sos, gain, out

    def sos_filter_zi(self, x: torch.Tensor, sos, zi, gain: Optional[torch.Tensor] = None,
                      out: Optional[torch.Tensor] = None):
        """``scipy.signal.sosfilt(sos, x, zi=zi)`` for x [B, C, T] (``b2a_sos_filter_zi_f32``, DESIGN.md K19) ->
        (y float32, zf float64 [S, B, C, 2]).  ``zi`` is scipy's layout for this x, [S, B, C, 2], float64 or float32;
        the state stays in double, so ``zf`` chained into the next segment's ``zi`` gives one pass over the whole row.
        ``sos`` and ``gain`` as in ``sos_filter``.  Three launches, no host sync."""
        x, sos, gain, out = self._sos_args(x, sos, gain, out, "x")
        B, C, T = x.shape
        S = sos.shape[1]
        zi = torch.as_tensor(zi)
        self._refuse_grad(zi, "zi")
        if tuple(zi.shape) != (S, B, C, 2):
            raise ValueError(f"sosfilt: zi must be [{S}, {B}, {C}, 2] for x {tuple(x.shape)}, got {tuple(zi.shape)}")
        zi = zi.to(device=x.device, dtype=torch.float64).contiguous()
        zf = torch.empty(S, B, C, 2, dtype=torch.float64, device=x.device)
        ws_bytes = int(self.lib.b2a_sos_filter_workspace_bytes(B, C, T, S))
        if ws_bytes == 0:
            raise _lib.B2AError(f"sosfilt: unsupported shape {tuple(x.shape)}")
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
        self._call(self.lib.b2a_sos_filter_zi_f32, _dptr(x), _dptr(gain), B, C, T, _dptr(sos), sos.shape[0], S,
                   _dptr(zi), _dptr(out), _dptr(zf), _dptr(ws), self._stream(x))
        return out, zf

    SOS_PADTYPES = {None: 0, "odd": 1, "even": 2, "constant": 3}  # b2a_sos_filtfilt_f32

    def _filtfilt_args(self, x, sos, padtype, padlen, gain, out, name):
        if padtype not in self.SOS_PADTYPES:
            raise ValueError(f"sosfiltfilt: padtype must be 'odd', 'even', 'constant' or None, got {padtype!r}")
        if padlen is not None and int(padlen) < 0:
            raise ValueError(f"sosfiltfilt: padlen must be >= 0, got {padlen}")
        x, sos, gain, out = self._sos_args(x, sos, gain, out, name)
        B, C, T = x.shape
        S = sos.shape[1]
        pt = self.SOS_PADTYPES[padtype]
        pl = -1 if padlen is None else int(padlen)
        # the default is checked at its largest, 3 (2S + 1): the per-item value lives on the device
        edge = 0 if padtype is None else (3 * (2 * S + 1) if pl < 0 else pl)
        if T <= edge:
            raise ValueError(f"sosfiltfilt: the length of the input ({T}) must be greater than the padding ({edge})"
                             + (", the largest default for these sections" if pl < 0 else ""))
        ws_bytes = int(self.lib.b2a_sos_filtfilt_workspace_bytes(B, C, T, S, pt, pl))
        if ws_bytes == 0:
            raise _lib.B2AError(f"sosfiltfilt: unsupported shape {tuple(x.shape)}")
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
        return x, sos, gain, out, pt, pl, ws

    def sos_filtfilt(self, x: torch.Tensor, sos, padtype="odd", padlen: Optional[int] = None,
                     gain: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``scipy.signal.sosfiltfilt(sos, x, padtype=padtype, padlen=padlen)`` (method "pad") for x [B, C, T]
        (``b2a_sos_filtfilt_f32``, DESIGN.md K19).  ``padlen=None`` is scipy's default for each item's sections,
        3 (2S + 1 - min(#{b2 = 0}, #{a2 = 0})); T must exceed the padding, checked against 3 (2S + 1) for the default
        so that nothing is read back (this refuses rows of at most 51 samples that scipy would take).  ``sos`` and
        ``gain`` as in ``sos_filter``.  Six launches, no host sync."""
        x, sos, gain, out, pt, pl, ws = self._filtfilt_args(x, sos, padtype, padlen, gain, out, "x")
        B, C, T = x.shape
        self._call(self.lib.b2a_sos_filtfilt_f32, _dptr(x), _dptr(gain), B, C, T, _dptr(sos), sos.shape[0],
                   sos.shape[1], pt, pl, _dptr(out), _dptr(ws), self._stream(x))
        return out

    def sos_filtfilt_backward(self, grad_y: torch.Tensor, sos, padtype="odd", padlen: Optional[int] = None,
                              gain: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The gradient of ``sos_filtfilt`` with respect to x for the upstream gradient ``grad_y`` [B, C, T]
        (``b2a_sos_filtfilt_backward_f32``).  Seven launches, no host sync."""
        g, sos, gain, gx, pt, pl, ws = self._filtfilt_args(grad_y, sos, padtype, padlen, gain, None, "grad_y")
        B, C, T = g.shape
        self._call(self.lib.b2a_sos_filtfilt_backward_f32, _dptr(g), _dptr(gain), B, C, T, _dptr(sos), sos.shape[0],
                   sos.shape[1], pt, pl, _dptr(gx), _dptr(ws), self._stream(g))
        return gx

    def _rir_high_pass(self, out: torch.Tensor, sample_rate: float) -> torch.Tensor:
        """Allen & Berkley's 100 Hz high-pass, one second-order section, in place (three launches)."""
        w = 2 * math.pi * 100.0 / sample_rate
        r = math.exp(-w)
        return self.sos_filter(out, [[1.0, -(1.0 + r), r, 1.0, -2.0 * r * math.cos(w), r * r]], out=out)

    def rir_bands_kept(self, n_bands: int, sample_rate: float) -> int:
        """The octave bands of ``image_source_ir`` that are computed: those whose lower crossover 125 2^(k - 1/2) Hz is
        below sample_rate / 2 (``b2a_rir_bands_kept``)."""
        kept = self.lib.b2a_rir_bands_kept(int(n_bands), float(sample_rate))
        if kept < 1:
            raise ValueError(f"image_source_ir: bands = {n_bands}; 1 .. {_room.MAX_BANDS} are supported")
        return kept

    def octave_crossovers(self, sample_rate: float, n_bands: int, device):
        """(taps [n_bands - 1, 2 half + 1] float32 convolution taps, half) of the zero-phase windowed-sinc low-passes
        at the octave crossovers 125 2^(k + 1/2) Hz, k < n_bands - 1 (``_lowpass_bank``, julius arithmetic), all with
        the half-length julius.SplitBands(zeros=8) gives its lowest cutoff: int(8 / (e_0 / fs) / 2).  Designed once per
        (rate, band count, device) and cached, so the response path does no tensor arithmetic after the first call."""
        key = (float(sample_rate), int(n_bands), torch.device(device))
        hit = self._crossovers.get(key)
        if hit is None:
            import numpy as _np

            c = 125.0 * 2.0 ** (_np.arange(n_bands - 1) + 0.5) / float(sample_rate)
            half = int(8 / c[0] / 2)
            lp = self._lowpass_bank(torch.from_numpy(c).float(), torch.full((len(c),), half, dtype=torch.int64),
                                    device)
            hit = self._crossovers[key] = (torch.flip(lp, dims=[1]).contiguous(), half)
        return hit

    def image_source_ir(self, room: torch.Tensor, src: torch.Tensor, mics: torch.Tensor, beta: torch.Tensor,
                        length: int, sample_rate: float, sound_speed: float = 343.0, max_order: int = -1,
                        high_pass: bool = True, air: Optional[torch.Tensor] = None,
                        diffuse_after: Optional[torch.Tensor] = None,
                        seed: Optional[torch.Tensor] = None, mic_dir: Optional[torch.Tensor] = None,
                        src_dir: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Shoebox-room impulse responses by the image-source method (``b2a_rir_directional_f32``, DESIGN.md K20) -> [B, C, length]
        float32.  room [B, 3], src [B, 3], mics [B, C, 3] (metres), beta [B, 6, K] per wall and octave band (K = 1: a
        frequency-flat room) and ``air`` [B, K] dB/m or None are float64 tensors on the device, already checked
        (``core.room.image_source_ir``).  ``high_pass`` applies Allen & Berkley's 100 Hz high-pass as one second-order
        section through ``sos_filter`` (three launches).  No host sync.

        ``diffuse_after`` (float64 [B], seconds > 0) with ``seed`` (int64 [B], >= 0) keeps the images arriving before
        ceil(diffuse_after sample_rate) only and adds a diffuse tail after them; ``max_order`` must be -1 then.  One
        launch, two with the tail.

        ``mic_dir`` (float64 [B, C, 4]) and ``src_dir`` (float64 [B, 4]) give the microphones and the sources
        first-order patterns (p, v_x, v_y, v_z), p in [0, 1] and v a unit vector, already checked; None is
        omnidirectional (DESIGN.md K20 "Directivity").  They add no launch and no host sync.

        ``b2a_rir_directional_f32`` writes the K' kept bands' differences r_k - r_{k+1} and the last band r_{K'-1}; when K' > 1 the
        differences go through the zero-phase crossovers LP_k (``fftconv``, zero padding) and ``b2a_rir_band_sum_f32``
        adds them to the last band: y = r_{K'-1} + sum_k LP_k * (r_k - r_{k+1}), exactly 0 before the first sample the
        direct path (or the tail) reaches through the crossovers."""
        if mics.ndim != 3 or mics.shape[-1] != 3:
            raise ValueError(f"image_source_ir: mics must be [B, C, 3], got {tuple(mics.shape)}")
        B, C = mics.shape[:2]
        K = beta.shape[-1] if beta.ndim == 3 else 0
        if (tuple(room.shape) != (B, 3) or tuple(src.shape) != (B, 3) or tuple(beta.shape) != (B, 6, K)
                or (air is not None and tuple(air.shape) != (B, K))):
            raise ValueError(f"image_source_ir: room / source / beta / air must be [{B}, 3] / [{B}, 3] / [{B}, 6, K] "
                             f"/ [{B}, K], got {tuple(room.shape)} / {tuple(src.shape)} / {tuple(beta.shape)} / "
                             f"{None if air is None else tuple(air.shape)}")
        kept = 1 if K == 1 else self.rir_bands_kept(K, sample_rate)
        if B * C * K > _room.MAX_ROWS:
            raise ValueError(f"image_source_ir: {B * C * K} rows (items x microphones{' x bands' if K > 1 else ''}); "
                             f"at most {_room.MAX_ROWS}")
        if (diffuse_after is None) != (seed is None):
            raise ValueError("image_source_ir: diffuse_after and seed go together")
        if diffuse_after is not None:
            if max_order != -1:
                raise ValueError(f"image_source_ir: max_order = {max_order} with a diffuse tail; the tail has every "
                                 "order")
            if tuple(diffuse_after.shape) != (B,) or tuple(seed.shape) != (B,):
                raise ValueError(f"image_source_ir: diffuse_after and seed must be [{B}]")
        if mic_dir is not None and tuple(mic_dir.shape) != (B, C, 4):
            raise ValueError(f"image_source_ir: mic_dir must be [{B}, {C}, 4], got {tuple(mic_dir.shape)}")
        if src_dir is not None and tuple(src_dir.shape) != (B, 4):
            raise ValueError(f"image_source_ir: src_dir must be [{B}, 4], got {tuple(src_dir.shape)}")
        room, src, mics, beta = (self._prep(t, n, torch.float64) for t, n in
                                 ((room, "room"), (src, "source"), (mics, "mics"), (beta, "beta")))
        air = None if air is None else self._prep(air, "air", torch.float64)
        td = None if diffuse_after is None else self._prep(diffuse_after, "diffuse_after", torch.float64)
        sd = None if seed is None else self._prep(seed, "seed", torch.int64)
        md = None if mic_dir is None else self._prep(mic_dir, "mic_dir", torch.float64)
        sdir = None if src_dir is None else self._prep(src_dir, "src_dir", torch.float64)
        L = int(length)
        bands = torch.empty(kept, B, C, L, dtype=torch.float32, device=room.device)
        self._call(self.lib.b2a_rir_directional_f32, _dptr(room), _dptr(src), _dptr(mics), _dptr(beta), _dptr(air),
                   _dptr(td), _dptr(sd), _dptr(md), _dptr(sdir), B, C, K, L, float(sample_rate), float(sound_speed),
                   int(max_order), _dptr(bands), self._stream(room))
        if kept == 1:
            out = bands[0]
        else:
            taps, half = self.octave_crossovers(sample_rate, kept, room.device)
            conv = self.fftconv(bands[:kept - 1], taps, rows_per_filt=B * C, offset0=half, pad_mode="constant")
            out = torch.empty(B, C, L, dtype=torch.float32, device=room.device)
            self._call(self.lib.b2a_rir_band_sum_f32, _dptr(src), _dptr(mics), _dptr(td), B, C, L, float(sample_rate),
                       float(sound_speed), half, _dptr(bands), _dptr(conv), kept - 1, _dptr(out), self._stream(room))
        return self._rir_high_pass(out, sample_rate) if high_pass else out

    def gain(self, x: torch.Tensor, gain: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``x[b] * gain[b]`` (ref:audiotools/core/effects.py:219,237)."""
        x = self._prep(x, "x")
        B = x.shape[0]
        gain = self._prep(gain.reshape(-1), "gain")
        assert gain.numel() == B
        if out is None:
            out = torch.empty_like(x)
        self._call(self.lib.b2a_gain_f32, _dptr(x), _dptr(out), B, x.numel() // B, _dptr(gain), self._stream(x))
        return out

    # ------------------------------------------------------------------ collate (csrc/collate.cu)
    def pack_rows(self, items, T_out: int, offsets=None) -> torch.Tensor:
        """Ragged ``items`` (tensors [C, T_i] or [b_i, C, T_i], float32, one device, same C) -> one zero-padded /
        truncated batch [sum b_i, C, T_out] in ONE launch (ref:audiotools/core/audio_signal.py:380-470).
        ``offsets`` (one int per item): the window starts at that sample of the item (negative / past-the-end
        samples read as zero) -- the excerpt gather of ``salient_excerpt``."""
        views, C = [], None
        for k, t in enumerate(items):
            t = self._prep(t, "item")
            t3 = t if t.ndim == 3 else t.reshape(1, *t.shape[-2:])
            C = t3.shape[1] if C is None else C
            assert t3.shape[1] == C, "pack_rows: items must have the same number of channels"
            off = 0 if offsets is None else int(offsets[k])
            for b in range(t3.shape[0]):
                views.append((t3[b], off))
        dev = views[0][0].device
        n = len(views)
        table = torch.tensor([[v.data_ptr(), v.shape[-1], v.stride(0) if v.shape[0] > 1 else v.shape[-1], o]
                              for v, o in views], dtype=torch.int64).t().contiguous()
        table = table.to(dev, non_blocking=True)  # [4, n]: pointers, lengths, row strides, offsets
        out = torch.empty(n, C, int(T_out), dtype=torch.float32, device=dev)
        self._call(self.lib.b2a_pack_rows_f32, _dptr(table[0]), _dptr(table[1]), _dptr(table[2]), _dptr(table[3]), n,
                   int(C), int(T_out), _dptr(out), self._stream(out))
        out._b2a_keepalive = [v for v, _ in views]  # the sources must outlive the (asynchronous) gather
        return out

    # ------------------------------------------------------------------ element-wise / peak effects (csrc/effects.cu)
    def row_absmax(self, x: torch.Tensor) -> torch.Tensor:
        """``x.abs().max(dim=-1, keepdim=True)`` for x [..., T] (ref:audiotools/core/effects.py:155,176,194)."""
        x = self._prep(x, "x")
        T = x.shape[-1]
        rows = x.numel() // T
        peak = torch.empty(*x.shape[:-1], 1, dtype=torch.float32, device=x.device)
        self._call(self.lib.b2a_row_absmax_f32, _dptr(x), rows, T, _dptr(peak), self._stream(x))
        return peak

    def limit_peak(self, x: torch.Tensor, max_abs: float = 1.0, peak: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``ensure_max_of_audio`` (ref :181-198): rows whose peak exceeds ``max_abs`` are scaled by max_abs / peak."""
        x = self._prep(x, "x")
        T = x.shape[-1]
        rows = x.numel() // T
        if peak is None:
            peak = self.row_absmax(x)
        out = torch.empty_like(x)
        self._call(self.lib.b2a_limit_peak_f32, _dptr(x), _dptr(out), rows, T, _dptr(peak), float(max_abs),
                   self._stream(x))
        return out

    def peak_scale_backward(self, grad_out: torch.Tensor, y: torch.Tensor, x_ref: Optional[torch.Tensor] = None,
                            max_abs: float = 1.0, bypass: Optional[torch.Tensor] = None):
        """Gradients of the per-row peak rescales: :meth:`limit_peak` (``x_ref`` None) -> (dL/dy, None), or apply_ir's
        restore ``y * clamp(max|x_ref|, 1e-8) / clamp(max|y|, 1e-8)`` -> (dL/dy, dL/dx_ref).  ``bypass`` [B]: items whose
        scale was 1 (restore only)."""
        g = self._prep(grad_out, "grad_out")
        y = self._prep(y, "y")
        assert g.shape == y.shape
        T = y.shape[-1]
        rows = y.numel() // T
        gx = None
        if x_ref is not None:
            x_ref = self._prep(x_ref, "x_ref")
            assert x_ref.shape == y.shape
            gx = torch.empty_like(y)
        if bypass is not None:
            bypass = torch.as_tensor(bypass).reshape(-1).to(y.device)
            bypass = self._bypass(bypass.repeat_interleave(rows // bypass.numel()), rows, y.device)
        gy = torch.empty_like(y)
        self._call(self.lib.b2a_peak_scale_backward_f32, _dptr(g), _dptr(y), _dptr(x_ref), rows, T, float(max_abs),
                   _dptr(bypass), _dptr(gy), _dptr(gx), self._stream(y))
        return gy, gx

    def mix(self, x: torch.Tensor, other: torch.Tensor, other_gain: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``x + other_gain[item] * other`` (ref :27-64: the noise's normalize() multiply and the add, one pass)."""
        x = self._prep(x, "x")
        other = self._prep(other, "other")
        assert other.shape == x.shape, (other.shape, x.shape)
        B = x.shape[0]
        if other_gain is not None:
            other_gain = self._prep(other_gain.reshape(-1), "other_gain")
            assert other_gain.numel() == B
        out = torch.empty_like(x)
        self._call(self.lib.b2a_mix_f32, _dptr(x), _dptr(other), _dptr(other_gain), _dptr(out), B, x.numel() // B,
                   self._stream(x))
        return out

    def quantize(self, x: torch.Tensor, channels: torch.Tensor, mulaw: bool = False) -> torch.Tensor:
        """Linear (ref :463-491) or mu-law (ref :493-523) quantisation to ``channels`` (1 or B values) levels."""
        x = self._prep(x, "x")
        B = x.shape[0]
        channels = self._per_item(channels, B, "channels", x.device)
        out = torch.empty_like(x)
        self._call(self.lib.b2a_quantize_f32, _dptr(x), _dptr(out), B, x.numel() // B, _dptr(channels), int(mulaw),
                   self._stream(x))
        return out

    def order_stats(self, row: torch.Tensor, k: torch.Tensor) -> torch.Tensor:
        """The ``k[i]``-th smallest values (0-based) of a 1-D float32 tensor, exactly (radix selection, no sort)."""
        row = self._prep(row.reshape(-1), "row")
        k = k.to(row.device).reshape(-1).to(torch.int64).contiguous()
        out = torch.empty(k.numel(), dtype=torch.float32, device=row.device)
        self._call(self.lib.b2a_order_stats_f32, _dptr(row), row.numel(), _dptr(k), k.numel(), _dptr(out),
                   self._stream(row))
        return out

    def quantile(self, row: torch.Tensor, q: torch.Tensor) -> torch.Tensor:
        """``torch.quantile(row, q)`` (linear interpolation; aten's float32 rank arithmetic and lerp) for a 1-D row.
        A row that holds a NaN gives NaN for every q, as in aten, which moves every rank to the last one: the largest
        order statistic, computed in the same launch, is NaN exactly then."""
        n = row.numel()
        q = q.to(row.device).reshape(-1).float()
        nq = q.numel()
        ranks = q * (n - 1)
        below = ranks.floor()
        w = ranks - below
        ks = torch.cat([below.to(torch.int64), ranks.ceil().to(torch.int64),
                        torch.full((1,), n - 1, dtype=torch.int64, device=ranks.device)])
        v = self.order_stats(row, ks)
        a, b, last = v[:nq], v[nq:2 * nq], v[2 * nq:]
        out = torch.where(w < 0.5, a + w * (b - a), b - (b - a) * (1 - w))
        return torch.where(last.isnan(), last, out)

    def clamp_items(self, x: torch.Tensor, lo: torch.Tensor, hi: torch.Tensor) -> torch.Tensor:
        """``x.clamp(lo[item], hi[item])`` (ref :459)."""
        x = self._prep(x, "x")
        B = x.shape[0]
        lo = self._per_item(lo, B, "lo", x.device)
        hi = self._per_item(hi, B, "hi", x.device)
        out = torch.empty_like(x)
        self._call(self.lib.b2a_clamp_items_f32, _dptr(x), _dptr(out), B, x.numel() // B, _dptr(lo), _dptr(hi),
                   self._stream(x))
        return out

    # ------------------------------------------------------------------ STFT / mel
    def _packed_len(self, mel_lo: torch.Tensor, mel_hi: torch.Tensor, n_fft: int) -> int:
        """Floats of the shared-memory band table of csrc/spectral.cu: row m is filter m's 4-aligned band, padded
        to the widest of the (up to) 4 CONSECUTIVE filters {4g .. 4g + 3} that one warp instruction projects together
        (group g = w + 8i for warp w, step i; neighbouring filters have nearly equal widths, so the padding is small),
        rounded up to an even number of float4s (the projection loop is unrolled by two, no remainder).
        The cache entry keeps the two tensors alive, so their addresses cannot be reused by another filterbank."""
        key = (mel_lo.data_ptr(), mel_hi.data_ptr(), mel_lo.numel())
        if key not in self._packed_cache:
            lo, hi = mel_lo.cpu().numpy().astype("int64"), mel_hi.cpu().numpy().astype("int64")
            n4 = ((((hi + 3) & ~3) - (lo & ~3)) >> 2).clip(min=0)
            n, total = len(n4), 0
            for g in range(0, n, 4):
                grp = range(g, min(g + 4, n))
                total += ((int(max(n4[m] for m in grp)) + 1) & ~1) * len(grp)  # rows padded to an even width
            self._packed_cache[key] = (4 * total, mel_lo, mel_hi)
        return self._packed_cache[key][0]

    def spectral_kernel_name(self, n_fft: int, hop: int, want_mel: bool = True, want_stft: bool = False) -> str:
        """Name of the kernel ``spectral`` launches for this geometry (bench.py / profiles label their numbers with it)."""
        route = self.route(n_fft, hop, 0)
        if route in (_lib.ROUTE_LARGE, _lib.ROUTE_DENSE):
            name = f"stft_large_kernel<{int(math.log2(n_fft))}>" if route == _lib.ROUTE_LARGE else "dft_forward_kernel"
            return name + " + mel_from_stft_kernel" if want_mel else name
        if n_fft in (32, 4096):
            return f"spectral_kernel<{int(math.log2(n_fft)) - 1}>"
        mode = 2 if (want_stft and want_mel) else (1 if want_stft else 0)
        return f"spectral_warp_kernel<{int(math.log2(n_fft)) - 1},{mode}>"

    @staticmethod
    def num_frames(T: int, n_fft: int, hop: int, pad: int = 0, right_pad: int = 0, drop_edge: int = 0) -> int:
        """``b2a_stft_num_frames`` evaluated on the host (same integer formula; tests/test_abi.py checks they agree):
        a foreign-function call per ``stft()`` is measurable at batch=4 x 1 s, where the call is launch-latency bound."""
        if T < 1 or n_fft < 2 or hop < 1 or pad < 0 or right_pad < 0 or drop_edge < 0:
            return -1
        return 1 + (T + 2 * pad + right_pad - (n_fft & 1)) // hop - 2 * drop_edge

    def spectral(self, x: torch.Tensor, n_fft: int, hop: int, window: torch.Tensor, pad: int = 0,
                 right_pad: int = 0, pad_mode: str = "reflect", drop_edge: int = 0,
                 gain: Optional[torch.Tensor] = None, want_scaled: bool = False,
                 mel_fb: Optional[torch.Tensor] = None, mel_lo: Optional[torch.Tensor] = None,
                 mel_hi: Optional[torch.Tensor] = None, post: int = _lib.POST_NONE, post_eps: float = 0.0,
                 post_power: float = 1.0, want_stft: bool = True):
        """Framing -> window -> rFFT -> (|.| -> banded mel -> post) over ``x`` [B, C, T], one ``b2a_spectral_f32`` call:
        one fused launch on the FFT route, gain pass + STFT + mel launches on the LARGE / DENSE routes.

        Returns dict(stft=[B,C,F,N] complex64 | None, mel=[B,C,n_mels,N] | None, scaled=[B,C,T] | None).
        """
        x = self._prep(x, "x")
        assert x.ndim == 3
        B, C, T = x.shape
        rows = B * C
        if pad_mode not in _lib.PAD_MODES:
            raise NotImplementedError(f"padding_type {pad_mode!r} (supported: {sorted(_lib.PAD_MODES)})")
        window = self._prep(window, "window")
        assert window.numel() == n_fft
        N = self.num_frames(T, n_fft, hop, pad, right_pad, drop_edge)
        if N < 1:
            raise _lib.B2AError(f"stft: no frames (T={T}, n_fft={n_fft}, hop={hop})")
        F = n_fft // 2 + 1
        dev = x.device
        route = self.route(n_fft, hop, 0)
        if route == _lib.ROUTE_NONE:
            raise self.route_error(n_fft, hop, 0)
        fft = route == _lib.ROUTE_FFT
        stft = torch.empty(B, C, F, N, dtype=torch.complex64, device=dev) if want_stft else None
        mel = None
        n_mels = 0
        packed_len = 0
        if mel_fb is not None:
            mel_fb = self._prep(mel_fb, "mel_fb")
            n_mels = mel_fb.shape[0]
            assert mel_fb.shape[1] == F, (mel_fb.shape, F)
            mel_lo = self._prep(mel_lo, "mel_lo", torch.int32)
            mel_hi = self._prep(mel_hi, "mel_hi", torch.int32)
            mel = torch.empty(B, C, n_mels, N, dtype=torch.float32, device=dev)
            if fft:
                packed_len = self._packed_len(mel_lo, mel_hi, n_fft)
        scaled = None
        rows_per_gain = 1
        if gain is not None:
            gain = self._prep(gain.reshape(-1), "gain")
            assert gain.numel() == B
            rows_per_gain = C
            if want_scaled:
                scaled = torch.empty_like(x)
        mat = self.dft_matrix(window, int(n_fft), inverse=0) if route == _lib.ROUTE_DENSE else None
        # LARGE / DENSE: the STFT and the scaled signal go to a workspace when the caller does not keep them
        nbytes = 0 if fft else int(self.lib.b2a_spectral_workspace_bytes(
            rows, T, n_fft, hop, pad, right_pad, drop_edge, stft is None, gain is not None and scaled is None))
        ws = torch.empty((nbytes + 3) // 4, dtype=torch.float32, device=dev) if nbytes else None
        self._call(self.lib.b2a_spectral_f32, _dptr(x), rows, T, n_fft, hop, _dptr(window), _dptr(mat), pad, right_pad,
                   _lib.PAD_MODES[pad_mode], drop_edge, _dptr(gain), rows_per_gain, _dptr(scaled), _dptr(mel_fb),
                   _dptr(mel_lo), _dptr(mel_hi), n_mels, packed_len, post, float(post_eps), float(post_power),
                   _dptr(mel), _dptr(stft), _dptr(ws), nbytes, self._stream(x))
        return {"stft": stft, "mel": mel, "scaled": scaled}

    def mel_dct(self, logmel: torch.Tensor, dct: torch.Tensor) -> torch.Tensor:
        """``(logmel.transpose(-1, -2) @ dct).transpose(-1, -2)`` for logmel [B, C, n_mels, N], dct [n_mels, n_mfcc]
        (ref:audiotools/core/audio_signal.py:1420-1426) as one launch of csrc/dft.cu (no library GEMM)."""
        logmel = self._prep(logmel, "logmel")
        B, C, n_mels, N = logmel.shape
        dct = self._prep(dct.to(logmel.device), "dct")
        assert dct.shape[0] == n_mels, (dct.shape, n_mels)
        n_mfcc = dct.shape[1]
        out = torch.empty(B, C, n_mfcc, N, dtype=torch.float32, device=logmel.device)
        self._call(self.lib.b2a_mel_dct_f32, _dptr(logmel), B * C, n_mels, N, _dptr(dct), n_mfcc, _dptr(out),
                   self._stream(logmel))
        return out

    # ------------------------------------------------------------------ FIR / convolution
    def _bypass(self, bypass, n: int, device):
        """[n] int32 device flags (non-zero = leave the rows of this filter / item untouched) or None."""
        if bypass is None:
            return None
        bypass = torch.as_tensor(bypass).reshape(-1).to(device=device, dtype=torch.int32).contiguous()
        assert bypass.numel() == n, (bypass.shape, n)
        return bypass

    def fftconv(self, x: torch.Tensor, taps: torch.Tensor, rows_per_filt: int, offset: Optional[torch.Tensor] = None,
                offset0: int = 0, pad_mode: str = "replicate", post_scale: Optional[torch.Tensor] = None,
                subtract_from_input: bool = False, bypass: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``out[row, n] = post * sum_k taps[f, k] * xv[row, n - k + offset0 + offset[f]]`` with
        ``f = row // rows_per_filt`` and ``xv`` = ``x`` extended by ``pad_mode`` ("constant" zeros,
        "replicate", "circular").  x: [..., T] (leading dims are flattened to rows); taps: [n_filt, L].
        ``bypass`` [n_filt] (bool / int): rows of those filters are copied through unchanged (mask-aware transforms)."""
        x = self._prep(x, "x")
        shape = x.shape
        T = shape[-1]
        rows = x.numel() // T
        taps = self._prep(taps.to(x.device), "taps")
        assert taps.ndim == 2
        n_filt, L = taps.shape
        if offset is not None:
            offset = self._prep(offset.reshape(-1).to(x.device), "offset", torch.int32)
            assert offset.numel() == n_filt
        if post_scale is not None:
            post_scale = self._prep(post_scale.reshape(-1).to(x.device), "post_scale")
            assert post_scale.numel() == n_filt
        bypass = self._bypass(bypass, n_filt, x.device)
        mode = {"constant": 1, "replicate": 2, "circular": 3}[pad_mode]
        ws_bytes = self.lib.b2a_fftconv_workspace_bytes(rows, T, n_filt, L)
        if ws_bytes == 0:
            raise _lib.B2AError("fftconv: bad shape")
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
        out = torch.empty_like(x)
        self._call(self.lib.b2a_fftconv_f32, _dptr(x), rows, T, _dptr(taps), n_filt, L, int(rows_per_filt),
                   _dptr(offset), int(offset0), mode, _dptr(post_scale), int(bool(subtract_from_input)), _dptr(bypass),
                   _dptr(out), _dptr(ws), ws_bytes, self._stream(x))
        return out

    DIRECT_FIR_MAX_TAPS = 320  # longer filters are cheaper through the FFT engine

    def fir_direct(self, x: torch.Tensor, taps: torch.Tensor, rows_per_filt: int, left: Optional[torch.Tensor] = None,
                   left0: int = 0, stride: int = 1, out_len: Optional[int] = None, pad_mode: str = "replicate",
                   subtract_from_input: bool = False, bypass: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``out[row, m] = sum_k taps[f, k] * xv[row, m*stride + k - left0 - left[f]]`` (correlation form);
        ``bypass`` [n_filt]: rows of those filters are copied through unchanged (stride 1)."""
        x = self._prep(x, "x")
        T = x.shape[-1]
        rows = x.numel() // T
        taps = self._prep(taps.to(x.device), "taps")
        n_filt, K = taps.shape
        if left is not None:
            left = self._prep(left.reshape(-1).to(x.device), "left", torch.int32)
        out_len = T if out_len is None else int(out_len)
        bypass = self._bypass(bypass, n_filt, x.device)
        out = torch.empty(*x.shape[:-1], out_len, dtype=torch.float32, device=x.device)
        self._call(self.lib.b2a_fir_direct_f32, _dptr(x), rows, T, _dptr(taps), n_filt, K, int(rows_per_filt),
                   _dptr(left), int(left0), int(stride), out_len, {"constant": 1, "replicate": 2}[pad_mode],
                   int(bool(subtract_from_input)), _dptr(bypass), _dptr(out), self._stream(x))
        return out

    @staticmethod
    def _sinc(x: torch.Tensor) -> torch.Tensor:
        return torch.where(x == 0, torch.ones_like(x), torch.sin(x) / x)

    def _lowpass_bank(self, cutoffs: torch.Tensor, half: torch.Tensor, device) -> torch.Tensor:
        """Windowed-sinc low-pass taps (julius.LowPassFilters arithmetic, float32) for per-filter
        normalised cutoffs [n] and half sizes [n]; filter i occupies taps[i, :2*half[i]+1], rest 0."""
        n = cutoffs.numel()
        hmax = int(half.max().item())
        c = cutoffs.to(device=device, dtype=torch.float32).reshape(n, 1)
        h = half.to(device=device).reshape(n, 1)
        j = torch.arange(2 * hmax + 1, device=device).reshape(1, -1)
        valid = j <= 2 * h
        t = (j - h).to(torch.float32)
        # torch.hann_window(2*half+1, periodic=False)[j] = 0.5 - 0.5 cos(2 pi j / (2 half))
        win = 0.5 - 0.5 * torch.cos(2 * math.pi * j.to(torch.float32) / (2 * h).clamp(min=1).to(torch.float32))
        f = 2 * c * win * self._sinc(2 * c * math.pi * t)
        f = torch.where(valid & (c > 0), f, torch.zeros_like(f))
        s = f.sum(dim=1, keepdim=True)
        return torch.where(s != 0, f / s, f)

    @staticmethod
    def _reverse_rows(f: torch.Tensor, lengths: torch.Tensor) -> torch.Tensor:
        """g[i, k] = f[i, lengths[i]-1-k] for k < lengths[i] (correlation taps -> convolution taps)."""
        n, L = f.shape
        k = torch.arange(L, device=f.device).reshape(1, -1)
        idx = (lengths.to(f.device).reshape(n, 1) - 1 - k)
        g = torch.gather(f, 1, idx.clamp(min=0))
        return torch.where(idx >= 0, g, torch.zeros_like(g))

    def sinc_filter(self, x: torch.Tensor, cutoffs_hz: torch.Tensor, sample_rate: int, zeros: int = 51,
                    highpass: bool = False, bypass: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Per-item windowed-sinc low-pass (or ``x - lowpass(x)``) of x [B, C, T]
        (ref:audiotools/core/dsp.py:153-215 -> julius.LowPassFilter(cutoff / sr, zeros), replicate padding)."""
        x = self._prep(x, "x")
        B, C, T = x.shape
        from .core import util as _util

        cut = _util.host_view(torch.as_tensor(cutoffs_hz)).reshape(-1).cpu()  # host mirror (util.prepare_batch): no sync
        if cut.numel() == 1:
            cut = cut.expand(B)
        assert cut.numel() == B
        # the reference divides a [B,1] tensor by the (python int) sample rate: float32 unless the input is float64
        cn = (cut / sample_rate)
        if cn.dtype not in (torch.float32, torch.float64):
            cn = cn.float()
        if (cn < 0).any():
            raise ValueError("Minimum cutoff must be larger than zero.")
        if (cn > 0.5).any():
            raise ValueError("A cutoff above 0.5 does not make sense.")
        if (cn == 0).any():
            raise ValueError("cutoff 0: julius.LowPassFilter has no positive cutoff to size the filter from")
        if bypass is not None:
            # items the mask does not select must not size the filter bank (their cutoff may ask for the longest
            # filter and push the call from the direct kernel to the FFT engine): give them the widest selected cutoff
            bh = _util.host_view(torch.as_tensor(bypass)).reshape(-1).cpu().bool()
            if bool((~bh).any()):
                cn = torch.where(bh, cn[~bh].max(), cn)
        half = (zeros / cn / 2).to(torch.int64)  # int(zeros / cutoff / 2), in the tensor's own precision
        f = self._lowpass_bank(cn, half, x.device)
        K = f.shape[1]
        if K <= self.DIRECT_FIR_MAX_TAPS and self.lib.b2a_fir_direct_supported(T, K, 1):
            # short filters: time-domain kernel, correlation taps as designed (filter b is centred at half[b])
            return self.fir_direct(x, f, rows_per_filt=C, left=half.to(torch.int32), pad_mode="replicate",
                                   subtract_from_input=highpass, bypass=bypass)
        g = self._reverse_rows(f, 2 * half + 1)
        return self.fftconv(x, g, rows_per_filt=C, offset=half.to(torch.int32), pad_mode="replicate",
                            subtract_from_input=highpass, bypass=bypass)

    @staticmethod
    def _split_band_cutoffs(sample_rate: float, n_bands: int):
        """julius.SplitBands cutoffs: HTK-mel spaced, normalised by the sample rate (float64)."""
        import numpy as _np

        lo, hi = 2595 * math.log10(1 + 0.0 / 700), 2595 * math.log10(1 + (sample_rate / 2) / 700)
        mels = _np.linspace(lo, hi, n_bands + 1)
        hz = 700 * (10 ** (mels / 2595) - 1)
        return hz[1:-1] / sample_rate

    def _band_lowpasses(self, sample_rate: float, n_bands: int, device):
        """(lp [n_bands-1, 2*half+1] float32 correlation taps, half) of julius.SplitBands(zeros=8)."""
        c = self._split_band_cutoffs(sample_rate, n_bands)
        half = int(8 / min(c) / 2)
        cn = torch.from_numpy(c)  # float64 scalars multiply float32 tensors as python scalars in julius
        lp = self._lowpass_bank(cn.float(), torch.full((len(c),), half, dtype=torch.int64), device)
        return lp, half

    def equalizer(self, x: torch.Tensor, sample_rate: int, db: torch.Tensor,
                  bypass: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Mel-band equaliser of x [B, C, T] (ref:audiotools/core/effects.py:405-433): band weights
        10**db [B or 1, n_bands]; split + weighted sum == one FIR per item,
        h = w_last * delta + sum_k (w_k - w_{k+1}) * lowpass_k."""
        x = self._prep(x, "x")
        B, C, T = x.shape
        h, half = self._equalizer_taps(sample_rate, db, B, x.device, bypass)
        if half is None:
            return self.gain(x, h)
        g = torch.flip(h, dims=[1]).contiguous()
        return self.fftconv(x, g, rows_per_filt=C, offset0=half, pad_mode="replicate", bypass=bypass)

    def _equalizer_taps(self, sample_rate: int, db: torch.Tensor, B: int, device, bypass=None):
        """(h [B, 2*half+1] correlation taps, half) of the equaliser's per-item FIR, or (gain [B], None) for one band."""
        db = torch.as_tensor(db)
        if db.ndim == 1:
            db = db.unsqueeze(0)
        n_bands = db.shape[-1]
        w = (10 ** db).to(device).float()
        if w.shape[0] == 1:
            w = w.expand(B, n_bands)
        assert w.shape[0] == B
        if n_bands == 1:
            g1 = w[:, 0].contiguous()
            if bypass is not None:
                g1 = torch.where(torch.as_tensor(bypass).to(device).bool().reshape(-1), torch.ones_like(g1), g1)
            return g1, None
        lp, half = self._band_lowpasses(sample_rate, n_bands, device)
        # [B, n_bands-1] x [n_bands-1, 2*half+1] as a broadcast multiply-add (a few KB: not worth a library GEMM call)
        h = ((w[:, :-1] - w[:, 1:]).unsqueeze(-1) * lp.unsqueeze(0)).sum(dim=1)
        h[:, half] += w[:, -1]
        return h, half

    def equalizer_backward(self, grad_out: torch.Tensor, sample_rate: int, db: torch.Tensor,
                           bypass: Optional[torch.Tensor] = None) -> torch.Tensor:
        """dL/dx of :meth:`equalizer`: the zero-padded correlation with the reversed taps (``fftconv`` in constant mode
        with the correlation taps as convolution taps) plus the replicate edge fold (:meth:`fir_pad_fold`)."""
        g = self._prep(grad_out, "grad_out")
        B, C, T = g.shape
        h, half = self._equalizer_taps(sample_rate, db, B, g.device, bypass)
        if half is None:
            return self.gain(g, h)
        gx = self.fftconv(g, h, rows_per_filt=C, offset0=half, pad_mode="constant", bypass=bypass)
        return self.fir_pad_fold(g, h, rows_per_filt=C, left0=half, bypass=bypass, grad_x=gx)

    def fir_pad_fold(self, grad_out: torch.Tensor, taps: torch.Tensor, rows_per_filt: int,
                     left: Optional[torch.Tensor] = None, left0: int = 0, bypass: Optional[torch.Tensor] = None,
                     grad_x: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Adds to ``grad_x`` (in place) what the replicate padding of the stride-1 correlation
        ``y[m] = sum_k taps[f, k] xv[m + k - left0 - left[f]]`` carries back to the edge samples of every row."""
        g = self._prep(grad_out, "grad_out")
        T = g.shape[-1]
        rows = g.numel() // T
        taps = self._prep(taps.to(g.device), "taps")
        n_filt, K = taps.shape
        if left is not None:
            left = self._prep(left.reshape(-1).to(g.device), "left", torch.int32)
        bypass = self._bypass(bypass, n_filt, g.device)
        assert grad_x is not None and grad_x.shape == g.shape and grad_x.is_contiguous()
        ws_bytes = self.lib.b2a_fir_pad_fold_workspace_bytes(n_filt, K)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=g.device)
        self._call(self.lib.b2a_fir_pad_fold_f32, _dptr(g), rows, T, _dptr(taps), n_filt, K, int(rows_per_filt),
                   _dptr(left), int(left0), _dptr(bypass), _dptr(grad_x), _dptr(ws), ws_bytes, self._stream(g))
        return grad_x

    def mel_filterbank(self, x: torch.Tensor, sample_rate: int, n_bands: int) -> torch.Tensor:
        """julius.SplitBands(sample_rate, n_bands)(x).permute(1, 2, 3, 0) -> [B, C, T, n_bands]
        (ref:audiotools/core/effects.py:386-403)."""
        x = self._prep(x, "x")
        B, C, T = x.shape
        if n_bands == 1:
            return x.unsqueeze(-1).clone()
        lp, half = self._band_lowpasses(sample_rate, n_bands, x.device)
        h = torch.zeros(n_bands, 2 * half + 1, device=x.device)
        h[0] = lp[0]
        h[1:-1] = lp[1:] - lp[:-1]
        h[-1] = -lp[-1]
        h[-1, half] += 1.0
        g = torch.flip(h, dims=[1]).contiguous()
        bands = [self.fftconv(x, g[k:k + 1], rows_per_filt=B * C, offset0=half, pad_mode="replicate")
                 for k in range(n_bands)]
        return torch.stack(bands, dim=-1)

    def circular_convolve(self, x: torch.Tensor, ir: torch.Tensor, roll_to_peak: bool = True,
                          bypass: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``EffectMixin.convolve`` (ref:audiotools/core/effects.py:66-123): circular convolution with period T,
        the IR rolled to its peak, scaled by 1/max(max|ir|, 1e-5).  x: [B, C, T]; ir: [B or 1, 1 or C, L] (a batch-1
        impulse response is shared by all items, as the reference's broadcasting product does).  ``bypass`` [B]:
        items left untouched."""
        x = self._prep(x, "x")
        B, C, T = x.shape
        ir, n_ir, L, rows_per_ir, bypass = self._circconv_filters(x.shape, ir, bypass, x.device)
        ws_bytes = self.lib.b2a_circconv_workspace_bytes(B * C, T, n_ir, L)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
        out = torch.empty_like(x)
        self._call(self.lib.b2a_circconv_f32, _dptr(x), B * C, T, _dptr(ir), n_ir, L, rows_per_ir,
                   int(bool(roll_to_peak)), _dptr(bypass), _dptr(out), _dptr(ws), ws_bytes, self._stream(x))
        return out

    def _circconv_filters(self, shape, ir: torch.Tensor, bypass, device):
        """The IR bank of :meth:`circular_convolve` for x of ``shape`` [B, C, T]: (ir [n_ir, L] truncated to T, n_ir, L,
        rows_per_ir, bypass [n_ir] or None)."""
        B, C, T = shape
        ir = self._prep(ir, "ir")
        assert ir.ndim == 3 and ir.shape[0] in (1, B) and ir.shape[1] in (1, C), ir.shape
        if ir.shape[0] == 1 and B > 1 and (ir.shape[1] != 1 or bypass is not None):
            ir = ir.expand(B, -1, -1).contiguous()  # per-channel / per-item flags need one filter per item
        if ir.shape[-1] > T:
            ir = ir[..., :T].contiguous()
        L = ir.shape[-1]
        n_ir = ir.shape[0] * ir.shape[1]
        rows_per_ir = (B * C if ir.shape[0] == 1 else C) if ir.shape[1] == 1 else 1
        if bypass is not None:
            bypass = torch.as_tensor(bypass).reshape(-1).to(device)
            if ir.shape[1] != 1:
                bypass = bypass.repeat_interleave(C)
            bypass = self._bypass(bypass, n_ir, device)
        return ir, n_ir, L, rows_per_ir, bypass

    MOVING_IR_MIN_HOP = 1024  # csrc/fftconv.cu's block: with a shorter hop a block would meet more than 3 waypoints

    def circular_convolve_moving(self, x: torch.Tensor, irs: torch.Tensor, hop: int, roll_to_peak: bool = True,
                                 bypass: Optional[torch.Tensor] = None) -> torch.Tensor:
        """:meth:`circular_convolve` along a path of K impulse responses (DESIGN.md K22): waypoint k sits at sample
        k hop, and the output crossfades the K static convolutions linearly between neighbouring waypoints,
        y = sum_k v_k(t) (h_k (*) x)(t), the last waypoint holding from its sample on.  Every waypoint of a row takes
        the roll and scale of the row's first waypoint.  x: [B, C, T]; irs: [B, K, C or 1, L] (1: shared by the
        channels), truncated to T; ``hop`` >= 1024 samples and K = (T - 1) // hop + 1.  ``bypass`` [B]: items left
        untouched."""
        x = self._prep(x, "x")
        irs = self._prep(irs, "irs")
        B, C, T = x.shape
        if isinstance(hop, bool) or not isinstance(hop, (int, np.integer)):
            raise ValueError(f"circular_convolve_moving: hop = {hop!r}; an int number of samples")
        hop = int(hop)
        if irs.ndim != 4 or irs.shape[0] != B or irs.shape[2] not in (1, C) or irs.shape[3] < 1:
            raise ValueError(f"circular_convolve_moving: irs must be [{B}, K, {C} or 1, L] for x {tuple(x.shape)}, "
                             f"got {tuple(irs.shape)}")
        if hop < self.MOVING_IR_MIN_HOP:
            raise ValueError(f"circular_convolve_moving: hop = {hop} samples; at least {self.MOVING_IR_MIN_HOP}")
        K = irs.shape[1]
        if K != (T - 1) // hop + 1:
            raise ValueError(f"circular_convolve_moving: {K} waypoints every {hop} samples for T = {T}; the path "
                             f"must cover the signal exactly, (T - 1) // hop + 1 = {(T - 1) // hop + 1} waypoints")
        n_ch = irs.shape[2]
        irs = irs[..., :T].contiguous()
        L = irs.shape[-1]
        rows_per_ir = 1 if n_ch == C else C
        if bypass is not None:
            bypass = torch.as_tensor(bypass).reshape(-1).to(x.device).repeat_interleave(n_ch)
            bypass = self._bypass(bypass, B * n_ch, x.device)
        ws_bytes = self.lib.b2a_circconv_path_workspace_bytes(B * C, T, K, L, rows_per_ir, n_ch, hop)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
        out = torch.empty_like(x)
        self._call(self.lib.b2a_circconv_path_f32, _dptr(x), B * C, T, _dptr(irs), K, L, rows_per_ir, n_ch, hop,
                   int(bool(roll_to_peak)), _dptr(bypass), _dptr(out), _dptr(ws), ws_bytes, self._stream(x))
        return out

    def circular_convolve_backward(self, grad_out: torch.Tensor, ir: torch.Tensor, roll_to_peak: bool = True,
                                   bypass: Optional[torch.Tensor] = None) -> torch.Tensor:
        """dL/dx of :meth:`circular_convolve` (the IR is a constant): circular correlation with the rolled, scaled IR,
        on the same overlap-save engine (csrc/fftconv.cu)."""
        g = self._prep(grad_out, "grad_out")
        B, C, T = g.shape
        ir, n_ir, L, rows_per_ir, bypass = self._circconv_filters(g.shape, ir, bypass, g.device)
        ws_bytes = self.lib.b2a_circconv_backward_workspace_bytes(B * C, T, n_ir, L)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=g.device)
        gx = torch.empty_like(g)
        self._call(self.lib.b2a_circconv_backward_f32, _dptr(g), B * C, T, _dptr(ir), n_ir, L, rows_per_ir,
                   int(bool(roll_to_peak)), _dptr(bypass), _dptr(gx), _dptr(ws), ws_bytes, self._stream(g))
        return gx


    # ------------------------------------------------------------------ resample
    def _resample_kernel(self, old_sr: int, new_sr: int, device, zeros: int = 24, rolloff: float = 0.945):
        """julius.ResampleFrac._init_kernels (float32 arithmetic), transposed to [K, new]; cached."""
        key = (old_sr, new_sr, str(device), zeros, rolloff)
        if key not in self._packed_cache:
            gcd = math.gcd(old_sr, new_sr)
            old, new = old_sr // gcd, new_sr // gcd
            sr = min(new, old) * rolloff
            width = math.ceil(zeros * old / sr)
            idx = torch.arange(-width, width + old, device=device).float()
            i = torch.arange(new, device=device).float().reshape(-1, 1)
            t = (-i / new + idx.reshape(1, -1) / old) * sr
            t = t.clamp(-zeros, zeros) * math.pi
            window = torch.cos(t / zeros / 2) ** 2
            kernel = self._sinc(t) * window
            kernel = kernel / kernel.sum(dim=1, keepdim=True)
            self._packed_cache[key] = (kernel.t().contiguous(), width, old, new)
        return self._packed_cache[key]

    def resample(self, x: torch.Tensor, old_sr: int, new_sr: int) -> torch.Tensor:
        """julius.resample_frac(x, old_sr, new_sr) for x [..., T] (ref:audiotools/core/audio_signal.py:732-734)."""
        x = self._prep(x, "x")
        if int(old_sr) == int(new_sr):
            return x
        kt, width, old, new = self._resample_kernel(int(old_sr), int(new_sr), x.device)
        T = x.shape[-1]
        rows = x.numel() // T
        out_len = int(self.lib.b2a_resample_out_len(T, old, new))
        if new == 1 and self.lib.b2a_fir_direct_supported(T, kt.shape[0], old):
            # single output phase (48k -> 16k, ...): a decimating FIR, register-tiled direct kernel
            return self.fir_direct(x, kt.reshape(1, -1), rows_per_filt=rows, left0=width, stride=old, out_len=out_len,
                                   pad_mode="replicate")
        out = torch.empty(*x.shape[:-1], out_len, dtype=torch.float32, device=x.device)
        self._call(self.lib.b2a_resample_f32, _dptr(x), rows, T, old, new, width, _dptr(kt), _dptr(out), self._stream(x))
        return out

    def resample_backward(self, grad_out: torch.Tensor, T: int, old_sr: int, new_sr: int) -> torch.Tensor:
        """dL/dx [..., T] of :meth:`resample` (either route) for dL/dout [..., out_len]."""
        g = self._prep(grad_out, "grad_out")
        kt, width, old, new = self._resample_kernel(int(old_sr), int(new_sr), g.device)
        assert g.shape[-1] == int(self.lib.b2a_resample_out_len(T, old, new)), (g.shape, T)
        rows = g.numel() // g.shape[-1]
        gx = torch.empty(*g.shape[:-1], int(T), dtype=torch.float32, device=g.device)
        self._call(self.lib.b2a_resample_backward_f32, _dptr(g), rows, int(T), old, new, width, _dptr(kt), _dptr(gx),
                   self._stream(g))
        return gx


    # ------------------------------------------------------------------ pitch shift
    MAX_PITCH_GROUPS = 8

    def pitch_shift(self, x: torch.Tensor, sample_rate: int, n_semitones, quick: bool = True,
                    return_positions: bool = False):
        """Shift the pitch of x [B, C, T] keeping T (ref:audiotools/core/effects.py:247-277).  ``n_semitones`` is one
        value for the batch (the reference's API) or one value per item (host list / tensor with B entries): all
        items go through the same launches, grouped by their shift; a shift of 0 copies the item.
        ``return_positions`` (single shift only; parity tests): also return the WSOLA splice positions the search
        kernel chose, int32 [rows, J] -- the integer part of the result that must match the oracle exactly."""
        x = self._prep(x, "x")
        T = x.shape[-1]
        rows = x.numel() // T
        vals = np.asarray(torch.as_tensor(n_semitones).detach().cpu().reshape(-1).numpy(), dtype=np.float32)
        if vals.size == 1:
            if float(vals[0]) == 0.0:
                return x.clone()
            uniq, row_group = vals, None
        else:
            B = x.shape[0]
            assert vals.size == B, f"{vals.size} shifts for a batch of {B}"
            uniq, inv = np.unique(vals, return_inverse=True)
            if uniq.size == 1:
                return self.pitch_shift(x, sample_rate, float(uniq[0]), quick)
            if uniq.size > self.MAX_PITCH_GROUPS:  # more distinct shifts than one launch takes: split the batch
                out = torch.empty_like(x)
                for i in range(0, uniq.size, self.MAX_PITCH_GROUPS):
                    sel = np.nonzero(np.isin(vals, uniq[i:i + self.MAX_PITCH_GROUPS]))[0]
                    idx = torch.as_tensor(sel, device=x.device)
                    out[idx] = self.pitch_shift(x[idx], sample_rate, vals[sel], quick)
                return out
            per_row = np.repeat(inv.astype(np.int32), rows // B)
            row_group = torch.from_numpy(per_row).to(x.device, non_blocking=True)
        sem = np.ascontiguousarray(uniq, dtype=np.float32)
        sem_p = sem.ctypes.data_as(ctypes.c_void_p)
        ws_bytes = self.lib.b2a_pitch_shift_multi_workspace_bytes(rows, T, int(sample_rate), sem_p, int(sem.size))
        if ws_bytes == 0:
            raise NotImplementedError(f"pitch_shift: unsupported shifts {sem.tolist()} (|semitones| <= 24)")
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
        out = torch.empty_like(x)
        self._call(self.lib.b2a_pitch_shift_multi_f32, _dptr(x), rows, T, int(sample_rate), sem_p, int(sem.size),
                   _dptr(row_group), _dptr(out), _dptr(ws), ws_bytes, self._stream(x))
        if return_positions:
            assert row_group is None, "return_positions: one shift for the whole batch"
            jmax = self.lib.b2a_pitch_shift_num_frames(T, int(sample_rate), float(sem[0]))
            pos = ws[: rows * jmax * 4].view(torch.int32).reshape(rows, jmax).clone()
            return out, pos
        return out


    def time_stretch(self, x: torch.Tensor, sample_rate: int, factor: float, return_positions: bool = False):
        """Speed x [B, C, T] up by ``factor`` without changing its pitch -> [B, C, round(T / factor)]
        (ref:audiotools/core/effects.py:279-309; SoX ``tempo`` there): the WSOLA stages of the pitch shifter."""
        x = self._prep(x, "x")
        T = x.shape[-1]
        rows = x.numel() // T
        factor = float(factor)
        out_len = int(self.lib.b2a_time_stretch_out_len(T, factor))
        ws_bytes = self.lib.b2a_time_stretch_workspace_bytes(rows, T, int(sample_rate), factor)
        if out_len < 1 or ws_bytes == 0:
            raise NotImplementedError(f"time_stretch: factor {factor} (supported: 0.25 ... 4)")
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
        out = torch.empty(*x.shape[:-1], out_len, dtype=torch.float32, device=x.device)
        self._call(self.lib.b2a_time_stretch_f32, _dptr(x), rows, T, int(sample_rate), factor, _dptr(out), _dptr(ws),
                   ws_bytes, self._stream(x))
        if return_positions and factor != 1.0:
            st = float(np.float32(12.0 * math.log2(1.0 / factor)))
            jmax = self.lib.b2a_pitch_shift_num_frames(T, int(sample_rate), st)
            return out, ws[: rows * jmax * 4].view(torch.int32).reshape(rows, jmax).clone()
        return out

    # ------------------------------------------------------------------ STOI (csrc/stoi.cu)
    STOI_RATE = 10000

    @staticmethod
    def stoi_ratio(sample_rate: int):
        """(up, down): 10000 / sample_rate reduced by the gcd, resample_poly's ratio."""
        g = math.gcd(Engine.STOI_RATE, int(sample_rate))
        return Engine.STOI_RATE // g, int(sample_rate) // g

    @staticmethod
    def stoi_taps(sample_rate: int) -> np.ndarray:
        """float64 filter of ``resample_poly(x, up, down, window=h / h.sum())`` as pystoi's ``resample_oct`` designs it
        (Octave's 60 dB Kaiser-windowed sinc, cutoff 1 / (2 max(up, down)), roll-off a tenth of it), times up.  [1] at
        10 kHz, where pystoi does not resample."""
        up, down = Engine.stoi_ratio(sample_rate)
        if up == down == 1:
            return np.ones(1)
        fc = 1.0 / (2 * max(up, down))
        L = np.ceil((60.0 - 8) / (28.714 * fc / 10))
        t = np.arange(-L, L + 1)
        h = np.kaiser(2 * L + 1, 0.1102 * (60.0 - 8.7)) * 2 * up * fc * np.sinc(2 * fc * t)
        return h / h.sum() * up

    def _stoi_taps(self, sample_rate: int, device) -> torch.Tensor:
        key = ("stoi_taps", int(sample_rate), device)
        taps = self._packed_cache.get(key)
        if taps is None:
            taps = self._packed_cache[key] = torch.from_numpy(self.stoi_taps(sample_rate)).to(device)
        return taps

    def stoi(self, est: torch.Tensor, ref: torch.Tensor, sample_rate: int, extended: bool = False,
             return_workspace: bool = False):
        """STOI (or extended STOI) of the estimates against the clean references, both [B, C, T] (mixed to mono first)
        -> (score [B] float64, kept [B] int32 frames kept by the silence removal, short [B] bool: fewer than 30 STFT
        frames were left and the score is 1e-5).  Detached inputs, as the reference's wrapper.  ``return_workspace``:
        also return the forward's workspace (uint8; the 10 kHz signals, kept-frame lists, counts and band envelopes)
        as a fourth value, the input of :meth:`stoi_backward`."""
        est = self._prep(est.detach(), "estimates")
        ref = self._prep(ref.detach(), "references")
        if est.shape != ref.shape or est.ndim != 3:
            raise ValueError(f"stoi: estimates {tuple(est.shape)} and references {tuple(ref.shape)} must be the same "
                             "[batch, channels, samples] shape")
        B, C, T = est.shape
        up, down = self.stoi_ratio(sample_rate)
        n10 = -(-T * up // down)
        if n10 <= 256:
            raise ValueError(f"stoi: {T} samples at {sample_rate} Hz leave no full 256-sample frame at 10 kHz")
        taps = self._stoi_taps(sample_rate, est.device)
        nbytes = int(self.lib.b2a_stoi_workspace_bytes(B, T, up, down))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=est.device)
        out = torch.empty(B, dtype=torch.float64, device=est.device)
        kept = torch.empty(B, dtype=torch.int32, device=est.device)
        short = torch.empty(B, dtype=torch.int32, device=est.device)
        self._call(self.lib.b2a_stoi_f32, _dptr(est), _dptr(ref), B, C, T, int(bool(extended)), _dptr(taps),
                   taps.numel(), up, down, _dptr(out), _dptr(kept), _dptr(short), _dptr(ws), nbytes, self._stream(est))
        if return_workspace:
            return out, kept, short.bool(), ws
        return out, kept, short.bool()

    def stoi_backward(self, grad_score: torch.Tensor, ws: torch.Tensor, shape, sample_rate: int,
                      extended: bool = False) -> torch.Tensor:
        """dL/d estimates [B, C, T] float32 of :meth:`stoi` for dL/dscore [B] (float64), from the forward workspace
        ``ws`` that ``stoi(..., return_workspace=True)`` returned for estimates of ``shape``.  Items scored 1e-5 get
        a zero gradient."""
        B, C, T = (int(v) for v in shape)
        g = self._prep(grad_score, "grad_score", dtype=torch.float64)
        assert g.shape == (B,), (tuple(g.shape), B)
        up, down = self.stoi_ratio(sample_rate)
        taps = self._stoi_taps(sample_rate, ws.device)
        nbytes = int(self.lib.b2a_stoi_backward_workspace_bytes(B, T, up, down))
        bws = torch.empty(nbytes, dtype=torch.uint8, device=ws.device)
        gx = torch.empty(B, C, T, dtype=torch.float32, device=ws.device)
        self._call(self.lib.b2a_stoi_backward_f32, _dptr(g), _dptr(ws), ws.numel(), B, C, T, int(bool(extended)),
                   _dptr(taps), taps.numel(), up, down, _dptr(gx), _dptr(bws), nbytes, self._stream(ws))
        return gx


_ENGINE = None


def get_engine() -> Engine:
    """The product engine: the in-tree CUDA library, CUDA tensors only."""
    global _ENGINE
    if _ENGINE is None:
        _ENGINE = Engine(_lib.get_lib(), require_cuda=True)
    return _ENGINE
