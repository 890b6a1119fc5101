"""``torch.autograd.Function``s over the engine: the differentiable forms of the spectral front end
(ref:audiotools/core/audio_signal.py:1123-1296, 1333-1426 and effects.py:200-238, differentiable through torch there;
ref:tests/core/test_grad.py) and of the time-domain effects (resample, equalizer, convolve, apply_ir,
ensure_max_of_audio, mix, quantization, sos_filter, sosfiltfilt; gradients with respect to the waveform only) and of the spectral masks and the
spectral gate (ref:audiotools/core/dsp.py:217-334, ml/layers/spectral_gate.py:58-127; gradients to the spectrogram)
and of STOI and the integrated loudness (``metrics.quality.STOILoss``, ``metrics.LoudnessLoss``; gradients to the
estimates).  ``AudioSignal`` uses them only when grad mode is on and the input requires a gradient;
otherwise it calls the engine directly, with exactly the launches it always made.

Each forward is the engine call of the no-gradient path; each backward is one launch sequence of csrc/grad.cu (or an
existing kernel: the DCT and the gain are their own transposes) and is ``once_differentiable``.  Windows, filterbanks,
DCT bases and gains are constants: no gradient flows to them.
"""
import torch
from torch.autograd.function import once_differentiable


def _engine():
    from ..engine import get_engine

    return get_engine()


class Spectral(torch.autograd.Function):
    """x [B, C, T] -> (STFT [B, C, F, N] complex64 or None, mel [B, C, n_mels, N] or None), one ``Engine.spectral``
    launch.  With a mel output the STFT is materialised too (the mel backward needs it: 8 F N bytes per row)."""

    @staticmethod
    def forward(ctx, x, n_fft, hop, window, pad, right_pad, pad_mode, drop_edge, mel, want_stft):
        ctx.set_materialize_grads(False)  # an output nobody used has no gradient (None), not a tensor of zeros
        eng = _engine()
        kw = {}
        if mel is not None:
            fb, lo, hi, post, eps, power = mel
            kw = dict(mel_fb=fb, mel_lo=lo, mel_hi=hi, post=post, post_eps=eps, post_power=power)
        out = eng.spectral(x, n_fft, hop, window, pad=pad, right_pad=right_pad, pad_mode=pad_mode, drop_edge=drop_edge,
                           want_stft=True, **kw)
        ctx.geo = (x.shape[-1], n_fft, hop, window, pad, right_pad, pad_mode, drop_edge)
        ctx.mel = mel
        ctx.save_for_backward(out["stft"] if mel is not None else None)
        if mel is None:
            return out["stft"], None
        stft = out["stft"] if want_stft else None
        return stft, out["mel"]

    @staticmethod
    @once_differentiable
    def backward(ctx, g_stft, g_mel):
        eng = _engine()
        T, n_fft, hop, window, pad, right_pad, pad_mode, drop_edge = ctx.geo
        g = g_stft
        if g_mel is not None:
            (stft,) = ctx.saved_tensors
            fb, lo, hi, post, eps, power = ctx.mel
            gm = eng.mel_backward(stft, g_mel, fb, lo, hi, post, eps, power)
            g = gm if g is None else g + gm
        if g is None:
            return (None,) * 10
        gx = eng.stft_backward(g, T, n_fft, hop, window, pad, right_pad, pad_mode, drop_edge)
        return gx, None, None, None, None, None, None, None, None, None


class ISTFT(torch.autograd.Function):
    """spec [B, C, F, N] complex -> [B, C, length] (``Engine.istft``)."""

    @staticmethod
    def forward(ctx, spec, n_fft, hop, window, length, pad_frames, trim):
        ctx.geo = (spec.shape[-1], n_fft, hop, window, pad_frames, trim)
        return _engine().istft(spec, n_fft, hop, window, length=length, pad_frames=pad_frames, trim=trim)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        n_frames, n_fft, hop, window, pad_frames, trim = ctx.geo
        gs = _engine().istft_backward(g, n_frames, n_fft, hop, window, pad_frames=pad_frames, trim=trim)
        return gs, None, None, None, None, None, None


class MelDCT(torch.autograd.Function):
    """log-mel [B, C, n_mels, N] -> mfcc [B, C, n_mfcc, N] (``Engine.mel_dct``); the backward is the same kernel with
    the transposed basis."""

    @staticmethod
    def forward(ctx, logmel, dct):
        ctx.dct = dct
        return _engine().mel_dct(logmel, dct)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return _engine().mel_dct(g, ctx.dct.t().contiguous()), None


class Gain(torch.autograd.Function):
    """x [B, ...] * gain[b] (``Engine.gain``); the gain is a constant (normalize's gain comes from the loudness, which
    is not differentiable in the reference either)."""

    @staticmethod
    def forward(ctx, x, gain):
        ctx.gain = gain
        return _engine().gain(x, gain)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return _engine().gain(g, ctx.gain), None


class SpectralLoss(torch.autograd.Function):
    """(x, y) [B, C, T] -> one scale of the reference's L1 spectral loss, a 0-dim tensor (``Engine.spectral_loss``: one
    launch plus the partials' sum).  The forward writes dL/dX (and dL/dY when y requires a gradient) of the two STFTs;
    the backward is the STFT adjoint of that buffer, scaled by the upstream gradient on the device."""

    @staticmethod
    def forward(ctx, x, y, n_fft, hop, window, pad, right_pad, pad_mode, drop_edge, mel, clamp_eps, pow, log_weight,
                mag_weight):
        loss, gx, gy = _engine().spectral_loss(
            x, y, n_fft, hop, window, pad=pad, right_pad=right_pad, pad_mode=pad_mode, drop_edge=drop_edge, mel=mel,
            clamp_eps=clamp_eps, pow=pow, log_weight=log_weight, mag_weight=mag_weight,
            want_grad_x=ctx.needs_input_grad[0], want_grad_y=ctx.needs_input_grad[1])
        ctx.geo = (x.shape[-1], n_fft, hop, window, pad, right_pad, pad_mode, drop_edge)
        ctx.grads = (gx, gy)
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        eng = _engine()
        T, n_fft, hop, window, pad, right_pad, pad_mode, drop_edge = ctx.geo
        out = []
        for gs in ctx.grads:
            if gs is None:
                out.append(None)
                continue
            gw = eng.stft_backward(gs, T, n_fft, hop, window, pad, right_pad, pad_mode, drop_edge)
            out.append(eng.gain(gw, g.reshape(1).expand(gw.shape[0])))
        ctx.grads = None
        return (out[0], out[1]) + (None,) * 12


class Resample(torch.autograd.Function):
    """x [..., T] -> [..., floor(new T / old)] (``Engine.resample``); backward: ``Engine.resample_backward``."""

    @staticmethod
    def forward(ctx, x, old_sr, new_sr):
        ctx.geo = (x.shape[-1], old_sr, new_sr)
        return _engine().resample(x, old_sr, new_sr)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        T, old_sr, new_sr = ctx.geo
        return _engine().resample_backward(g, T, old_sr, new_sr), None, None


class Equalizer(torch.autograd.Function):
    """x [B, C, T] -> the mel-band equaliser (``Engine.equalizer``); the band gains are constants."""

    @staticmethod
    def forward(ctx, x, sample_rate, db, bypass):
        ctx.save_for_backward(db)  # saved, not kept: an in-place change before backward() is then an error
        ctx.args = (sample_rate, bypass)
        return _engine().equalizer(x, sample_rate, db, bypass=bypass)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (db,) = ctx.saved_tensors
        sample_rate, bypass = ctx.args
        return _engine().equalizer_backward(g, sample_rate, db, bypass=bypass), None, None, None


class CircConv(torch.autograd.Function):
    """x [B, C, T] -> circular convolution with the rolled, peak-scaled IR (``Engine.circular_convolve``); the IR is a
    constant."""

    @staticmethod
    def forward(ctx, x, ir, roll_to_peak, bypass):
        ctx.save_for_backward(ir)
        ctx.args = (roll_to_peak, bypass)
        return _engine().circular_convolve(x, ir, roll_to_peak=roll_to_peak, bypass=bypass)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (ir,) = ctx.saved_tensors
        roll_to_peak, bypass = ctx.args
        return _engine().circular_convolve_backward(g, ir, roll_to_peak=roll_to_peak, bypass=bypass), None, None, None


class PeakScale(torch.autograd.Function):
    """A per-row rescale by a factor that depends on the row's peak: ``ensure_max_of_audio`` (``x_ref`` None: y * p,
    p = max_abs / max|y| where that exceeds max_abs) or apply_ir's restore (y * clamp(max|x_ref|) / clamp(max|y|)).
    ``fwd(y)`` is the no-gradient path's computation; the backward recomputes the arg-maxes from y and x_ref."""

    @staticmethod
    def forward(ctx, y, x_ref, max_abs, bypass, fwd):
        ctx.save_for_backward(y, x_ref)
        ctx.args = (max_abs, bypass)
        return fwd(y)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        y, x_ref = ctx.saved_tensors
        max_abs, bypass = ctx.args
        gy, gx = _engine().peak_scale_backward(g, y, x_ref, max_abs=max_abs, bypass=bypass)
        return gy, (gx if ctx.needs_input_grad[1] else None), None, None, None


class Mix(torch.autograd.Function):
    """x + other_gain[item] * other (``Engine.mix``); the gain is a constant (it comes from the loudness)."""

    @staticmethod
    def forward(ctx, x, other, other_gain):
        ctx.gain = other_gain
        return _engine().mix(x, other, other_gain)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        go = None
        if ctx.needs_input_grad[1]:
            go = _engine().gain(g, ctx.gain) if ctx.gain is not None else g.clone()
        return (g if ctx.needs_input_grad[0] else None), go, None


class StraightThrough(torch.autograd.Function):
    """``fwd(x)`` with the identity as its gradient: the reference's quantisers return x - (x - q).detach()."""

    @staticmethod
    def forward(ctx, x, fwd):
        return fwd(x)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return g, None


class SpecBandMask(torch.autograd.Function):
    """spec [B, C, F, N] complex64 -> a copy with the band lo[item] <= axis_vals < hi[item] filled
    (``Engine.spec_band_mask_out``); the band is a constant (a comparison in the reference)."""

    @staticmethod
    def forward(ctx, spec, axis_vals, lo, hi, axis, val):
        ctx.save_for_backward(spec)
        ctx.args = (axis_vals, lo, hi, axis)
        return _engine().spec_band_mask_out(spec, axis_vals, lo, hi, axis, val)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (spec,) = ctx.saved_tensors
        return _engine().spec_band_mask_backward(g, spec, *ctx.args), None, None, None, None, None


class SpecMaskLow(torch.autograd.Function):
    """``mask_low_magnitudes`` out of place (``Engine.spec_mask_low_out``); the backward reuses the forward's maximum
    |X|^2 and recomputes the mask from the saved spectrogram."""

    @staticmethod
    def forward(ctx, spec, db_cutoff, val):
        out, ws = _engine().spec_mask_low_out(spec, db_cutoff, val)
        ctx.save_for_backward(spec)
        ctx.args = (db_cutoff, val, ws)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (spec,) = ctx.saved_tensors
        db_cutoff, val, ws = ctx.args
        return _engine().spec_mask_low_backward(g, spec, db_cutoff, val, ws), None, None


class SpecGate(torch.autograd.Function):
    """The spectral gate's ``spec * (1 - amount * mask)`` (``Engine.spec_gate``).  The noise spectrogram and the amount
    are constants; the backward recomputes the mask from the saved spectrogram and the forward's thresholds."""

    @staticmethod
    def forward(ctx, spec, nz_spec, n_std, amount, smooth_f, smooth_t):
        out, thresh = _engine().spec_gate(spec, nz_spec, n_std, amount, smooth_f, smooth_t)
        ctx.save_for_backward(spec)
        ctx.args = (thresh, amount, smooth_f, smooth_t)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (spec,) = ctx.saved_tensors
        return _engine().spec_gate_backward(g, spec, *ctx.args), None, None, None, None, None


class STOI(torch.autograd.Function):
    """(estimates, references) [B, C, T] -> STOI scores [B] float64 on the device (``Engine.stoi``).  The forward keeps
    its workspace (10 kHz signals, kept frames, band envelopes); the backward (``Engine.stoi_backward``) recomputes
    only the estimate's frame spectra from it.  The silence mask depends on the references alone, and the references
    are constants: no gradient flows to them."""

    @staticmethod
    def forward(ctx, est, ref, sample_rate, extended):
        score, _, _, ws = _engine().stoi(est, ref, sample_rate, extended, return_workspace=True)
        ctx.ws = ws
        ctx.args = (tuple(est.shape), sample_rate, extended)
        return score

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        shape, sample_rate, extended = ctx.args
        return _engine().stoi_backward(g, ctx.ws, shape, sample_rate, extended), None, None, None


class Loudness(torch.autograd.Function):
    """(x [B, C, T], gain [B] or None) -> loud [B] = max(lufs, -70), bit for bit ``loudness()``'s value of the samples
    float32(gain x) zero-extended to ``padded_length`` (``Engine.lufs`` with its block energies).  The forward keeps
    x, the block energies and the unclamped loudness; the backward (``Engine.lufs_backward``) rebuilds the gate
    decisions from them (constants of the backward: they are piecewise constant) and recomputes the K-weighted
    signal.  The gain is a constant."""

    @staticmethod
    def forward(ctx, x, gain, sample_rate, padded_length):
        eng = _engine()
        xs = x if gain is None else eng.gain(x, gain)
        out = eng.lufs(xs, sample_rate, padded_length=padded_length, want_blocks=True)
        ctx.save_for_backward(x)
        ctx.args = (gain, sample_rate, padded_length, out["blocks"], out["lufs"])
        return out["loud"]

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        gain, sample_rate, padded_length, blocks, lufs = ctx.args
        gx = _engine().lufs_backward(g, x, sample_rate, blocks, lufs, padded_length=padded_length, gain=gain)
        return gx, None, None, None


class SOSFilter(torch.autograd.Function):
    """x [B, C, T] -> the cascade of second-order sections (``Engine.sos_filter``), after an optional per-item gain.
    The adjoint of a zero-state linear time-invariant filter is the same filter run backwards in time, so the backward
    is ``Engine.sos_filter(g, sos, gain, reverse=True)``; the sections and the gain are constants."""

    @staticmethod
    def forward(ctx, x, sos, gain):
        ctx.args = (sos, gain)
        return _engine().sos_filter(x, sos, gain=gain)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        sos, gain = ctx.args
        return _engine().sos_filter(g, sos, gain=gain, reverse=True), None, None


class SOSFiltFilt(torch.autograd.Function):
    """x [B, C, T] -> the zero-phase cascade (``Engine.sos_filtfilt``), after an optional per-item gain.  The backward
    (``Engine.sos_filtfilt_backward``) composes the adjoints of the two passes, the rank-one terms of their start
    states (each is linear in one sample) and the fold of the edge extension; the sections and the gain are
    constants."""

    @staticmethod
    def forward(ctx, x, sos, gain, padtype, padlen):
        ctx.args = (sos, gain, padtype, padlen)
        return _engine().sos_filtfilt(x, sos, padtype, padlen, gain=gain)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        sos, gain, padtype, padlen = ctx.args
        return _engine().sos_filtfilt_backward(g, sos, padtype, padlen, gain=gain), None, None, None, None


def refuse_param_grad(method: str, name: str, t) -> None:
    """Gradients reach audio_data only: a parameter (IR, db, snr) that requires one raises at forward time."""
    if torch.is_tensor(t) and wants_grad(t):
        raise NotImplementedError(f"{method}: {name} requires a gradient; gradients flow to audio_data only "
                                  f"({name} is a constant of the backward pass)")


def wants_grad(t) -> bool:
    return t is not None and t.requires_grad and torch.is_grad_enabled()


MAX_ROWS = 65535     # rows (items x channels) of one backward launch (grid y of csrc/grad.cu)
MAX_MELS = 1600      # mel filters of the mel backward (their gradients for 32 frames sit in 200 KB of shared memory)


def check_supported(method: str, n_fft: int, hop: int, rows: int, n_mels: int = 0):
    """Raise at forward time, not inside backward(), for a geometry without a backward pass."""
    eng = _engine()
    if not eng.backward_supported(n_fft, hop):
        raise eng.route_error(n_fft, hop, 1, backward_of=method)
    if rows > MAX_ROWS or n_mels > MAX_MELS:
        raise NotImplementedError(f"{method}: no backward for {rows} rows (items x channels) / {n_mels} mel filters: "
                                  f"gradients support up to {MAX_ROWS} rows and {MAX_MELS} mel filters")

