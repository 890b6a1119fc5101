"""``torch.autograd.Function``s over the engine: the differentiable forms of the spectral front end
(ref:audiotools/core/audio_signal.py:1123-1296, 1333-1426 and effects.py:200-238, differentiable through torch there;
ref:tests/core/test_grad.py).  ``AudioSignal`` uses them only when grad mode is on and the input requires a gradient;
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

