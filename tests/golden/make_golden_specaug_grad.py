"""Golden gradients of the REAL reference's spectral masks and spectral gate (its AudioSignal differentiates through
torch; the julius shims as in ``make_golden.py``; run here only):
``python tests/golden/make_golden_specaug_grad.py`` -> ``reference_golden_specaug_grad.npz``
(ref:audiotools/core/dsp.py:217-334 mask_frequencies / mask_timesteps / mask_low_magnitudes,
ref:audiotools/ml/layers/spectral_gate.py:58-127 SpectralGate, ref:audiotools/data/transforms.py FrequencyMask, TimeMask,
MaskLowMagnitudes, TimeNoise, SpectralDenoising).

Two kinds of case, both run by ``run_case`` (shared with the tests; ``pkg`` is the package to run, the reference's
``audiotools`` here, ``audiotools_b200`` in the tests):
* spectral-domain VJPs: the same complex X [3, 1, F, N] is a leaf ``stft_data`` on both sides; the golden keeps the
  gradient dL/dX of L = <out, G> and the reference's boolean mask.  X has exact zeros: item 2 is silent and item 0 has
  zero frames at both ends (zero padding).  The gate's STFTs come from a signal class whose ``stft()`` hands out the
  leaf (and the noise spectrogram) and whose ``istft()`` keeps the spectrogram, so the reference's own gate runs on X.
* end-to-end waveform gradients: stft -> mask -> istft, seeded SpecAugment transforms with prob 1, TimeNoise (its noise
  fills masked cells: constants, so the gradient does not depend on the draw), SpectralGate and SpectralDenoising.

Mask decisions near a threshold (a db_cutoff, the gate's per-bin threshold) may flip between two float32
implementations.  ``main`` records, through wrappers around the reference's methods, how far every cell's dB value lies
from its threshold and asserts that none is within MARGIN_DB: the seeded inputs keep every decision clear of it."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)

MARGIN_DB = 1e-3
F, N, NZ_N = 33, 70, 50  # > one gate tile (16 bins x 64 frames) in both directions
SR_SPEC = 16000          # the sample rate of the spectral-domain signals: F bins over [0, 8 kHz]
DUR_SPEC = 0.5           # their duration: N frames over [0, 0.5 s]

FMIN, FMAX = torch.tensor([1000.0, 2100.0, 300.0]), torch.tensor([3100.0, 5200.0, 900.0])
TMIN, TMAX = torch.tensor([0.101, 0.0, 0.2]), torch.tensor([0.203, 0.06, 0.45])
DBCUT = torch.tensor([-20.0, -5.0, -60.0])

# key -> (kind, method, arguments)
CASES = {
    "freq_val0": ("spec", "mask_frequencies", dict(val=0.0)),
    "freq_val025": ("spec", "mask_frequencies", dict(val=0.25)),
    "time_val0": ("spec", "mask_timesteps", dict(val=0.0)),
    "time_val025": ("spec", "mask_timesteps", dict(val=0.25)),
    "low_val0": ("spec", "mask_low_magnitudes", dict(val=0.0)),
    "low_val05": ("spec", "mask_low_magnitudes", dict(val=0.5)),
    "gate_shared_scalar": ("spec", "gate", dict(nz="shared", amount=0.9)),
    "gate_shared_items": ("spec", "gate", dict(nz="shared", amount=[1.0, 0.6, 0.8])),
    "gate_items_scalar": ("spec", "gate", dict(nz="items", amount=0.7)),
    "gate_items_items": ("spec", "gate", dict(nz="items", amount=[0.5, 1.0, 0.9])),
    "e2e_freq_time_low": ("wave", "stft_mask_istft", {}),
    "e2e_compose": ("wave", "compose", {}),
    "e2e_time_noise": ("wave", "time_noise", {}),
    "e2e_gate": ("wave", "gate", {}),
    "e2e_denoising": ("wave", "denoising", {}),
}
SEEDS = [11, 12]


def spec_input(seed=0):
    """[3, 1, F, N] complex64: magnitudes spread over ~80 dB, item 2 silent, item 0 with 3 + 2 zero edge frames."""
    g = torch.Generator().manual_seed(300 + seed)
    re, im = torch.randn(2, 3, 1, F, N, generator=g)
    scale = 10.0 ** (-4.0 * torch.rand(3, 1, F, N, generator=g))
    X = torch.complex(re * scale, im * scale)
    X[2] = 0
    X[0, ..., :3] = 0
    X[0, ..., -2:] = 0
    return X


def noise_spec(kind, seed=0):
    g = torch.Generator().manual_seed(400 + seed + (kind == "items"))
    shape = (1, 1, F, NZ_N) if kind == "shared" else (3, 1, F, NZ_N)
    re, im = 0.01 * torch.randn(2, *shape, generator=g)
    return torch.complex(re, im)


def cotangent(shape, seed, complex_=False):
    g = torch.Generator().manual_seed(seed)
    if complex_:
        return torch.randn(shape, dtype=torch.complex64, generator=g)
    return torch.randn(*shape, generator=g)


def wave_input(sr, T, seed=0):
    """[2, 1, T] float32: a chirp plus seeded noise, item 1 quieter."""
    g = torch.Generator().manual_seed(600 + seed)
    t = torch.arange(T, dtype=torch.float64) / sr
    chirp = 0.3 * torch.sin(2 * np.pi * (200.0 * t + 0.5 * 0.4 * sr * t * t / (T / sr)))
    x = chirp + 0.05 * torch.randn(2, 1, T, generator=g, dtype=torch.float64)
    return (x * torch.tensor([1.0, 0.3], dtype=torch.float64)[:, None, None]).float()


def leaf_signal_class(pkg, spectra: dict):
    """A subclass of pkg.AudioSignal whose stft() hands out spectra["x"] (samples 0) or spectra["nz"] (samples 1) and
    whose istft() keeps stft_data: the gate's own code then runs on a given spectrogram."""

    class LeafSignal(pkg.AudioSignal):
        def stft(self, *a, **k):
            key = "nz" if float(self.audio_data.reshape(-1)[0]) == 1.0 else "x"
            self.stft_data = spectra[key] * 1  # not the leaf itself: the reference's gate multiplies in place
            return self.stft_data

        def istft(self, *a, **k):
            return self

    return LeafSignal


def unrolled(pkg, t, sig, kw):
    """``t(sig, **kw)`` for an all-true mask without the reference's ``signal[mask] = ...`` scatter: that in-place
    write into samples the STFT saved is an error under autograd there.  Each (sub-)transform runs as
    SpectralTransform.transform does: stft -> _transform -> istft (BaseTransforms: _transform)."""
    params = kw[t.name]
    for sub in getattr(t, "transforms", [t]):
        p = params if sub is t else params[sub.name]
        assert bool(p["mask"].all())
        args = {k: v for k, v in p.items() if k != "mask"}
        if isinstance(sub, pkg.data.transforms.SpectralTransform):
            sig.stft()
            sig = sub._transform(sig, **args)
            sig.istft()
        else:
            sig = sub._transform(sig, **args)
    return sig


def run_case(pkg, key, device="cpu", seed=0, public=True):
    """(output, dL/dinput, input) of L = <output, cotangent> for one case, with ``pkg`` the package to run (the
    reference's ``audiotools`` or ``audiotools_b200``).  ``public``: transforms run through ``t(signal, **kwargs)``,
    else through ``unrolled`` (the reference)."""
    kind, method, args = CASES[key]
    ct_seed = 7000 + sorted(CASES).index(key)
    if kind == "spec":
        X = spec_input(seed).to(device).requires_grad_()
        if method == "gate":
            spectra = {"x": X, "nz": noise_spec(args["nz"], seed).to(device)}
            Sig = leaf_signal_class(pkg, spectra)
            gate = pkg.ml.layers.SpectralGate().to(device)
            amount = torch.tensor(args["amount"], device=device)
            s = gate(Sig(torch.zeros(3, 1, 16, device=device), SR_SPEC), Sig(torch.ones(3, 1, 16, device=device), SR_SPEC),
                     amount)
        else:
            s = pkg.AudioSignal(torch.zeros(3, 1, int(SR_SPEC * DUR_SPEC), device=device), SR_SPEC)
            s.stft_data = X
            if method == "mask_frequencies":
                s.mask_frequencies(FMIN, FMAX, val=args["val"])
            elif method == "mask_timesteps":
                s.mask_timesteps(TMIN, TMAX, val=args["val"])
            else:
                s.mask_low_magnitudes(DBCUT, val=args["val"])
        out = s.stft_data
        G = cotangent(out.shape, ct_seed, complex_=True).to(device)
        L = (torch.view_as_real(out) * torch.view_as_real(G)).sum()
        (gX,) = torch.autograd.grad(L, X)
        return out.detach(), gX, X.detach()

    tfm = pkg.data.transforms
    if method in ("gate", "denoising"):
        sr, T = 44100, 8192  # few cells (2 x 1025 x 17): few near the gate's thresholds
    else:
        sr, T = 16000, 8000
    x = wave_input(sr, T, seed).to(device).requires_grad_()
    sig = pkg.AudioSignal(x * 1.0, sr)
    if method == "stft_mask_istft":
        sig.stft()
        sig.mask_frequencies(FMIN[:2], FMAX[:2]).mask_timesteps(TMIN[:2] / 2, TMAX[:2] / 2)
        sig.mask_low_magnitudes(torch.tensor([-30.0, -45.0]))
        out = sig.istft().audio_data
    elif method in ("compose", "time_noise"):
        if method == "compose":
            t = tfm.Compose([tfm.FrequencyMask(), tfm.TimeMask(), tfm.MaskLowMagnitudes()])
        else:
            t = tfm.TimeNoise(t_width=("const", 0.2))
        kw = t.batch_instantiate([s + 100 * seed for s in SEEDS], pkg.AudioSignal(x.detach().clone(), sr))
        kw = pkg.core.util.prepare_batch(kw, device)
        out = (t(sig, **kw) if public else unrolled(pkg, t, sig, kw)).audio_data
    elif method == "gate":
        nz = 0.05 * torch.randn(2, 1, 22050, generator=torch.Generator().manual_seed(500 + seed)).to(device)
        gate = pkg.ml.layers.SpectralGate().to(device)
        out = gate(sig, pkg.AudioSignal(nz, sr), torch.tensor([0.9, 0.8], device=device)).audio_data
    else:
        t = tfm.SpectralDenoising()
        kw = t.batch_instantiate([s + 100 * seed for s in SEEDS], pkg.AudioSignal(x.detach().clone(), sr))
        kw = pkg.core.util.prepare_batch(kw, device)
        out = (t(sig, **kw) if public else unrolled(pkg, t, sig, kw)).audio_data
    ct = cotangent(out.shape, ct_seed).to(device)
    (gx,) = torch.autograd.grad((out * ct).sum(), x)
    return out.detach(), gx, x.detach()


def ref_mask(key, X, seed):
    """The reference's boolean mask of a spectral-domain case, restated (dsp.py:244-250 / :290-296, the comparison of
    :326-330 on log_magnitude(), spectral_gate.py:102-112)."""
    from oracle import signal_path as sp

    kind, method, args = CASES[key]
    B = X.shape[0]
    if method == "mask_frequencies":
        bins = torch.linspace(0, SR_SPEC / 2, F)[None, None, :, None]
        return ((FMIN.reshape(B, 1, 1, 1) <= bins) & (bins < FMAX.reshape(B, 1, 1, 1))).expand(X.shape)
    if method == "mask_timesteps":
        bins = torch.linspace(0, DUR_SPEC, N)[None, None, None, :]
        return ((TMIN.reshape(B, 1, 1, 1) <= bins) & (bins < TMAX.reshape(B, 1, 1, 1))).expand(X.shape)
    if method == "mask_low_magnitudes":
        return sp.log_magnitude(X) < DBCUT.reshape(B, 1, 1, 1)
    db, thresh = gate_db_thresh(X, noise_spec(args["nz"], seed))
    return db < thresh


def gate_db_thresh(X, nz_X, n_std=3.0):
    """The gate's dB values of X and per-bin thresholds (ref:audiotools/ml/layers/spectral_gate.py:97-105)."""
    nz_db = 20 * nz_X.abs().clamp(1e-4).log10()
    thresh = nz_db.mean(keepdim=True, dim=-1) + nz_db.std(keepdim=True, dim=-1) * n_std
    return 20 * X.abs().clamp(1e-4).log10(), thresh


def install_margin_probes(at, margins: list):
    """Wrap the reference's mask_low_magnitudes and SpectralGate.forward so that each call appends the smallest
    |dB - threshold| over its cells to ``margins``; the wrapped methods run unchanged."""
    AS = at.AudioSignal
    low = AS.mask_low_magnitudes

    def mask_low(self, db_cutoff, val=0.0):
        with torch.no_grad():
            lm = self.log_magnitude()
            cut = at.core.util.ensure_tensor(db_cutoff, ndim=lm.ndim).to(lm)
            margins.append(float((lm - cut).abs().min()))
        return low(self, db_cutoff, val)

    AS.mask_low_magnitudes = mask_low
    Gate = at.ml.layers.SpectralGate
    fwd = Gate.forward

    def gate(self, audio_signal, nz_signal, denoise_amount=1.0, n_std=3.0, win_length=2048, hop_length=512):
        with torch.no_grad():
            p = at.STFTParams(win_length, hop_length, "sqrt_hann")
            a, n = audio_signal.clone(), nz_signal.clone()
            a.stft_data, a.stft_params, n.stft_params = None, p, p
            db, thresh = gate_db_thresh(a.stft(), n.stft(), n_std)
            margins.append(float((db - thresh).abs().min()))
        return fwd(self, audio_signal, nz_signal, denoise_amount, n_std, win_length, hop_length)

    Gate.forward = gate


def main():
    from tests.golden.make_golden import import_reference

    at = import_reference()
    import audiotools.data.transforms  # noqa: F401
    import audiotools.ml.layers  # noqa: F401

    out = {}
    for key, (kind, method, _) in CASES.items():
        for seed in range(20):  # the first seed whose mask decisions all stand clear of their thresholds
            margins = []
            saved = (at.AudioSignal.mask_low_magnitudes, at.ml.layers.SpectralGate.forward)
            install_margin_probes(at, margins)
            try:
                y, g, inp = run_case(at, key, seed=seed, public=False)
            finally:
                at.AudioSignal.mask_low_magnitudes, at.ml.layers.SpectralGate.forward = saved
            if all(m > MARGIN_DB for m in margins):
                break
        assert all(m > MARGIN_DB for m in margins), (key, margins)
        out[f"{key}_seed"] = np.int64(seed)
        out[f"{key}_grad"] = g.numpy()
        out[f"{key}_margin_db"] = np.float64(min(margins, default=np.inf))
        if kind == "spec":
            out[f"{key}_mask"] = ref_mask(key, inp, seed).numpy()
        print(f"{key}: seed {seed}, |grad| max {g.abs().max():.3g}, "
              f"smallest threshold distance {min(margins, default=np.inf):.3g} dB")
    path = os.path.join(HERE, "reference_golden_specaug_grad.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
