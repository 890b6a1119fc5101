"""Float64 references and the per-frame error model of the spectral accuracy tests (tests/test_gpu_spectral_accuracy.py
on the H100, tests/test_sim_spectral_accuracy.py on the simulator).

An FP32 transform's error scales with the norm of the frame it transforms, not with the tensor's largest value, so
every error here is measured per frame: ``frame_rel`` = ||X^ - X||_2 / ||X||_2 over the bins of one frame, and
``bin_err`` = |X^_k - X_k| / rms_k |X_k| (the bin's error in units of the frame's RMS bin magnitude).  Each route has a
budget C u g(n) on the worst ``bin_err`` (u = 2^-24; g = log2 n for the FFT routes, sqrt n for the dense DFT, whose
bins are direct FP32 sums of n products); frame_rel is the RMS of bin_err over a frame, so the same bound covers it.

The torch.stft / torch.istft / mel references are those of tests/grad_cases.py; ``dft64`` and ``dft_stft64`` add a
direct float64 DFT that does not go through any FFT library."""
import math

import numpy as np
import torch

from tests.grad_cases import istft64, mel64, padding, stft64, window64  # noqa: F401  (re-exported references)

U = 2.0 ** -24
LG2_APPROX = 2.0 ** -22  # lg2.approx.f32: absolute error in log2 units (PTX ISA), i.e. 7.2e-8 in log10 units

# Per-route budget constants C of |X^_k - X_k| <= C u g(n) rms(|X|): set once from the H100 measurement in DESIGN.md
# ("Spectral accuracy"; H100 80GB HBM3, 700 W power limit) with about 2x headroom over the worst case measured there
# and on the simulator.  Route names are those of ``route``.
BUDGET_C = {
    "cta32": 2.0,      # spectral_kernel<4>, n_fft 32
    "warp": 2.0,       # spectral_warp_kernel<5..9>, n_fft 64 .. 1024
    "warp_lean": 2.0,  # spectral_warp_kernel<10>, n_fft 2048 (twiddles formed from products: one more rounding)
    "cta4096": 2.0,    # spectral_kernel<11>, n_fft 4096
    "large": 2.0,      # stft_large_kernel, n_fft 8192 .. 32768
    "dense": 6.0,      # dft_forward_kernel, any other n_fft <= 8192 (g = sqrt n)
}


def route(n_fft: int) -> str:
    """The forward kernel ``Engine.spectral`` launches for a window length (hop <= n_fft)."""
    if n_fft & (n_fft - 1) == 0 and 32 <= n_fft <= 32768:
        return {32: "cta32", 2048: "warp_lean", 4096: "cta4096"}.get(n_fft, "warp" if n_fft < 4096 else "large")
    return "dense"


def growth(n_fft: int, rt: str) -> float:
    return math.sqrt(n_fft) if rt == "dense" else math.log2(n_fft)


def budget(n_fft: int) -> float:
    """The bound on ``bin_err`` of a route at a window length (in units of the frame's RMS bin magnitude)."""
    rt = route(n_fft)
    return BUDGET_C[rt] * U * growth(n_fft, rt)


def dft64(n_fft: int, bins=None) -> np.ndarray:
    """[len(bins), n_fft] complex128 rows exp(-2 pi i ((k n) mod n_fft) / n_fft): the exponent reduced in integers,
    the angle and its cosine / sine in float64 (no FFT library)."""
    k = np.arange(n_fft // 2 + 1, dtype=np.int64) if bins is None else np.asarray(bins, dtype=np.int64)
    r = (k[:, None] * np.arange(n_fft, dtype=np.int64)[None, :]) % n_fft
    ang = (-2.0 * np.pi / n_fft) * r.astype(np.float64)
    return np.cos(ang) + 1j * np.sin(ang)


def frames64(x: torch.Tensor, n_fft: int, hop: int) -> torch.Tensor:
    """torch.stft(center=True, pad_mode="reflect")'s frames of x [..., T] in float64: [..., N, n_fft]."""
    lead = x.shape[:-1]
    y = torch.nn.functional.pad(x.double().reshape(-1, 1, x.shape[-1]), (n_fft // 2, n_fft // 2), mode="reflect")
    return y.reshape(*lead, -1).unfold(-1, n_fft, hop)


def dft_stft64(x: torch.Tensor, n_fft: int, hop: int, window: torch.Tensor) -> torch.Tensor:
    """The centred STFT of x [..., T] (reflect padding) by the direct float64 DFT: [..., F, N] complex128."""
    fr = (frames64(x, n_fft, hop) * window.double().to(x.device)).cpu().numpy()
    out = np.einsum("...nj,kj->...kn", fr, dft64(n_fft))
    return torch.from_numpy(out)


def impulse_signal(n_fft: int, offsets) -> torch.Tensor:
    """[T] float32 with one unit impulse per interior frame of a centred STFT with hop = n_fft: frame f = 1 + i holds
    its impulse at in-frame offset offsets[i].  Under a rectangular window frame f's spectrum is then
    exp(-2 pi i k offsets[i] / n_fft) exactly (see ``impulse_spectrum``): frames 1 .. len(offsets); the edge frames
    hold none."""
    offsets = np.asarray(offsets, dtype=np.int64)
    T = (len(offsets) + 2) * n_fft
    x = torch.zeros(T, dtype=torch.float32)
    # frame f covers x[f n - n/2, f n + n/2)
    x[torch.from_numpy((np.arange(1, len(offsets) + 1) * n_fft - n_fft // 2 + offsets))] = 1.0
    return x


def impulse_spectrum(n_fft: int, offsets) -> torch.Tensor:
    """[F, len(offsets)] complex128: exp(-2 pi i ((k j) mod n) / n) with the exponent reduced in integers."""
    offsets = np.asarray(offsets, dtype=np.int64)
    k = np.arange(n_fft // 2 + 1, dtype=np.int64)
    r = (k[:, None] * offsets[None, :]) % n_fft
    ang = (-2.0 * np.pi / n_fft) * r.astype(np.float64)
    return torch.from_numpy(np.cos(ang) + 1j * np.sin(ang))


def frame_errors(got: torch.Tensor, want: torch.Tensor):
    """(frame_rel [..., N], bin_err [..., F, N]) of a complex spectrogram [..., F, N] against its float64 reference.
    Frames whose reference is all zero have frame_rel = bin_err = 0 if ``got`` is zero there too, inf otherwise."""
    got = got.detach().cpu().to(torch.complex128)
    want = want.detach().cpu().to(torch.complex128)
    d = (got - want).abs()
    norm = want.abs().pow(2).sum(-2).sqrt()
    dn = d.pow(2).sum(-2).sqrt()
    rms = norm / math.sqrt(want.shape[-2])
    frame_rel = torch.where(norm > 0, dn / norm.clamp_min(1e-300), torch.where(dn > 0, math.inf, 0.0))
    bin_err = torch.where(rms[..., None, :] > 0, d / rms[..., None, :].clamp_min(1e-300),
                          torch.where(d > 0, math.inf, 0.0))
    return frame_rel, bin_err


def worst(got: torch.Tensor, want: torch.Tensor):
    """(max frame_rel, max bin_err) as floats."""
    fr, be = frame_errors(got, want)
    return fr.max().item(), be.max().item()


def mel_bound(fb: torch.Tensor, want_stft: torch.Tensor, delta: float, rtol: float) -> torch.Tensor:
    """Per-cell bound rtol mel + sum_k fb[m, k] delta_k of a mel spectrogram [..., M, N] whose STFT has per-bin errors
    delta_k = delta rms(|X|) (the frame's budget; ``want_stft`` [..., F, N] is the float64 STFT)."""
    want_stft = want_stft.detach().cpu().to(torch.complex128)
    fb = fb.detach().cpu().double()
    mag = want_stft.abs()
    rms = mag.pow(2).mean(-2).sqrt()
    mel = (mag.transpose(-1, -2) @ fb.T).transpose(-1, -2)
    return rtol * mel + fb.sum(-1)[:, None] * (delta * rms[..., None, :]), mel


def istft_errors(got: torch.Tensor, want: torch.Tensor, spec: torch.Tensor, window: torch.Tensor, hop: int,
                 keep: slice):
    """Per-sample error of an inverse STFT (centred, length = the output's) in units of the local scale: the RMS bin
    magnitude of the frames that cover the sample, weighted by the window and divided by the envelope sum w^2 there.
    ``keep`` selects the samples compared (the envelope vanishes in the last 2 hop)."""
    n_fft = window.numel()
    w = window.detach().double().cpu()
    spec = spec.detach().cpu().to(torch.complex128)
    N = spec.shape[-1]
    rms = spec.abs().pow(2).mean(-2).sqrt()  # [..., N]
    L = (N - 1) * hop + n_fft
    num = torch.zeros(*rms.shape[:-1], L, dtype=torch.float64)
    env = torch.zeros(L, dtype=torch.float64)
    for f in range(N):
        num[..., f * hop:f * hop + n_fft] += rms[..., f:f + 1] * w.abs()
        env[f * hop:f * hop + n_fft] += w * w
    scale = (num / env.clamp_min(1e-30))[..., n_fft // 2:]
    T = got.shape[-1]
    scale = scale[..., :T]
    d = (got.detach().cpu().double() - want.detach().cpu().double()).abs()
    return (d / scale.clamp_min(1e-300))[..., keep]


# --------------------------------------------------------------------------- checks shared by the GPU and simulator tests
# Impulse (DFT-matrix) checks have their own constants: each output is one column of the transform, so the error is
# the twiddle products' alone.  FFT routes: C_IMPULSE u log2 n (measured <= 0.58).  Dense route: one matrix entry, whose
# cosine and sine are each rounded once from float64: |error| <= u / sqrt 2 (measured 0.70 u).
C_IMPULSE = 1.0
DENSE_IMPULSE = 0.75 * U
# An impulse at offset 1 puts the untangle twiddle exp(-i pi k / N) itself in every bin (the packed transform is i at
# every point): bound by an accurate sincospif (the simulator, correctly rounded: <= 0.71 u; the H100's sincospif is
# accurate to about 1 ulp).  The lean 2048 kernel forms it as a product of two rounded twiddles (measured 1.46 u).
UNTANGLE = {"warp_lean": 3.0 * U}
UNTANGLE_DEFAULT = 1.5 * U
# Inverse STFT: per-sample error in units of the local scale (``istft_errors``), C_INVERSE u log2 n on every route
# (measured <= 0.23 at n = 32, <= 0.06 elsewhere)
C_INVERSE = 1.0
# Mel: |mel^ - mel| <= MEL_RTOL mel + sum_k fb[m, k] budget_k (sqrt.approx: 2 ulp, plus the band's FP32 sum; measured
# within the STFT term alone)
MEL_RTOL = 8 * U


def impulse_offsets(n_fft: int, n_max: int, seed: int = 0):
    """Every in-frame offset when n_fft <= n_max, else n_max sampled offsets (0, 1 and n_fft - 1 always included)."""
    if n_fft <= n_max:
        return np.arange(n_fft)
    rng = np.random.default_rng(seed + n_fft)
    return np.unique(np.concatenate([[0, 1, n_fft - 1], rng.choice(n_fft, n_max - 3, replace=False)]))


def impulse_error(spectral, n_fft: int, offsets, dev) -> float:
    """Worst |X^_k - exp(-2 pi i k j / n)| of the STFT of ``impulse_signal`` (rectangular window, hop = n_fft) over
    every bin of every interior frame.  ``spectral(x [1, 1, T], n_fft, hop, window)`` returns the complex STFT."""
    x = impulse_signal(n_fft, offsets)[None, None].to(dev)
    got = spectral(x, n_fft, n_fft, torch.ones(n_fft, device=dev))[0, 0, :, 1:1 + len(offsets)]
    return (got.cpu().to(torch.complex128) - impulse_spectrum(n_fft, offsets)).abs().max().item()


def untangle_budget(n_fft: int) -> float:
    """The bound on ``impulse_error`` at offset 1."""
    return UNTANGLE.get(route(n_fft), UNTANGLE_DEFAULT)


def impulse_budget(n_fft: int) -> float:
    rt = route(n_fft)
    return DENSE_IMPULSE if rt == "dense" else C_IMPULSE * U * math.log2(n_fft)


def signals(n_fft: int, hop: int, frames: int, seed: int = 0):
    """{name: x [2, 1, T] float32}: Gaussian noise at three levels, a full-scale tone on a bin centre and one between
    bins over noise 120 dB down, a DC offset plus small noise, and the alternating +-1 sequence (bins 0 and n/2)."""
    T = (frames - 1) * hop + 1
    g = torch.Generator().manual_seed(seed + n_fft)
    t = torch.arange(T, dtype=torch.float64)
    noise = torch.randn(2, 1, T, generator=g, dtype=torch.float64)
    k0 = max(1, n_fft // 8)
    tones = (torch.cos(2 * math.pi * k0 * t / n_fft) + torch.cos(2 * math.pi * (k0 + 3.5) * t / n_fft + 0.3))
    out = {
        "noise": noise, "noise_1e-3": 1e-3 * noise, "noise_1e-6": 1e-6 * noise,
        "tones_120dB": tones + 1e-6 * noise,
        "dc": 1.0 + 1e-4 * noise,
        "nyquist": (1.0 - 2.0 * (t % 2)) + 0 * noise,
    }
    return {k: v.float() for k, v in out.items()}


def windows(n_fft: int, dev, seed: int = 0):
    """hann, sqrt_hann and a random positive window (float32 [n_fft])."""
    from audiotools_b200 import AudioSignal

    g = torch.Generator().manual_seed(seed + 7 * n_fft)
    return {"hann": AudioSignal.get_window("hann", n_fft, dev),
            "sqrt_hann": AudioSignal.get_window("sqrt_hann", n_fft, dev),
            "random": (0.1 + torch.rand(n_fft, generator=g)).to(dev)}


def stft_ref(x: torch.Tensor, n_fft: int, hop: int, window: torch.Tensor, pad=0, right_pad=0, pad_mode="reflect",
             drop_edge=0, dtype=torch.float64) -> torch.Tensor:
    """The engine's STFT geometry through torch.stft, on x's device: float64 (complex128) by default; float32 gives
    torch's own FP32 arithmetic (cuFFT on the GPU) for comparison."""
    y = torch.nn.functional.pad(x.to(dtype), (pad, pad + right_pad), mode=pad_mode) if (pad or right_pad) else x.to(dtype)
    X = torch.stft(y.reshape(-1, y.shape[-1]), n_fft, hop, window=window.to(x.device, dtype), center=True,
                   return_complex=True, pad_mode="reflect")
    X = X.reshape(*x.shape[:-1], *X.shape[-2:])
    return X[..., drop_edge:X.shape[-1] - drop_edge] if drop_edge else X


def adjoint_scale(G: torch.Tensor, window: torch.Tensor, hop: int, T: int) -> torch.Tensor:
    """Local scale of the STFT's adjoint (its VJP) at each sample of x [..., T] under centred reflect framing:
    sum over the frames f and window taps n that read the sample of |w[n]| ||G_f||_2 (float64, CPU)."""
    n_fft = window.numel()
    w = window.detach().double().cpu().abs()
    norm = G.detach().cpu().to(torch.complex128).abs().pow(2).sum(-2).sqrt()  # [..., N]
    N = norm.shape[-1]
    L = (N - 1) * hop + n_fft
    sp = torch.zeros(*norm.shape[:-1], L, dtype=torch.float64)
    for f in range(N):
        sp[..., f * hop:f * hop + n_fft] += norm[..., f:f + 1] * w
    p = torch.arange(L) - n_fft // 2  # padded position -> x index, reflected at both ends
    p = torch.where(p < 0, -p, p)
    p = torch.where(p > T - 1, 2 * (T - 1) - p, p)
    out = torch.zeros(*norm.shape[:-1], T, dtype=torch.float64)
    ok = (p >= 0) & (p < T)
    return out.index_add_(-1, p[ok], sp[..., ok]).clamp_min(1e-300)
