"""Every spectral route on the H100 (``-m gpu``) against float64, bin by bin and frame by frame (tests/spectral64.py):
the DFT matrix itself through impulses, noise under three windows and three levels, high dynamic range, DC and
Nyquist, every padding mode, mel with empty and one-bin bands, the inverse STFT, the
backward passes, and exact invariances (power-of-two scaling, row independence, frame shift, kernel modes).  Each
error is held to its route's budget (tests/spectral64.py, measured on an H100 80GB HBM3 at a 700 W power limit) and to
a stated factor of cuFFT's error (torch.stft / torch.istft in float32 on the same GPU and input).
tests/probes/spectral_accuracy_probe.py prints the table of DESIGN.md "Spectral accuracy"."""
import math

import pytest
import torch

from tests import spectral64 as s64

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
FFT_LENGTHS = [32, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768]
DENSE_LENGTHS = [2, 3, 400, 1001, 4095, 8191]
# ours <= factor x cuFFT's error, worst bin (FFT routes; measured <= 1.05) and worst inverse sample (measured <= 1.2).
# The dense DFT sums n products directly (error ~ sqrt n, against cuFFT's log n): measured 12.7x (forward, 8191) and
# 5.4x (inverse, 4095); its absolute budget is the bound that matters there.
CUFFT_FACTOR = {"fft": 2.0, "dense": 16.0}
INV_CUFFT_FACTOR = {"fft": 2.0, "dense": 8.0}
C_STFT_VJP = 4.0   # STFT VJP per sample: C u log2 n of sum_f |w| ||G_f|| (measured <= 0.94 on the simulator)
C_MEL_VJP = 32.0   # mel VJP per bin: C u of sum_m |fb[m, k] dmel'[m]| (measured 20.1 at 8192, POST_LOG10)


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


class _NoTorchSpectral:
    """torch.stft / torch.istft / torch.fft.* raise inside the block: the engine may not delegate to them."""

    def __enter__(self):
        self.saved = (torch.stft, torch.istft, {n: getattr(torch.fft, n) for n in ("rfft", "irfft", "fft", "ifft")})

        def forbidden(*a, **k):
            raise AssertionError("torch.stft / torch.istft / torch.fft called")

        torch.stft = torch.istft = forbidden
        for n in self.saved[2]:
            setattr(torch.fft, n, forbidden)

    def __exit__(self, *exc):
        torch.stft, torch.istft, fft = self.saved
        for n, f in fft.items():
            setattr(torch.fft, n, f)


def _ours(eng):
    def f(x, n, hop, w, **kw):
        with _NoTorchSpectral():
            return eng.spectral(x.to(DEV), n, hop, w.to(DEV), **kw)["stft"]
    return f


def _cufft(x, n, hop, w):
    X = torch.stft(x.reshape(-1, x.shape[-1]).to(DEV), n, hop, window=w.to(DEV), center=True, pad_mode="reflect",
                   return_complex=True)
    return X.reshape(*x.shape[:-1], *X.shape[-2:])


def _kind(n):
    return "dense" if s64.route(n) == "dense" else "fft"


@pytest.mark.parametrize("n_fft", FFT_LENGTHS + DENSE_LENGTHS)
def test_dft_matrix_by_impulses(eng, n_fft):
    """Rectangular window, hop = n_fft, one unit impulse per interior frame: frame f's spectrum is exp(-2 pi i k j_f / n)
    exactly, so every twiddle slot, lane role and untangle entry is checked on its own, against a closed form (no FFT
    library).  Every in-frame offset up to 4096, 1024 sampled offsets beyond."""
    offs = s64.impulse_offsets(n_fft, 4096 if n_fft <= 4096 else 1024)
    err = s64.impulse_error(_ours(eng), n_fft, offs, DEV)
    assert err <= s64.impulse_budget(n_fft), (n_fft, err, s64.impulse_budget(n_fft))
    err1 = s64.impulse_error(_ours(eng), n_fft, [1], DEV)  # the untangle twiddles themselves
    assert err1 <= s64.untangle_budget(n_fft), (n_fft, err1 / s64.U)


@pytest.mark.parametrize("n_fft", FFT_LENGTHS + DENSE_LENGTHS)
def test_forward_per_bin_against_float64(eng, n_fft):
    """Noise (three windows, levels 1 / 1e-3 / 1e-6): every bin within the route's budget in units of its frame's RMS
    bin.  Two tones over noise 120 dB down, DC plus small noise, and the alternating sequence (bins 0 and n/2): each
    frame's L2 error within the budget.  The worst bin and the mean frame error within a factor of cuFFT's on the same
    input."""
    hop = max(1, n_fft // 4)
    frames = 24 if n_fft <= 4096 else 8
    sig = s64.signals(n_fft, hop, frames)
    ours = _ours(eng)
    bud = s64.budget(n_fft)
    fac = CUFFT_FACTOR[_kind(n_fft)]
    for wname, w in s64.windows(n_fft, DEV).items():
        for name, x in sig.items():
            if wname != "hann" and name not in ("noise", "tones_120dB"):
                continue
            ref = s64.stft_ref(x.to(DEV), n_fft, hop, w)
            fr, be = s64.frame_errors(ours(x, n_fft, hop, w), ref)
            frc, bec = s64.frame_errors(_cufft(x, n_fft, hop, w), ref)
            if name.startswith("noise"):
                assert be.max().item() <= bud, (n_fft, wname, name, be.max().item() / bud)
            else:  # a sparse spectrum: a few bins set the RMS, so the frame's L2 error is the measure
                assert fr.max().item() <= bud, (n_fft, wname, name, fr.max().item() / bud)
            if _kind(n_fft) == "fft" or name.startswith("noise"):  # (the dense sums' error grows with ||x||_1)
                assert be.max().item() <= fac * max(bec.max().item(), s64.U), (n_fft, wname, name, be.max().item(),
                                                                               bec.max().item())
                assert fr.mean().item() <= fac * max(frc.mean().item(), s64.U), (n_fft, wname, name)


@pytest.mark.parametrize("n_fft", [32, 256, 2048, 4096, 8192, 400, 1001])
@pytest.mark.parametrize("pad_mode", ["reflect", "constant", "replicate"])
def test_padding_modes_per_bin(eng, n_fft, pad_mode):
    """Every padding mode with and without match_stride (the reference's extra padding and the 2 dropped edge frames),
    at lengths that end mid-tile: every bin within the route's budget."""
    hop = n_fft // 4
    for ms in (False, True):
        T = 13 * hop + hop // 2 + 3
        x = torch.randn(2, 1, T, generator=torch.Generator().manual_seed(n_fft + T)).to(DEV)
        w = s64.windows(n_fft, DEV)["hann"]
        right_pad, pad = s64.padding(T, n_fft, hop, ms)
        drop = 2 if ms else 0
        with _NoTorchSpectral():
            got = eng.spectral(x, n_fft, hop, w, pad=pad, right_pad=right_pad, pad_mode=pad_mode, drop_edge=drop)["stft"]
        ref = s64.stft_ref(x, n_fft, hop, w, pad, right_pad, pad_mode, drop)
        assert got.shape == ref.shape
        fr, be = s64.frame_errors(got, ref)
        # edge frames of replicate / constant padding are partly flat (sparse spectra): their L2 error is the measure
        assert be[..., 2:-2].max().item() <= s64.budget(n_fft), (n_fft, pad_mode, ms, be.max().item())
        assert fr.max().item() <= s64.budget(n_fft), (n_fft, pad_mode, ms, fr.max().item())


MEL_CASES = [(2048, 320, 44100), (32, 5, 44100), (8192, 128, 44100), (400, 40, 44100), (512, 160, 44100),
             (4096, 128, 16000)]


def _mel_check(eng, n_fft, n_mels, sr):
    from audiotools_b200 import AudioSignal, _lib

    hop = n_fft // 4
    x = s64.signals(n_fft, hop, 24)
    fb, lo, hi = AudioSignal._mel_tables(sr, n_fft, n_mels, 0.0, None, DEV)
    widths = (hi - lo).cpu()
    w = s64.windows(n_fft, DEV)["hann"]
    for name in ("noise", "tones_120dB", "dc"):
        xs = x[name].to(DEV)
        with _NoTorchSpectral():
            mel = eng.spectral(xs, n_fft, hop, w, mel_fb=fb, mel_lo=lo, mel_hi=hi, want_stft=False)["mel"]
            lg = eng.spectral(xs, n_fft, hop, w, mel_fb=fb, mel_lo=lo, mel_hi=hi, post=_lib.POST_LOG10,
                              post_eps=1e-5, post_power=2.0, want_stft=False)["mel"]
        ref = s64.stft_ref(xs, n_fft, hop, w)
        bound, mel64 = s64.mel_bound(fb, ref, s64.budget(n_fft), s64.MEL_RTOL)
        err = (mel.cpu().double() - mel64).abs()
        assert bool((err <= bound).all()), (n_fft, n_mels, name, (err / bound).max().item())
        # log-mel: for cells above post_eps, error <= power (relative mel bound) / ln 10 + lg2.approx's error
        above = mel64 > 1e-5
        rel = bound / mel64.clamp_min(1e-300)
        lbound = 2.0 * (rel / math.log(10) + s64.LG2_APPROX * math.log10(2)) + 4 * s64.U * (2 * mel64.clamp_min(1e-5).log10().abs())
        lerr = (lg.cpu().double() - 2.0 * mel64.clamp_min(1e-5).log10()).abs()
        assert bool((lerr <= lbound)[above].all()), (n_fft, n_mels, name, (lerr / lbound)[above].max().item())
    return int((widths <= 0).sum()), int((widths == 1).sum())


@pytest.mark.parametrize("n_fft,n_mels,sr", MEL_CASES)
def test_mel_and_log_mel_per_band(eng, n_fft, n_mels, sr):
    """|mel^ - mel| <= rtol mel + sum_k fb[m, k] delta_k per band, delta_k the route's per-bin STFT budget (the fused
    kernel reads |X| through sqrt.approx, so this pins it too); log-mel per band above post_eps within the relative
    mel bound / ln 10 plus lg2.approx's stated error.  The filterbanks include empty and one-bin bands."""
    empty, one = _mel_check(eng, n_fft, n_mels, sr)
    if (n_fft, n_mels) in ((2048, 320), (512, 160)):
        assert one > 0  # the shapes where a band reads a single bin


@pytest.mark.parametrize("n_fft", FFT_LENGTHS + [400, 1001, 4095, 8191])
def test_inverse_per_sample_against_float64(eng, n_fft):
    """istft of complex64 spectra (a consistent STFT and a randomly perturbed, inconsistent one) against float64
    torch.istft of the same input: each sample's error in units of the RMS of the frames that cover it over the
    envelope there; the last 2 hop samples, where the envelope vanishes, are excluded."""
    hop = n_fft // 4
    frames = 24 if n_fft <= 4096 else 8
    x = s64.signals(n_fft, hop, frames)["noise"].to(DEV)
    w = s64.windows(n_fft, DEV)["hann"]
    S = _ours(eng)(x, n_fft, hop, w)
    g = torch.Generator().manual_seed(n_fft)
    pert = S + 0.3 * S.abs().mean() * torch.randn(S.shape, dtype=torch.complex64, generator=g).to(DEV)
    L = x.shape[-1]
    bud = s64.C_INVERSE * s64.U * math.log2(n_fft)
    fac = INV_CUFFT_FACTOR[_kind(n_fft)]
    for name, spec in (("consistent", S), ("perturbed", pert)):
        with _NoTorchSpectral():
            y = eng.istft(spec, n_fft, hop, w, length=L)
        flat = spec.reshape(-1, *spec.shape[-2:])
        yd = torch.istft(flat.to(torch.complex128), n_fft, hop, window=w.double(), center=True, length=L)
        yc = torch.istft(flat, n_fft, hop, window=w, center=True, length=L)
        keep = slice(0, L - 2 * hop)
        e = s64.istft_errors(y, yd.reshape(y.shape), spec, w, hop, keep)
        ec = s64.istft_errors(yc.reshape(y.shape), yd.reshape(y.shape), spec, w, hop, keep)
        assert e.max().item() <= bud, (n_fft, name, e.max().item() / (s64.U * math.log2(n_fft)))
        assert e.max().item() <= fac * max(ec.max().item(), s64.U), (n_fft, name, e.max().item(), ec.max().item())


@pytest.mark.parametrize("n_fft", [32, 64, 256, 2048, 4096, 8192, 400])
def test_backward_per_element(eng, n_fft):
    """The VJPs of stft, istft and mel (POST_NONE, POST_LOG10, POST_LN) against float64 autograd, each element in
    units of its local scale: the stft VJP per sample over sum_f |w| ||G_f||, the istft and mel VJPs per bin over
    their frame's RMS."""
    from audiotools_b200 import AudioSignal, _lib
    from tests import grad_cases as gc

    hop = n_fft // 4
    frames = 16 if n_fft <= 4096 else 6
    x = s64.signals(n_fft, hop, frames)["noise"].to(DEV)
    T = x.shape[-1]
    w = s64.windows(n_fft, DEV)["hann"]
    g = torch.Generator().manual_seed(n_fft)
    S = _ours(eng)(x, n_fft, hop, w)
    G = torch.randn(S.shape, dtype=torch.complex64, generator=g).to(DEV)
    C = C_STFT_VJP * s64.U * math.log2(n_fft)
    with _NoTorchSpectral():
        gx = eng.stft_backward(G, T, n_fft, hop, w)
    xd = x.double().requires_grad_()
    (want,) = torch.autograd.grad(gc.real_inner(s64.stft_ref(xd, n_fft, hop, w), G.to(torch.complex128)), xd)
    scale = s64.adjoint_scale(G, w, hop, T)
    e = (gx.double() - want).abs().cpu() / scale
    assert e.max().item() <= C, (n_fft, "stft vjp", e.max().item() / (s64.U * math.log2(n_fft)))

    gy = torch.randn(2, 1, T, generator=g).to(DEV)
    with _NoTorchSpectral():
        gS = eng.istft_backward(gy, S.shape[-1], n_fft, hop, w)
    Sd = S.to(torch.complex128).requires_grad_()
    yd = torch.istft(Sd.reshape(-1, *S.shape[-2:]), n_fft, hop, window=w.double(), center=True, length=T)
    (wantS,) = torch.autograd.grad((yd.reshape(gy.shape) * gy.double()).sum(), Sd)
    _, be = s64.frame_errors(gS, wantS)
    assert be.max().item() <= s64.budget(n_fft), (n_fft, "istft vjp", be.max().item() / (s64.U * math.log2(n_fft)))

    sr = 44100
    fb, lo, hi = AudioSignal._mel_tables(sr, n_fft, 40 if n_fft >= 256 else 5, 0.0, None, DEV)
    for post, eps, power in ((_lib.POST_NONE, 0.0, 1.0), (_lib.POST_LOG10, 1e-5, 2.0), (_lib.POST_LN, 1e-6, 1.0)):
        gm = torch.randn(2, 1, fb.shape[0], S.shape[-1], generator=g).to(DEV)
        with _NoTorchSpectral():
            gX = eng.mel_backward(S, gm, fb, lo, hi, post, eps, power)
        Sd = S.to(torch.complex128).requires_grad_()
        m = (Sd.abs().transpose(2, -1) @ fb.double().T).transpose(-1, 2)
        if post == _lib.POST_LOG10:
            m = power * m.clamp(eps).log10()
        elif post == _lib.POST_LN:
            m = (m + eps).log()
        (wantX,) = torch.autograd.grad((m * gm.double()).sum(), Sd)
        # bound: a few u of sum_m |fb[m, k] dmel'[m]| (the projection may cancel), dmel' the post-op's derivative
        mel = (S.to(torch.complex128).abs().transpose(2, -1) @ fb.double().T).transpose(-1, 2)
        d = gm.double() * (power / (math.log(10) * mel) * (mel >= eps) if post == _lib.POST_LOG10 else
                           1.0 / (mel + eps) if post == _lib.POST_LN else 1.0)
        scale = (d.abs().transpose(2, -1) @ fb.double()).transpose(-1, 2)
        e = (gX.to(torch.complex128) - wantX).abs() / scale.clamp_min(1e-300)
        assert e.max().item() <= C_MEL_VJP * s64.U, (n_fft, post, e.max().item() / s64.U)


INV_LENGTHS = [32, 64, 256, 2048, 4096, 8192, 32768, 400, 1001]


@pytest.mark.parametrize("n_fft", INV_LENGTHS)
def test_power_of_two_scaling_is_exact(eng, n_fft):
    """stft(2^k x) = 2^k stft(x) and istft likewise, bit for bit, for k in [-40, 20] (no subnormals on the way).  The
    mel is exact for k in [-20, 20] here: sqrt.approx.ftz flushes |X|^2 < 2^-126 to zero, which a bin of 2^-40 x
    reaches (|X| ~ 2^-40 sqrt(n) << 2^-63), so the mel's exact range ends where a bin's |X| falls below 2^-63."""
    from audiotools_b200 import AudioSignal

    hop = n_fft // 4
    x = s64.signals(n_fft, hop, 10)["noise"].to(DEV)
    w = s64.windows(n_fft, DEV)["hann"]
    fb, lo, hi = AudioSignal._mel_tables(16000, n_fft, 40 if n_fft >= 256 else 5, 0.0, None, DEV)
    base = eng.spectral(x, n_fft, hop, w, mel_fb=fb, mel_lo=lo, mel_hi=hi)
    y0 = eng.istft(base["stft"], n_fft, hop, w, length=x.shape[-1])
    for k in (-40, -17, -1, 1, 9, 20):
        s = 2.0 ** k
        out = eng.spectral(x * s, n_fft, hop, w, mel_fb=fb, mel_lo=lo, mel_hi=hi)
        assert torch.equal(out["stft"], base["stft"] * s), (n_fft, k)
        if -20 <= k:
            assert torch.equal(out["mel"], base["mel"] * s), (n_fft, k, "mel")
        assert torch.equal(eng.istft(base["stft"] * s, n_fft, hop, w, length=x.shape[-1]), y0 * s), (n_fft, k)


@pytest.mark.parametrize("n_fft", [32, 256, 2048, 4096, 8192, 400])
def test_rows_are_independent(eng, n_fft):
    """Row r of a launch of 1, 7 or 300 rows equals the same row launched alone (the persistent kernels distribute
    their tiles differently in each case), for the STFT, the mel and the inverse."""
    from audiotools_b200 import AudioSignal

    hop = n_fft // 4
    T = 6 * hop + n_fft // 2 + 5 if n_fft <= 4096 else 3 * n_fft
    fb, lo, hi = AudioSignal._mel_tables(16000, n_fft, 40 if n_fft >= 256 else 5, 0.0, None, DEV)
    w = s64.windows(n_fft, DEV)["hann"]
    x = torch.randn(300, 1, T, generator=torch.Generator().manual_seed(n_fft)).to(DEV)
    alone = {r: eng.spectral(x[r:r + 1], n_fft, hop, w, mel_fb=fb, mel_lo=lo, mel_hi=hi) for r in (0, 3, 6, 299)}
    inv_alone = {r: eng.istft(alone[r]["stft"], n_fft, hop, w, length=T) for r in alone}
    for rows in (1, 7, 300):
        out = eng.spectral(x[:rows], n_fft, hop, w, mel_fb=fb, mel_lo=lo, mel_hi=hi)
        inv = eng.istft(out["stft"], n_fft, hop, w, length=T)
        for r in alone:
            if r < rows:
                assert torch.equal(out["stft"][r:r + 1], alone[r]["stft"]), (n_fft, rows, r)
                assert torch.equal(out["mel"][r:r + 1], alone[r]["mel"]), (n_fft, rows, r)
                assert torch.equal(inv[r:r + 1], inv_alone[r]), (n_fft, rows, r)


@pytest.mark.parametrize("n_fft", [32, 64, 256, 1024, 2048, 4096, 8192, 400])
def test_frame_shift_is_exact(eng, n_fft):
    """The interior frames of x and of x delayed by s hop are identical (STFT and mel): a frame's arithmetic does not
    depend on its slot in a tile."""
    from audiotools_b200 import AudioSignal

    hop = n_fft // 4
    T = 40 * hop + n_fft if n_fft <= 4096 else 12 * hop + n_fft
    x = torch.randn(1, 1, T, generator=torch.Generator().manual_seed(n_fft)).to(DEV)
    fb, lo, hi = AudioSignal._mel_tables(16000, n_fft, 40 if n_fft >= 256 else 5, 0.0, None, DEV)
    w = s64.windows(n_fft, DEV)["hann"]
    a = eng.spectral(x, n_fft, hop, w, mel_fb=fb, mel_lo=lo, mel_hi=hi)
    edge = n_fft // hop  # frames that read the padding
    for s in (1, 3, 7):
        xs = torch.cat([torch.randn(1, 1, s * hop, device=DEV), x], -1)
        b = eng.spectral(xs, n_fft, hop, w, mel_fb=fb, mel_lo=lo, mel_hi=hi)
        N = a["stft"].shape[-1]
        assert torch.equal(b["stft"][..., s + edge:s + N - edge], a["stft"][..., edge:N - edge]), (n_fft, s)
        assert torch.equal(b["mel"][..., s + edge:s + N - edge], a["mel"][..., edge:N - edge]), (n_fft, s)


@pytest.mark.parametrize("n_fft", [64, 128, 256, 512, 1024, 2048])
def test_warp_kernel_modes_agree(eng, n_fft):
    """spectral_warp_kernel's modes 0 (mel), 1 (STFT) and 2 (both) give bit-identical mel and STFT."""
    from audiotools_b200 import AudioSignal

    hop = n_fft // 4
    x = torch.randn(3, 2, 37 * hop + 11, generator=torch.Generator().manual_seed(n_fft)).to(DEV)
    fb, lo, hi = AudioSignal._mel_tables(44100, n_fft, 80, 0.0, None, DEV)
    w = s64.windows(n_fft, DEV)["hann"]
    k = int(math.log2(n_fft)) - 1
    assert eng.spectral_kernel_name(n_fft, hop, True, True) == f"spectral_warp_kernel<{k},2>"
    m0 = eng.spectral(x, n_fft, hop, w, mel_fb=fb, mel_lo=lo, mel_hi=hi, want_stft=False)
    s1 = eng.spectral(x, n_fft, hop, w)
    b2 = eng.spectral(x, n_fft, hop, w, mel_fb=fb, mel_lo=lo, mel_hi=hi, want_stft=True)
    assert torch.equal(m0["mel"], b2["mel"]) and torch.equal(s1["stft"], b2["stft"]), n_fft
