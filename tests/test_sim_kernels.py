"""The product's kernel SOURCES, compiled for the CPU by tests/cusim (CUDA threads -> host
threads), against the oracle.  This checks indexing and arithmetic of the exact code that ships
before it ever reaches a GPU; the GPU parity tests proper are tests/test_gpu_parity.py.
Sizes are small: every CUDA thread is a host thread here."""
import numpy as np
import pytest
import torch

from audiotools_b200 import _lib
from audiotools_b200.core import mel as melmod
from oracle import signal_path as sp
from tests.conftest import rel_err
from tests.cusim.sim_engine import sim_engine
from tests.golden import cases


@pytest.fixture(scope="module")
def eng():
    return sim_engine()


def padded_len(T, sr):
    return T + int((0.5 - T / sr) * sr) if T / sr < 0.5 else T


@pytest.mark.parametrize("name", ["short", "lufs48k", "lufs11k", "cfg2"])
def test_lufs_blocks_and_gating(eng, golden, name):
    x, sr = cases.make_input(name), cases.sample_rate(name)
    T = x.shape[-1]
    out = eng.lufs(x, sr, padded_length=padded_len(T, sr), target_db=torch.tensor([-24.0]), want_blocks=True)
    z_ref = sp.Meter(sr).block_energies(torch.nn.functional.pad(x, (0, padded_len(T, sr) - T)).permute(0, 2, 1))
    assert out["blocks"].shape == z_ref.shape  # block indexing is bit-exact
    assert rel_err(out["blocks"], z_ref) < 1e-4
    ref = torch.from_numpy(golden["cfg2_lufs" if name == "cfg2" else {"short": "lufs_short"}.get(name, name)])
    assert torch.allclose(out["loud"], ref, atol=1e-3)  # dB; 1e-4 relative of a ~-20 LUFS value is 2e-3
    if name == "cfg2":
        assert out["lufs"][1].item() == float("-inf") and out["loud"][1].item() == -70.0
        assert rel_err(z_ref * 0 + torch.from_numpy(golden["cfg2_z"]), z_ref) < 1e-6
    gain_ref = torch.exp((torch.tensor(-24.0) - ref) * sp.GAIN_FACTOR)
    assert torch.allclose(out["gain"], gain_ref, rtol=1e-4)


def test_lufs_single_stage_and_errors(eng):
    x = cases.make_input("short")
    with pytest.raises(NotImplementedError):
        eng.lufs(x, 16000, filter_class="Fenton/Lee 1")
    with pytest.raises(_lib.B2AError, match="unsupported geometry"):
        eng.lufs(x, 500)  # gating stride would be < 64 samples


@pytest.mark.parametrize("n_fft,hop,wtype,match_stride,T", [
    (512, 128, "hann", False, 16000),        # BASELINE cfg1
    (256, 64, "sqrt_hann", True, 16000),     # match_stride, T % hop == 0
    (256, 64, "hann", True, 15999),          # match_stride with right_pad
    (2048, 512, "hann", False, 16000),       # cfg2 transform size
    (64, 16, "hann", False, 3000),
    (1024, 256, "hann", False, 9000),
    (256, 77, "average", False, 5000),       # odd hop, non-hann window
    (4096, 1024, "hann", False, 16000),
])
def test_stft_vs_torch_stft(eng, n_fft, hop, wtype, match_stride, T):
    x = cases.make_input("cfg1")[:2, :, :T]
    right_pad, pad = sp.compute_stft_padding(T, n_fft, hop, match_stride)
    out = eng.spectral(x, n_fft, hop, sp.get_window(wtype, n_fft), pad=pad, right_pad=right_pad,
                       drop_edge=2 if match_stride else 0)["stft"]
    ref = sp.stft(x, 16000, n_fft, hop, wtype, match_stride, "reflect")
    assert out.shape == ref.shape  # frame indexing is bit-exact
    assert rel_err(torch.view_as_real(out), torch.view_as_real(ref)) < 1e-5


def test_cfg1_against_reference_golden(eng, golden):
    x = cases.make_input("cfg1")
    out = eng.spectral(x, 512, 128, sp.get_window("hann", 512))["stft"]
    ref = torch.from_numpy(golden["cfg1_stft"])
    assert out.shape == ref.shape == (4, 1, 257, 126)
    assert rel_err(torch.view_as_real(out), torch.view_as_real(ref)) < 1e-5


@pytest.mark.parametrize("mode", ["constant", "replicate"])
def test_stft_other_padding_types(eng, mode):
    x = cases.make_input("cfg1")[:1, :, :4000]
    right_pad, pad = sp.compute_stft_padding(4000, 256, 64, True)
    out = eng.spectral(x, 256, 64, sp.get_window("hann", 256), pad=pad, right_pad=right_pad, pad_mode=mode,
                       drop_edge=2)["stft"]
    ref = sp.stft(x, 16000, 256, 64, "hann", True, mode)
    assert out.shape == ref.shape and rel_err(torch.view_as_real(out), torch.view_as_real(ref)) < 1e-5


def _mel_tables(sr, n_fft, n_mels, fmin=0.0, fmax=None):
    fb = melmod.mel_filters(sr, n_fft, n_mels, fmin, fmax)
    lo, hi = melmod.band_table(fb)
    return torch.from_numpy(np.array(fb)), torch.from_numpy(lo), torch.from_numpy(hi)


def test_fused_normalize_logmel_cfg2_golden(eng, golden):
    """normalize(-24) -> log-mel(2048/512/128) in two launches, against the real reference."""
    x, sr = cases.make_input("cfg2"), 44100
    lu = eng.lufs(x, sr, target_db=torch.tensor([-24.0]))
    fb, lo, hi = _mel_tables(sr, 2048, 128)
    out = eng.spectral(x, 2048, 512, sp.get_window("hann", 2048), gain=lu["gain"], want_scaled=True, mel_fb=fb,
                       mel_lo=lo, mel_hi=hi, post=_lib.POST_LOG10, post_eps=1e-5, post_power=2.0, want_stft=False)
    assert rel_err(out["scaled"], torch.from_numpy(golden["cfg2_norm"])) < 1e-4
    assert out["mel"].shape == golden["cfg2_logmel"].shape
    assert rel_err(out["mel"], torch.from_numpy(golden["cfg2_logmel"])) < 1e-4
    plain = eng.spectral(x, 2048, 512, sp.get_window("hann", 2048), mel_fb=fb, mel_lo=lo, mel_hi=hi, want_stft=False)
    ref = sp.mel_spectrogram(x, sr, 128, window_length=2048, hop_length=512, window_type="hann")
    assert rel_err(plain["mel"], ref) < 1e-5
    assert eng.gain(x, lu["gain"]).equal(out["scaled"])


def test_mel_variants_golden(eng, golden):
    x = cases.make_input("cfg1")
    fb, lo, hi = _mel_tables(16000, 512, 80)
    mel = eng.spectral(x, 512, 128, sp.get_window("hann", 512), mel_fb=fb, mel_lo=lo, mel_hi=hi, want_stft=False)["mel"]
    assert rel_err(mel, torch.from_numpy(golden["cfg1_mel80"])) < 1e-5
    fb, lo, hi = _mel_tables(16000, 1024, 40, 100.0, 6000.0)
    mel = eng.spectral(x[:2], 1024, 256, sp.get_window("hann", 1024), mel_fb=fb, mel_lo=lo, mel_hi=hi,
                       want_stft=False)["mel"]
    assert rel_err(mel, torch.from_numpy(golden["cfg1_mel40_fmin_fmax"])) < 1e-5


def test_spectral_modes_agree(eng, golden):
    """The warp kernel has three instantiations (mel only / staged STFT only / STFT + mel straight from registers):
    the same launch parameters must give the same numbers whichever one serves them, with and without a gain."""
    x = cases.make_input("cfg1")
    w = sp.get_window("hann", 512)
    fb, lo, hi = _mel_tables(16000, 512, 80)
    gain = torch.tensor([0.5, 2.0, 1.0, 0.25])
    for g in (None, gain):
        both = eng.spectral(x, 512, 128, w, gain=g, mel_fb=fb, mel_lo=lo, mel_hi=hi, want_stft=True)     # mode 2
        mel = eng.spectral(x, 512, 128, w, gain=g, mel_fb=fb, mel_lo=lo, mel_hi=hi, want_stft=False)     # mode 0
        stft = eng.spectral(x, 512, 128, w, gain=g, want_stft=True)                                      # mode 1
        assert torch.equal(both["mel"], mel["mel"])
        assert torch.equal(both["stft"], stft["stft"])
        scale = 1.0 if g is None else g[:, None, None, None]
        assert rel_err(torch.view_as_real(stft["stft"]), torch.view_as_real(torch.from_numpy(golden["cfg1_stft"]) * scale)) < 1e-5
    # odd hop (scalar load path), window 256 / hop 100, all three modes
    w2 = sp.get_window("average", 256)
    a = eng.spectral(x[:2], 256, 100, w2, want_stft=True)["stft"]
    assert rel_err(torch.view_as_real(a), torch.view_as_real(torch.from_numpy(golden["cfg1_stft_average_hop100"]))) < 1e-5
    fb2, lo2, hi2 = _mel_tables(16000, 256, 20)
    b = eng.spectral(x[:2], 256, 100, w2, mel_fb=fb2, mel_lo=lo2, mel_hi=hi2, want_stft=True)
    assert torch.equal(b["stft"], a)
    assert torch.equal(b["mel"], eng.spectral(x[:2], 256, 100, w2, mel_fb=fb2, mel_lo=lo2, mel_hi=hi2, want_stft=False)["mel"])


def test_fft_kernels_random_geometries(eng):
    """The fused FFT kernels (window lengths 32 .. 4096, incl. the lean-twiddle N = 1024 case) at random hops, lengths,
    padding modes, per-item gains and mel sizes against torch.stft + the reference's |X| @ fb.T: frame counts exactly,
    STFT to 2e-6 of the tensor maximum, mel to 1e-5, the scaled waveform exactly x * gain."""
    rng = np.random.RandomState(7)
    for it in range(14):
        n_fft = int(rng.choice([32, 64, 128, 256, 512, 1024, 2048, 2048, 4096]))
        hop = int(rng.choice([n_fft // 4, n_fft // 2, n_fft, max(1, n_fft // 8), int(rng.randint(max(1, n_fft // 16), n_fft + 1))]))
        T = int(rng.randint(n_fft // 2 + 1, 5 * n_fft + 300))
        mode = ["reflect", "constant", "replicate"][it % 3]
        B, C = int(rng.randint(1, 3)), int(rng.randint(1, 3))
        g = torch.Generator().manual_seed(100 + it)
        x = torch.randn(B, C, T, generator=g)
        w = torch.hann_window(n_fft) + 0.05 + 0.1 * torch.rand(n_fft, generator=g)
        gain = 0.25 + torch.rand(B, generator=g)
        n_mels = int(rng.choice([8, 20, 40]))
        fb, lo, hi = _mel_tables(16000, n_fft, n_mels)
        out = eng.spectral(x, n_fft, hop, w, pad_mode=mode, gain=gain, want_scaled=True, mel_fb=fb, mel_lo=lo, mel_hi=hi,
                           want_stft=True)
        xs = x * gain[:, None, None]
        ref = torch.stft(xs.reshape(B * C, T), n_fft, hop, window=w, center=True, return_complex=True)
        ref = ref.reshape(B, C, *ref.shape[1:])
        assert out["stft"].shape == ref.shape, (n_fft, hop, T)
        assert torch.equal(out["scaled"], xs)
        assert rel_err(torch.view_as_real(out["stft"]), torch.view_as_real(ref)) < 2e-6, (n_fft, hop, T, mode)
        mel_ref = (ref.abs().transpose(2, 3) @ fb.T).transpose(2, 3)
        assert rel_err(out["mel"], mel_ref) < 1e-5, (n_fft, hop, T, n_mels)


def test_istft_random_geometries(eng):
    """Random (n_fft, hop, frames, length) against torch.istft: segment boundaries, warm-up, carries, tail fill."""
    rng = np.random.RandomState(0)
    for it in range(14):
        n_fft = int(rng.choice([64, 128, 256, 512, 1024, 2048]))
        hop = int(rng.choice([n_fft // 4, n_fft // 2, n_fft, n_fft // 8, max(1, n_fft // 3),
                              int(rng.randint(max(4, n_fft // 8), n_fft + 1))]))
        rows, nfr = int(rng.randint(1, 4)), int(rng.randint(1, 40))
        T = max((nfr - 1) * hop, n_fft // 2 + 1 + 3 * hop)
        g = torch.Generator().manual_seed(it)
        w = torch.hann_window(n_fft) + 0.05 + 0.1 * torch.rand(n_fft, generator=g)
        X = torch.stft(torch.randn(rows, max(T, n_fft), generator=g), n_fft, hop, window=w, center=True, return_complex=True)
        X = X * (1 + 0.2 * torch.randn(X.shape, generator=g))
        length = int(rng.randint(1, (X.shape[-1] - 1) * hop + n_fft // 2 + 1))
        ref = torch.istft(X, n_fft, hop, window=w, center=True, length=length)
        out = eng.istft(X[:, None].contiguous(), n_fft, hop, w, length)[:, 0]
        keep = max(1, length - 2 * hop)  # the envelope -> 0 at the very end amplifies rounding
        assert rel_err(out[..., :keep], ref[..., :keep]) < 5e-5, (n_fft, hop, rows, X.shape[-1], length)


# ------------------------------------------------------------------------------------------
# dense DFT path (csrc/dft.cu): any window length, forward (+ mel from the materialised STFT) and inverse
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_fft,hop,T,pad_mode", [(400, 160, 3000, "reflect"), (96, 31, 1000, "constant"),
                                                  (201, 50, 1500, "replicate"), (30, 7, 400, "reflect"),
                                                  (480, 120, 4000, "reflect"), (1200, 300, 6000, "constant"),
                                                  (1001, 250, 5000, "replicate")])
def test_dense_dft_any_window_length(eng, n_fft, hop, T, pad_mode):
    g = torch.Generator().manual_seed(n_fft)
    x = torch.randn(2, 2, T, generator=g)
    w = torch.hann_window(n_fft) + 0.05 + 0.1 * torch.rand(n_fft, generator=g)
    out = eng.spectral(x, n_fft, hop, w, pad_mode=pad_mode)
    ref = torch.stft(x.reshape(4, T), n_fft, hop, window=w, center=True, return_complex=True).reshape(2, 2, n_fft // 2 + 1, -1)
    assert out["stft"].shape == ref.shape  # frame indexing exact
    assert rel_err(torch.view_as_real(out["stft"]), torch.view_as_real(ref)) < 2e-6
    # match_stride-style call: explicit F.pad + dropped edge frames, resolved per sample inside the kernel
    pad, right_pad = (n_fft - hop) // 2, (-T) % hop
    xp = torch.nn.functional.pad(x, (pad, pad + right_pad), pad_mode)
    ref2 = torch.stft(xp.reshape(4, -1), n_fft, hop, window=w, center=True, return_complex=True)[..., 2:-2]
    out2 = eng.spectral(x, n_fft, hop, w, pad=pad, right_pad=right_pad, pad_mode=pad_mode, drop_edge=2)["stft"]
    assert out2.shape[-1] == ref2.shape[-1] and rel_err(torch.view_as_real(out2.reshape(4, *ref2.shape[1:])), torch.view_as_real(ref2)) < 2e-6
    # mel from the materialised STFT, with a gain riding along
    fb, lo, hi = _mel_tables(16000, n_fft, 20)
    gain = torch.tensor([0.5, 2.0])
    m = eng.spectral(x, n_fft, hop, w, pad_mode=pad_mode, gain=gain, want_scaled=True, mel_fb=fb, mel_lo=lo, mel_hi=hi,
                     post=_lib.POST_LOG10, post_eps=1e-5, post_power=2.0, want_stft=False)
    assert m["stft"] is None and torch.equal(m["scaled"], x * gain[:, None, None])
    mel_ref = torch.log10(((ref.abs() * gain[:, None, None, None]).transpose(2, 3) @ fb.T).transpose(2, 3).clamp(1e-5) ** 2)
    assert (m["mel"] - mel_ref).abs().max() < 1e-4
    # inverse: dense transposed product + fold
    length = T
    y = eng.istft(out["stft"], n_fft, hop, w, length)
    y_ref = torch.istft(ref.reshape(4, *ref.shape[2:]), n_fft, hop, window=w, center=True, length=length).reshape(2, 2, -1)
    assert y.shape == y_ref.shape and rel_err(y, y_ref) < 5e-5


def test_dense_dft_random_geometries(eng):
    """Random (window length, hop, length, padding) on the dense path against torch.stft / torch.istft: tile edges of the
    64 x 64 x 16 product (lengths around the multiples), hop > window, single-frame signals, odd everything."""
    rng = np.random.RandomState(1)
    for it in range(12):
        n_fft = int(rng.choice([2, 3, 17, 63, 65, 100, 127, 129, 250, 513, 600, 777]))
        hop = int(rng.choice([1, max(1, n_fft // 4), max(1, n_fft // 2), n_fft, n_fft + 3, int(rng.randint(1, n_fft + 1))]))
        hop = max(hop, n_fft // 64 + 1)  # keep the frame count (CPU time) bounded
        T = int(rng.randint(n_fft // 2 + 1, 6 * n_fft + 200))
        mode = ["reflect", "constant", "replicate"][it % 3]
        g = torch.Generator().manual_seed(it)
        x = torch.randn(2, 1, T, generator=g)
        w = torch.hann_window(n_fft) + 0.05 + 0.1 * torch.rand(n_fft, generator=g) if n_fft > 2 else torch.ones(n_fft)
        out = eng.spectral(x, n_fft, hop, w, pad_mode=mode)["stft"]
        ref = torch.stft(x.reshape(2, T), n_fft, hop, window=w, center=True, return_complex=True)
        assert out.shape[2:] == ref.shape[1:], (n_fft, hop, T)
        assert rel_err(torch.view_as_real(out[:, 0]), torch.view_as_real(ref)) < 5e-6, (n_fft, hop, T)
        if hop <= n_fft and (hop <= n_fft // 2 or n_fft <= 3):  # the envelope does not vanish
            length = int(rng.randint(1, T + 1))
            try:
                y_ref = torch.istft(ref, n_fft, hop, window=w, center=True, length=length)
            except RuntimeError:
                continue
            y = eng.istft(out, n_fft, hop, w, length)[:, 0]
            keep = max(1, length - 2 * hop)
            assert rel_err(y[..., :keep], y_ref[..., :keep]) < 1e-4, (n_fft, hop, T, length)


def test_bypass_flags_and_batch1_impulse_response(eng):
    """The per-filter bypass flags of fir_direct / fftconv / circconv copy the flagged rows through EXACTLY and leave the
    others bit-identical to the un-flagged launch; a batch-1 impulse response is shared by every item (the reference's
    broadcasting product, ref:audiotools/core/effects.py:106-114)."""
    g = torch.Generator().manual_seed(2)
    x = torch.randn(3, 2, 5000, generator=g)
    byp = torch.tensor([False, True, False])
    cut = torch.tensor([3000.0, 5000.0, 7000.0])
    for zeros, hp in ((51, False), (51, True), (600, False)):  # 137 taps: direct kernel; 1601 taps: FFT engine
        full = eng.sinc_filter(x, cut, 16000, zeros, highpass=hp)
        part = eng.sinc_filter(x, cut, 16000, zeros, highpass=hp, bypass=byp)
        assert torch.equal(part[1], x[1])
        assert (part[[0, 2]] - full[[0, 2]]).abs().max() <= 2e-6 * full.abs().max()  # (the bank is sized by the selected items)
    db = -torch.rand(3, 6, generator=g)
    full, part = eng.equalizer(x, 16000, db), eng.equalizer(x, 16000, db, bypass=byp)
    assert torch.equal(part[1], x[1]) and torch.equal(part[[0, 2]], full[[0, 2]])
    ir = torch.randn(3, 1, 700, generator=g) * torch.exp(-torch.arange(700) / 90.0)
    full, part = eng.circular_convolve(x, ir), eng.circular_convolve(x, ir, bypass=byp)
    assert torch.equal(part[1], x[1]) and torch.equal(part[[0, 2]], full[[0, 2]])
    one = eng.circular_convolve(x, ir[:1])  # batch-1 impulse response -> every item
    assert rel_err(one, sp.convolve(x, ir[:1].expand(3, -1, -1))) < 1e-5
    assert torch.equal(one, eng.circular_convolve(x, ir[:1].expand(3, -1, -1).contiguous()))


def test_alter_drr_multichannel_vs_oracle(eng):
    """b2a_alter_drr_f32 (one launch) against the oracle's restatement of decompose_ir / solve_alpha / alter_drr
    (ref:audiotools/core/effects.py:540-647): stereo impulse responses whose channels peak at different samples (the
    window is channel 0's early region for every channel), per-item targets, a response that needs the peak limit."""
    g = torch.Generator().manual_seed(5)
    sr, T = 16000, 6000
    t = torch.arange(T) / sr
    ir = 0.05 * torch.randn(3, 2, T, generator=g) * torch.exp(-t / 0.05)
    ir[0, 0, 40] = 1.0; ir[0, 1, 55] = 0.9      # channel 1's direct path 15 samples later: inside channel 0's window
    ir[1, 0, 200] = 0.7; ir[1, 1, 300] = 0.8    # ... and 100 samples later: outside it
    ir[2, 0, 10] = 2.5; ir[2, 1, 10] = -0.2     # peak > 1 after re-weighting; channel 1's maximum is elsewhere
    drr = torch.tensor([5.0, 20.0, -3.0])
    out = eng.alter_drr(ir, sr, drr)
    ref = sp.alter_drr(ir.clone(), sr, drr)
    assert out.shape == ref.shape
    # a channel whose early region misses channel 0's window has a = 0 in the quadratic: the reference's row is NaN
    assert torch.isnan(ref[1, 1]).all() and torch.isnan(ref[2, 1]).all()
    assert torch.equal(torch.isnan(out), torch.isnan(ref))
    ok = ~torch.isnan(ref)
    assert (out[ok] - ref[ok]).abs().max() < 1e-6


def test_mfcc_dct_kernel(eng):
    g = torch.Generator().manual_seed(1)
    logmel = torch.randn(2, 2, 80, 37, generator=g)
    dct = torch.randn(80, 40, generator=g)
    out = eng.mel_dct(logmel, dct)
    ref = (logmel.transpose(-1, -2) @ dct).transpose(-1, -2)
    assert out.shape == ref.shape == (2, 2, 40, 37) and rel_err(out, ref) < 1e-6
    out = eng.mel_dct(logmel[..., :5], dct[:, :33])  # a coefficient count that is not a multiple of the register tile
    assert rel_err(out, (logmel[..., :5].transpose(-1, -2) @ dct[:, :33]).transpose(-1, -2)) < 1e-6


# ------------------------------------------------------------------------------------------
# FIR / convolution / resample / pitch (csrc/fftconv.cu, resample.cu, pitch.cu)
# ------------------------------------------------------------------------------------------
def test_sinc_filters_and_equalizer_golden(eng, golden):
    x, sr = cases.make_input("fir"), 44100
    cut = torch.from_numpy(golden["fir_cut"])
    assert rel_err(eng.sinc_filter(x, cut, sr, 51, False), torch.from_numpy(golden["lp_peritem"])) < 1e-5
    assert rel_err(eng.sinc_filter(x, cut / 8, sr, 51, True), torch.from_numpy(golden["hp_peritem"])) < 1e-5
    assert rel_err(eng.sinc_filter(x, torch.tensor(4000), sr, 51, False), torch.from_numpy(golden["lp_scalar"])) < 1e-5
    assert rel_err(eng.equalizer(x, sr, golden["eq_db"]), torch.from_numpy(golden["eq_out"])) < 1e-5
    assert rel_err(eng.equalizer(x, sr, golden["eq_db"][0]), torch.from_numpy(golden["eq_out_1d"])) < 1e-5
    fb = eng.mel_filterbank(x[:1, :1], sr, 4)
    assert fb.shape == (1, 1, 12000, 4) and rel_err(fb, torch.from_numpy(golden["fbank4"])) < 1e-5
    with pytest.raises(ValueError):
        eng.sinc_filter(x, torch.tensor(30000.0), sr)


def test_circular_convolution_golden(eng, golden):
    x, ir = cases.make_input("fir"), cases.make_ir()
    assert rel_err(eng.circular_convolve(x, ir, True), torch.from_numpy(golden["conv_out"])) < 1e-5
    assert rel_err(eng.circular_convolve(x, ir, False), torch.from_numpy(golden["conv_out_nomax"])) < 1e-5
    for delay in (0, 777):  # ref:tests/core/test_effects.py:86-121: a delta IR is the identity
        d = torch.zeros(3, 1, 1000)
        d[..., delay] = 1.0
        assert torch.allclose(eng.circular_convolve(x, d, True), x, atol=1e-6)


@pytest.mark.parametrize("key,sl,old,new", [("rs_48k_16k", 24000, 48000, 16000), ("rs_44k_16k", 22050, 44100, 16000),
                                            ("rs_16k_44k", 8000, 16000, 44100), ("rs_16k_48k", 8001, 16000, 48000),
                                            ("rs_44k_48k", 4410, 44100, 48000)])
def test_resample_golden(eng, golden, key, sl, old, new):
    x = cases.make_input("rs")[..., :sl]
    y = eng.resample(x, old, new)
    ref = torch.from_numpy(golden[key])
    assert y.shape == ref.shape  # floor(new*T/old), bit-exact
    assert rel_err(y, ref) < 1e-5


def test_pitch_shift_properties(eng):
    sr, T = 16000, 12000
    t = torch.arange(T) / sr
    x = torch.stack([0.5 * torch.sin(2 * np.pi * 440 * t), 0.3 * torch.sin(2 * np.pi * 1000 * t)])[:, None, :]
    for st in (3, -2, 12):
        y = eng.pitch_shift(x, sr, st)
        assert y.shape == x.shape  # length preserved exactly
        for i, f0 in enumerate((440.0, 1000.0)):
            spec = torch.fft.rfft(y[i, 0] * torch.hann_window(T)).abs()
            assert abs(spec.argmax().item() * sr / T - f0 * 2 ** (st / 12)) < 4.0  # pitch ratio 2^(n/12)
        assert torch.equal(eng.pitch_shift(x[:1], sr, st), y[:1])  # batch == per-item
        # amplitude is preserved and the output is (up to WSOLA's splice jitter) the shifted sinusoid
        n = np.arange(T) / sr
        f = 440.0 * 2 ** (st / 12)
        A = np.stack([np.sin(2 * np.pi * f * n), np.cos(2 * np.pi * f * n)], 1)[1500:-1500]
        coef = np.linalg.lstsq(A, y[0, 0, 1500:-1500].double().numpy(), rcond=None)[0]
        assert abs(np.hypot(*coef) - 0.5) < 0.01
        assert (y[0, 0, 1500:-1500].double().numpy() - A @ coef).std() < 0.06 * 0.5
    assert torch.equal(eng.pitch_shift(x, sr, 0), x)
    # several shifts in one launch == each group on its own; a shift of 0 copies the item bit for bit
    xm = torch.cat([x, x.flip(0)], 0)  # 4 items
    ym = eng.pitch_shift(xm, sr, [3.0, 0.0, -2.0, 3.0])
    assert torch.equal(ym[[0, 3]], eng.pitch_shift(xm[[0, 3]], sr, 3.0))
    assert torch.equal(ym[2:3], eng.pitch_shift(xm[2:3], sr, -2.0))
    assert torch.equal(ym[1], xm[1])
    stereo = eng.pitch_shift(xm.reshape(2, 2, -1), sr, [3.0, -2.0])  # group per item, both channels of an item together
    assert torch.equal(stereo[0], eng.pitch_shift(xm[:2].reshape(1, 2, -1), sr, 3.0)[0])
    assert torch.equal(stereo[1], eng.pitch_shift(xm[2:].reshape(1, 2, -1), sr, -2.0)[0])
    # overlap-add windows and interpolation weights both sum to one: a constant stays that constant
    dc = torch.full((1, 1, 9000), 0.25)
    for st in (2, -5):
        y = eng.pitch_shift(dc, 8000, st)
        assert torch.allclose(y[..., 600:-1200], dc[..., 600:-1200], atol=2e-6)


def test_direct_fir_paths(eng, golden):
    """Short filters take the time-domain kernel (csrc/fir.cu): cfg3's low_pass(8k)@16k (103 taps) after the
    single-phase 48k->16k resample (also fir.cu), per-item high-pass (x - y), zero vs replicate padding."""
    x = cases.make_input("rs")
    y = eng.resample(x, 48000, 16000)
    assert rel_err(y, torch.from_numpy(golden["rs_48k_16k"])) < 1e-5
    z = eng.sinc_filter(y, torch.tensor(8000.0), 16000, 51, False)
    assert rel_err(z, torch.from_numpy(golden["rs_48k_16k_lp8k"])) < 1e-5
    xs = cases.make_input("short")  # [2,1,4000] @16k
    cut = torch.tensor([4000.0, 2500.0])
    hp = eng.sinc_filter(xs, cut, 16000, 51, True)
    assert rel_err(hp, sp.high_pass(xs, 16000, cut)) < 1e-5
    lp = eng.sinc_filter(xs, cut, 16000, 51, False)
    assert rel_err(lp, sp.low_pass(xs, 16000, cut)) < 1e-5
    taps = torch.randn(1, 37)
    out = eng.fir_direct(xs, taps, rows_per_filt=2, left0=5, stride=2, out_len=1990, pad_mode="constant")
    ref = torch.nn.functional.conv1d(torch.nn.functional.pad(xs.reshape(2, 1, -1), (5, 40)), taps[None], stride=2)[..., :1990]
    assert rel_err(out, ref.reshape(2, 1, -1)) < 1e-5


# ------------------------------------------------------------------------------------------
# inverse STFT (csrc/istft.cu) against torch.istft
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_fft,hop,T,wtype", [(2048, 512, 30000, "hann"), (512, 128, 9000, "sqrt_hann"),
                                               (256, 64, 5000, "sqrt_hann"), (64, 16, 3000, "hann"),
                                               (1024, 300, 12000, "hann"), (128, 128, 4000, "boxcar"),
                                               (512, 37, 3000, "hann")])
def test_istft_matches_torch(eng, n_fft, hop, T, wtype):
    from scipy import signal as ss

    g = torch.Generator().manual_seed(n_fft + hop)
    x = torch.randn(3, T, generator=g)
    w = ss.get_window("hann" if wtype == "sqrt_hann" else wtype, n_fft)
    w = torch.from_numpy(np.sqrt(w) if wtype == "sqrt_hann" else w).float()
    X = torch.stft(x, n_fft, hop, window=w, center=True, return_complex=True)
    X = X + 0.01 * torch.randn(X.shape, generator=g)  # not a consistent STFT any more: exercises the plain OLA
    X[:, 0] = X[:, 0] + 0.5j  # imaginary parts of DC / Nyquist must be ignored (C2R semantics)
    X[:, -1] = X[:, -1] - 0.25j
    for length in (T, T - 77, (X.shape[-1] - 1) * hop):
        ref = torch.istft(X, n_fft, hop, window=w, center=True, length=length)
        out = eng.istft(X.reshape(3, 1, *X.shape[1:]), n_fft, hop, w, length)
        assert out.shape == (3, 1, length)
        assert rel_err(out[:, 0], ref) < 2e-5, (n_fft, hop, length)
    # match_stride handling of the reference: 2 zero frames back on either side, trim `pad` samples in front
    Xp = torch.nn.functional.pad(X, (2, 2))
    pad, length = (n_fft - hop) // 2, T - 100
    if (Xp.shape[-1] - 1) * hop + n_fft >= n_fft // 2 + pad + length:
        ref = torch.istft(Xp, n_fft, hop, window=w, center=True, length=length + 2 * pad)[..., pad:pad + length]
        out = eng.istft(X.reshape(3, 1, *X.shape[1:]), n_fft, hop, w, length, pad_frames=2, trim=pad)
        assert rel_err(out[:, 0], ref) < 2e-5


def test_istft_zero_tail_and_envelope_check(eng):
    n_fft, hop = 256, 64
    w = torch.hann_window(n_fft)
    X = torch.stft(torch.randn(1, 2000, generator=torch.Generator().manual_seed(3)), n_fft, hop, window=w,
                   center=True, return_complex=True)
    expected = (X.shape[-1] - 1) * hop + n_fft
    length = expected - n_fft // 2 + 333  # torch pads with zeros beyond the overlap-add's support
    out = eng.istft(X[:, None], n_fft, hop, w, length)
    assert torch.count_nonzero(out[..., expected - n_fft // 2:]) == 0
    ref = torch.istft(X, n_fft, hop, window=w, center=True, length=expected - n_fft // 2 - 1)
    assert rel_err(out[0, :, : ref.shape[-1] - 16], ref[..., :-16]) < 2e-5
    assert rel_err(out[0, :, : ref.shape[-1]], ref) < 1e-4  # the envelope -> 0 at the very end amplifies rounding
    with pytest.raises(RuntimeError):  # a window that vanishes inside the kept range (torch: "window overlap add min")
        wz = w.clone()
        wz[: n_fft // 2 + 10] = 0
        eng.istft(X[:, None], n_fft, n_fft, wz, 1500)
    with pytest.raises(NotImplementedError):  # (32 and 4096 run on the dense path now; 8192 is its limit)
        eng.istft(torch.zeros(1, 1, 5001, 5, dtype=torch.complex64), 10000, 2500, torch.ones(10000), 4096)


# ------------------------------------------------------------------------------------------
# one-sided peer exchange (csrc/peer.cu): two "ranks" in one process, buffers in host memory
# ------------------------------------------------------------------------------------------
def _peer_setup(lib, world, n_max):
    import ctypes

    bufs, peers = [], (ctypes.c_void_p * world)()
    for r in range(world):
        p, h = ctypes.c_void_p(), (ctypes.c_ubyte * 64)()
        lib.check(lib.b2a_peer_buffer_create(world, n_max, ctypes.byref(p), h))
        q = ctypes.c_void_p()
        lib.check(lib.b2a_peer_buffer_open(h, ctypes.byref(q)))
        assert q.value == p.value
        bufs.append(p.value)
        peers[r] = p.value
    return bufs, peers


def test_peer_put_collect_two_ranks(eng):
    import ctypes

    lib, world, n_max = eng.lib, 2, 8
    assert lib.b2a_peer_buffer_bytes(world, n_max) == (4 * world * n_max + 4 * world + 4) * 4
    assert lib.b2a_peer_buffer_bytes(17, 8) == 0
    bufs, peers = _peer_setup(lib, world, n_max)
    vals = {r: [torch.arange(5, dtype=torch.float32) + 10 * r + 100 * s for s in range(1, 7)] for r in range(world)}
    for s in range(1, 7):  # six steps: every slot, and a reuse of the first two
        for r in range(world):
            v = vals[r][s - 1]
            lib.check(lib.b2a_peer_put_f32(ctypes.c_void_p(v.data_ptr()), 5, peers, world, r, n_max, s, None))
        for r in range(world):
            out, seqs = torch.empty(world * 5), torch.zeros(world, dtype=torch.int32)
            lib.check(lib.b2a_peer_collect_f32(ctypes.c_void_p(bufs[r]), world, 5, n_max, s,
                                               ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(seqs.data_ptr()), None))
            assert torch.equal(out, torch.cat([vals[0][s - 1], vals[1][s - 1]]))
            assert seqs.tolist() == [s, s]
            out2 = torch.empty(world, 5)
            lib.check(lib.b2a_peer_latest_f32(ctypes.c_void_p(bufs[r]), world, 5, n_max,
                                              ctypes.c_void_p(out2.data_ptr()), ctypes.c_void_p(seqs.data_ptr()), None))
            assert torch.equal(out2.reshape(-1), out) and seqs.tolist() == [s, s]
    assert lib.b2a_peer_put_f32(None, 5, peers, world, 0, n_max, 1, None) != 0  # null source is refused
    st = torch.full((1,), -1, dtype=torch.int32)
    lib.check(lib.b2a_peer_status(ctypes.c_void_p(bufs[0]), world, n_max, ctypes.c_void_p(st.data_ptr()), None))
    assert st.item() == 0
    for b in bufs:
        lib.check(lib.b2a_peer_buffer_destroy(ctypes.c_void_p(b)))


def test_peer_exchange_skewed_ranks_never_return_a_wrong_vector(eng):
    """ADVICE r1 (medium): a rank that runs ahead must never make a slower rank accept a FUTURE vector for an old
    sequence number.  Rank 0 publishes 1..7 while rank 1 has only published 1: `latest` shows (7, 1) with the right
    payloads, the lock-step collect of a lapped sequence number reports the loss (NaN row, negative seq, status) instead
    of returning other data, and a sequence number still inside the four-slot window is returned exactly."""
    import ctypes

    lib, world, n_max = eng.lib, 2, 8
    bufs, peers = _peer_setup(lib, world, n_max)
    val = lambda r, s: torch.arange(6, dtype=torch.float32) + 10 * r + 100 * s  # noqa: E731
    keep = []
    for s in range(1, 8):
        v = val(0, s)
        keep.append(v)
        lib.check(lib.b2a_peer_put_f32(ctypes.c_void_p(v.data_ptr()), 6, peers, world, 0, n_max, s, None))
    v1 = val(1, 1)
    lib.check(lib.b2a_peer_put_f32(ctypes.c_void_p(v1.data_ptr()), 6, peers, world, 1, n_max, 1, None))
    for r in range(world):  # both ranks see the same picture
        out, seqs = torch.empty(world, 6), torch.zeros(world, dtype=torch.int32)
        lib.check(lib.b2a_peer_latest_f32(ctypes.c_void_p(bufs[r]), world, 6, n_max, ctypes.c_void_p(out.data_ptr()),
                                          ctypes.c_void_p(seqs.data_ptr()), None))
        assert seqs.tolist() == [7, 1]
        assert torch.equal(out[0], val(0, 7)) and torch.equal(out[1], val(1, 1))
    # sequence 1 of rank 0 was overwritten by 5 (same slot): the collect must say so, not hand back 5's data
    out, seqs = torch.empty(world * 6), torch.zeros(world, dtype=torch.int32)
    lib.check(lib.b2a_peer_collect_f32(ctypes.c_void_p(bufs[1]), world, 6, n_max, 1, ctypes.c_void_p(out.data_ptr()),
                                       ctypes.c_void_p(seqs.data_ptr()), None))
    assert torch.isnan(out[:6]).all() and torch.equal(out[6:], val(1, 1))
    assert seqs.tolist() == [-5, 1]
    st = torch.zeros(1, dtype=torch.int32)
    lib.check(lib.b2a_peer_status(ctypes.c_void_p(bufs[1]), world, n_max, ctypes.c_void_p(st.data_ptr()), None))
    assert st.item() == 1
    # rank 1 catches up to 6 (still inside rank 0's window 4..7): exact data for both
    for s in range(2, 7):
        v = val(1, s)
        keep.append(v)
        lib.check(lib.b2a_peer_put_f32(ctypes.c_void_p(v.data_ptr()), 6, peers, world, 1, n_max, s, None))
    lib.check(lib.b2a_peer_collect_f32(ctypes.c_void_p(bufs[0]), world, 6, n_max, 6, ctypes.c_void_p(out.data_ptr()),
                                       ctypes.c_void_p(seqs.data_ptr()), None))
    assert torch.equal(out, torch.cat([val(0, 6), val(1, 6)])) and seqs.tolist() == [6, 6]
    # nothing published yet -> NaN row and sequence number 0 from `latest`
    bufs2, _ = _peer_setup(lib, world, n_max)
    out, seqs = torch.zeros(world, 6), torch.ones(world, dtype=torch.int32)
    lib.check(lib.b2a_peer_latest_f32(ctypes.c_void_p(bufs2[0]), world, 6, n_max, ctypes.c_void_p(out.data_ptr()),
                                      ctypes.c_void_p(seqs.data_ptr()), None))
    assert torch.isnan(out).all() and seqs.tolist() == [0, 0]
    for b in bufs + bufs2:
        lib.check(lib.b2a_peer_buffer_destroy(ctypes.c_void_p(b)))


# ------------------------------------------------------------------------------------------
# SpecAugment band masks (csrc/specmask.cu) against the oracle restatement and the reference goldens
# ------------------------------------------------------------------------------------------
def test_spec_band_mask_matches_reference(eng, golden_spec):
    from tests.golden import make_golden_spectral as mg

    x = cases.make_input("cfg1")
    X = sp.stft(x, 16000).contiguous()  # [4, 1, 257, 126]
    bins_hz = torch.linspace(0, 8000, 257)
    Y = eng.spec_band_mask(X.clone(), bins_hz, mg.FMIN, mg.FMAX, 0)
    ref = torch.from_numpy(golden_spec["maskfreq_stft"])
    assert torch.equal(Y == 0, ref == 0)                      # exactly the reference's cells
    assert torch.equal(Y[Y != 0], X[Y != 0])                  # untouched cells keep their bits
    assert rel_err(torch.view_as_real(Y), torch.view_as_real(ref)) < 1e-5
    Y = eng.spec_band_mask(X.clone(), torch.linspace(0, 1.0, 126), mg.TMIN, mg.TMAX, 1)
    ref = torch.from_numpy(golden_spec["masktime_stft"])
    assert torch.equal(Y == 0, ref == 0) and rel_err(torch.view_as_real(Y), torch.view_as_real(ref)) < 1e-5
    Y = eng.spec_band_mask(X[:1].clone(), bins_hz, mg.FMIN[:1], mg.FMAX[:1], 0, val=0.25)
    assert rel_err(torch.view_as_real(Y), torch.view_as_real(torch.from_numpy(golden_spec["maskfreq_val_stft"]))) < 1e-5
    # stereo: an item's band applies to both of its channels; scalar band broadcasts over the batch
    Xs = X.reshape(2, 2, 257, 126).clone()
    Ys = eng.spec_band_mask(Xs.clone(), bins_hz, torch.tensor([1000.0, 2000.0]), torch.tensor([1500.0, 4000.0]), 0)
    want = sp.mask_frequencies(Xs, 16000, torch.tensor([1000.0, 2000.0]), torch.tensor([1500.0, 4000.0]))
    assert torch.equal(Ys == 0, want == 0)
    Y1 = eng.spec_band_mask(X.clone(), bins_hz, torch.tensor(100.0), torch.tensor(200.0), 0)
    assert torch.equal(Y1 == 0, sp.mask_frequencies(X, 16000, 100.0, 200.0) == 0)


def test_spec_rotate_and_mask_low_match_reference(eng, golden_spec):
    from tests.golden import make_golden_spectral as mg

    x = cases.make_input("cfg1")
    X = sp.stft(x, 16000).contiguous()
    Y = eng.spec_rotate(X.clone(), mg.SHIFT)  # per item
    assert rel_err(torch.view_as_real(Y[2:]), torch.view_as_real(torch.from_numpy(golden_spec["shift_stft"]))) < 1e-5
    corr = torch.from_numpy(golden_spec["corrupt_in"])
    Y = eng.spec_rotate(X.clone(), corr)  # per cell
    assert rel_err(torch.view_as_real(Y), torch.view_as_real(sp.shift_phase(X, corr))) < 1e-5
    Y = eng.spec_mask_low(X.clone(), mg.DBCUT)
    ref = torch.from_numpy(golden_spec["masklow_stft"])
    assert torch.equal(Y[:2] == 0, ref == 0)  # the same cells as the real reference, incl. the global top_db floor
    assert rel_err(torch.view_as_real(Y[:2]), torch.view_as_real(ref)) < 1e-5
    want = sp.mask_low_magnitudes(X, mg.DBCUT, val=0.5)  # non-zero fill keeps the phase
    got = eng.spec_mask_low(X.clone(), mg.DBCUT, val=0.5)
    assert rel_err(torch.view_as_real(got), torch.view_as_real(want)) < 1e-5


# ------------------------------------------------------------------------------------------
# randomised geometry sweeps (small sizes): padding modes, offsets, strides, partitions
# ------------------------------------------------------------------------------------------
def _extend(x, lo, hi, mode):
    """x[..., lo:hi] with out-of-range indices resolved by ``mode``."""
    T = x.shape[-1]
    idx = torch.arange(lo, hi)
    if mode == "replicate":
        return x[..., idx.clamp(0, T - 1)]
    if mode == "circular":
        return x[..., idx % T]
    v = torch.zeros(*x.shape[:-1], hi - lo)
    ok = (idx >= 0) & (idx < T)
    v[..., ok] = x[..., idx[ok]]
    return v


def test_fir_direct_random_geometries(eng):
    import torch.nn.functional as Fn

    rng = np.random.RandomState(1)
    for it in range(14):
        B, C, T = int(rng.randint(1, 4)), int(rng.randint(1, 3)), int(rng.randint(200, 5000))
        K, stride = int(rng.randint(1, 320)), int(rng.choice([1, 1, 2, 3, 4]))
        g = torch.Generator().manual_seed(it)
        x, taps = torch.randn(B, C, T, generator=g), torch.randn(B, K, generator=g)
        left, left0 = torch.from_numpy(rng.randint(0, K + 3, size=B)).int(), int(rng.randint(0, 5))
        mode = str(rng.choice(["constant", "replicate"]))
        out_len = int(rng.randint(1, (T + stride - 1) // stride + 1))
        sub = bool(stride == 1 and out_len <= T and rng.rand() < 0.3)
        out = eng.fir_direct(x, taps, rows_per_filt=C, left=left, left0=left0, stride=stride, out_len=out_len,
                             pad_mode=mode, subtract_from_input=sub)
        for b in range(B):
            L = left0 + int(left[b])
            xv = _extend(x[b], -L, (out_len - 1) * stride + K - L, mode)
            y = Fn.conv1d(xv[:, None, :], taps[b].reshape(1, 1, K), stride=stride)[:, 0, :out_len]
            ref = (x[b, :, :out_len] - y) if sub else y
            assert rel_err(out[b], ref) < 2e-5, (B, C, T, K, stride, mode, out_len, sub)


def test_preemphasis_kernel_config(eng):
    """DSPMixin.preemphasis (ref:audiotools/core/dsp.py:372-390) = conv1d([1, -coef, 0], padding=1): the direct FIR
    kernel with 3 taps, one shared filter for every row, zero padding."""
    import torch.nn.functional as Fn

    x = cases.make_input("short")  # [2, 1, 4000]
    taps = torch.tensor([[1.0, -0.85, 0.0]])
    out = eng.fir_direct(x, taps, rows_per_filt=2, left0=1, stride=1, pad_mode="constant")
    ref = Fn.conv1d(x.reshape(-1, 1, 4000), taps.view(1, 1, -1), padding=1).reshape(x.shape)
    assert out.shape == x.shape and torch.allclose(out, ref, atol=1e-7)


def test_fftconv_random_geometries(eng):
    import torch.nn.functional as Fn

    rng = np.random.RandomState(2)
    for it, Lf in enumerate([5, 641, 1024, 1025, 2500, 100]):  # 1 partition (product formed in the inverse FFT) and several
        B, C, T = int(rng.randint(1, 3)), int(rng.randint(1, 3)), int(rng.randint(1500, 7000))
        g = torch.Generator().manual_seed(100 + it)
        x, taps = torch.randn(B, C, T, generator=g), torch.randn(B, Lf, generator=g) / Lf ** 0.5
        off = torch.from_numpy(rng.randint(0, Lf, size=B)).int()
        mode, sub = str(rng.choice(["constant", "replicate", "circular"])), bool(rng.rand() < 0.3)
        out = eng.fftconv(x, taps, rows_per_filt=C, offset=off, offset0=0, pad_mode=mode, subtract_from_input=sub)
        for b in range(B):
            o = int(off[b])
            xv = _extend(x[b], o - (Lf - 1), T + o, mode)  # out[n] = sum_k taps[k] xv[n - k + o]
            y = Fn.conv1d(xv[:, None, :], taps[b].flip(0).reshape(1, 1, Lf))[:, 0, :T]
            ref = (x[b] - y) if sub else y
            assert rel_err(out[b], ref) < 5e-5, (B, C, T, Lf, mode, sub)


# ------------------------------------------------------------------------------------------
# 2048-point mel / log-mel kernel (spectral_warp_kernel<10,0>) under the simulator against the reference's mel_spectrogram
# ------------------------------------------------------------------------------------------
from tests.conftest import elementwise_ok as _elementwise_ok  # noqa: E402


@pytest.mark.parametrize("hop,T,n_mels", [(512, 20000, 128), (256, 9000, 80), (300, 7000, 64), (510, 12000, 128)])
def test_spectral_2048_mel_matches_reference(eng, hop, T, n_mels):
    sr = 44100
    g = torch.Generator().manual_seed(hop)
    x = 0.1 * torch.randn(3, 2, T, generator=g)
    x[1] *= 1e-4                                                     # a very quiet item
    x[2, 0] = 0.5 + 0.3 * torch.sin(torch.arange(T) * 0.013)          # DC offset + low tone: leakage, small bins
    x[2, 1, : T // 2] = 0.0                                           # silent stretch: all-zero tiles
    fb, lo, hi = _mel_tables(sr, 2048, n_mels)
    w = sp.get_window("hann" if hop != 300 else "sqrt_hann", 2048)
    gain = torch.tensor([0.7, -3.0, 1.5])
    assert eng.spectral_kernel_name(2048, hop) == "spectral_warp_kernel<10,0>"
    out = eng.spectral(x, 2048, hop, w, gain=gain, want_scaled=True, mel_fb=fb, mel_lo=lo, mel_hi=hi, want_stft=False)
    lg = eng.spectral(x, 2048, hop, w, mel_fb=fb, mel_lo=lo, mel_hi=hi, post=_lib.POST_LOG10, post_eps=1e-5,
                      post_power=2.0, want_stft=False)["mel"]
    assert torch.equal(out["scaled"], x * gain[:, None, None])
    ref = sp.mel_spectrogram(x * gain[:, None, None], sr, n_mels, window_length=2048, hop_length=hop,
                             window_type="hann" if hop != 300 else "sqrt_hann")
    assert out["mel"].shape == ref.shape
    for b in range(3):  # per item: the quiet item must be as accurate, relative to itself, as the loud one
        assert rel_err(out["mel"][b], ref[b]) < 2e-5, b
        assert _elementwise_ok(out["mel"][b], ref[b], 1e-4, 2e-6), b  # measured: 2.5e-7 of the frame max
    ref_log = sp.log_mel(sp.mel_spectrogram(x, sr, n_mels, window_length=2048, hop_length=hop,
                                            window_type="hann" if hop != 300 else "sqrt_hann"))
    # log10 units.  Items 0 / 1 (noise-like: every band well above the transform's error floor): tight; item 2 has
    # bands 120 dB below its DC line, where ANY fp32 transform differs from another by more than the value itself --
    # there the linear criterion above is the meaningful one
    assert (lg[:2] - ref_log[:2]).abs().max() < 2e-4


# ------------------------------------------------------------------------------------------
# pitch_shift / time_stretch against the independent specification oracle (VERDICT r1: "compared with nothing
# independent"): exact splice positions wherever the arg-max is decided by more than float32 rounding, waveform 1e-4
# ------------------------------------------------------------------------------------------
def _check_pitch_vs_golden(run, g, key, tol=1e-4, rows=slice(None)):
    """run() -> (y [rows, L] float32 tensor, positions [rows, J] int32 tensor)."""
    y, pos = run()
    ref_y, ref_pos, margin = g[key + "_y"][rows], g[key + "_pos"][rows], g[key + "_margin"][rows]
    assert tuple(y.shape) == ref_y.shape and tuple(pos.shape) == ref_pos.shape  # length and frame count exact
    pos = pos.numpy()
    decided = margin > 1e-5  # correlation margin relative to the size of the summed terms; fp32 sums resolve 1e-6
    assert decided.mean() > 0.95
    assert np.array_equal(pos[decided], ref_pos[decided])
    same = (pos == ref_pos).all(axis=1)  # rows whose every splice agrees (all of them unless a near-tie flipped)
    assert same.mean() >= 0.5
    err = np.abs(y.numpy()[same] - ref_y[same]).max() / np.abs(ref_y[same]).max()
    assert err < tol, err
    return same


def test_pitch_shift_and_time_stretch_match_spec_oracle(eng):
    import os

    from tests.golden import make_golden_pitch as mg

    g = np.load(os.path.join(os.path.dirname(mg.__file__), "pitch_golden.npz"))
    x = torch.from_numpy(g["x"][:2])[:, None, :]  # the simulator runs every CUDA thread as a host thread: 2 rows
    for st in (2.0, -2.0):
        _check_pitch_vs_golden(lambda: tuple(t.reshape(2, -1) for t in eng.pitch_shift(x, mg.SR, st, return_positions=True)),
                               g, f"pitch_{st:g}", rows=slice(0, 2))
    _check_pitch_vs_golden(lambda: tuple(t.reshape(2, -1) for t in eng.time_stretch(x, mg.SR, 1.25, return_positions=True)),
                           g, "stretch_1.25", rows=slice(0, 2))


# ------------------------------------------------------------------------------------------
# warp-autonomous K-weighting kernel (csrc/lufs.cu): rates with r != 0, rows of unequal phase, rows cut into several
# runs that each start with a warm-up (> 64 segments per row), short rows, unaligned lengths
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sr,T,B,C", [(11025, 30001, 2, 1), (48000, 70000, 1, 2), (16000, 140001, 1, 1), (44100, 5000, 3, 2),
                                      (22050, 33333, 2, 2)])
def test_lufs_warp_kernel_block_energies_and_loudness(eng, sr, T, B, C):
    g = torch.Generator().manual_seed(sr + T)
    x = 0.2 * torch.randn(B, C, T, generator=g) * torch.rand(B, 1, 1, generator=g)
    x[0, 0, : T // 3] += 0.3  # DC step: exercises the long tail of the 38 Hz high-pass across many segments
    Tp = padded_len(T, sr)
    out = eng.lufs(x, sr, padded_length=Tp, want_blocks=True)
    z_ref = sp.Meter(sr).block_energies(torch.nn.functional.pad(x, (0, Tp - T)).permute(0, 2, 1))
    assert out["blocks"].shape == z_ref.shape  # block indexing bit-exact
    assert rel_err(out["blocks"], z_ref) < 1e-4
    loud_ref = sp.loudness(x, sr)
    assert torch.allclose(out["loud"], loud_ref, atol=2e-3)


# ------------------------------------------------------------------------------------------
# element-wise / peak effects (csrc/effects.cu) against the REAL reference's outputs (fx_* goldens) and torch
# ------------------------------------------------------------------------------------------
def test_effect_kernels_match_reference(eng, golden_spec):
    g = golden_spec
    xs = cases.make_input("cfg1") * 0.3
    xs2 = torch.cat([xs, 0.5 * xs.flip(-1)], 1)
    G = lambda k: torch.from_numpy(g[k])  # noqa: E731
    q = torch.tensor([8, 16, 256, 3])
    assert torch.allclose(eng.quantize(xs2, q), G("fx_quant"), atol=1e-6)
    assert torch.allclose(eng.quantize(xs2, q, mulaw=True), G("fx_mulaw"), atol=1e-6)
    x5 = xs2 * 5
    assert torch.equal(eng.row_absmax(x5), x5.abs().max(dim=-1, keepdim=True).values)
    assert torch.allclose(eng.limit_peak(x5, 0.7), G("fx_maxaudio"), atol=1e-7)
    # clip_distortion: the reference's quantiles of row 0 (see EffectMixin.clip_distortion), then the clamp
    perc = torch.tensor([0.05, 0.2, 0.0, 0.5])
    qs = torch.cat([perc / 2, 1 - perc / 2])
    thr = eng.quantile(xs[0, 0], qs)
    assert torch.allclose(thr, torch.quantile(xs[0, 0], qs), atol=0, rtol=1e-6)
    assert torch.allclose(eng.clamp_items(xs, thr[:4], thr[4:]), G("fx_clip"), atol=1e-7)
    # order statistics are exact whatever the data (negative values, ties, odd length)
    rng = torch.Generator().manual_seed(5)
    row = torch.randn(10007, generator=rng).round(decimals=2)
    ks = torch.tensor([0, 1, 5003, 10005, 10006, 777])
    assert torch.equal(eng.order_stats(row, ks), row.sort().values[ks])
    # mix: x + g * other with the reference's two roundings
    other = torch.randn(xs2.shape, generator=rng) * 0.1
    gain = torch.tensor([0.5, 2.0, 0.0, 1.25])
    assert torch.equal(eng.mix(xs2, other, gain), xs2 + other * gain[:, None, None])
    assert torch.equal(eng.mix(xs2, other), xs2 + other)


# ------------------------------------------------------------------------------------------
# device collate (csrc/collate.cu): ragged items -> padded / truncated batch, excerpt windows with offsets
# ------------------------------------------------------------------------------------------
def test_pack_rows_pad_truncate_and_windows(eng):
    g = torch.Generator().manual_seed(11)
    items = [torch.randn(2, 1001, generator=g), torch.randn(3, 2, 1500, generator=g), torch.randn(2, 640, generator=g)]
    for T_out in (1500, 640, 1000, 2048):  # pad to the longest, truncate to the shortest, in between, beyond
        out = eng.pack_rows(items, T_out)
        ref = torch.zeros(5, 2, T_out)
        rows = [items[0][None], items[1], items[2][None]]
        i = 0
        for r in rows:
            n = min(T_out, r.shape[-1])
            ref[i:i + r.shape[0], :, :n] = r[..., :n]
            i += r.shape[0]
        assert torch.equal(out, ref), T_out
    long = torch.randn(1, 2, 5000, generator=g)
    offs = [0, 13, 4096, 4990, -7]
    win = eng.pack_rows([long] * len(offs), 512, offsets=offs)
    for k, o in enumerate(offs):
        ref = torch.zeros(2, 512)
        lo, hi = max(o, 0), min(o + 512, 5000)
        ref[:, lo - o: hi - o] = long[0, :, lo:hi]
        assert torch.equal(win[k], ref), o
