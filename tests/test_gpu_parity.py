"""GPU parity tests proper (run with ``-m gpu`` on an H100): the product path -- AudioSignal API ->
ctypes -> C ABI of libb2a.so -> sm_90a kernels -- against (a) the golden vectors produced by the
REAL reference, (b) the oracle on the same seeded inputs, and (c) at BASELINE.json's full sizes,
size-independent properties (linearity, batch == per-item, normalise-then-measure, round trips).

Tolerance: BASELINE.json asks for 1e-4 relative FP32 and bit-exact frame/block indexing.
"relative" = max|a-b| / max|b| (``rel_err``); LUFS values are compared in dB with atol 2e-3
(1e-4 of a ~-20 LUFS value).  Shapes (frame counts, block counts) are compared exactly.
"""
import numpy as np
import pytest
import torch

from tests.conftest import elementwise_ok, rel_err
from tests.golden import cases

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TOL = 1e-4
LUFS_ATOL = 2e-3


@pytest.fixture(scope="module")
def at():
    import __graft_entry__ as graft

    graft.build()
    import audiotools_b200

    return audiotools_b200


@pytest.fixture(scope="module")
def sp():
    from oracle import signal_path

    return signal_path


def G(golden, key):
    return torch.from_numpy(golden[key])


def sig_of(at, name, sl=slice(None), **kw):
    return at.AudioSignal(cases.make_input(name)[sl].clone(), cases.sample_rate(name), **kw).to(DEV)


# ------------------------------------------------------------------------------------------
# BASELINE configs[0]: batch=4 mono 1s@16kHz stft(n_fft=512, hop=128) -- reference parity
# ------------------------------------------------------------------------------------------
def test_cfg1_stft_matches_reference(at, golden):
    sig = sig_of(at, "cfg1")
    s = sig.stft(window_length=512, hop_length=128)
    ref = G(golden, "cfg1_stft")
    assert s.shape == ref.shape == (4, 1, 257, 126)  # frame indexing bit-exact
    assert s.dtype == torch.complex64 and sig.stft_data is s
    assert rel_err(torch.view_as_real(s.cpu()), torch.view_as_real(ref)) < TOL
    assert rel_err(torch.view_as_real(sig_of(at, "cfg1").stft().cpu()), torch.view_as_real(ref)) < TOL  # defaults


def test_stft_variants_match_reference(at, golden):
    p = at.STFTParams(256, 64, "sqrt_hann", True, "reflect")
    s = sig_of(at, "cfg1", slice(0, 2), stft_params=p).stft()
    ref = G(golden, "cfg1_stft_match_stride")
    assert s.shape == ref.shape and s.shape[-1] == 16000 // 64
    assert rel_err(torch.view_as_real(s.cpu()), torch.view_as_real(ref)) < TOL
    x = cases.make_input("cfg1")[:2, :, :15999]
    s = at.AudioSignal(x, 16000, stft_params=at.STFTParams(256, 64, "hann", True, "reflect")).to(DEV).stft()
    ref = G(golden, "cfg1_stft_match_stride_odd")
    assert s.shape == ref.shape and rel_err(torch.view_as_real(s.cpu()), torch.view_as_real(ref)) < TOL
    s = sig_of(at, "cfg1", slice(0, 2)).stft(window_length=256, hop_length=100, window_type="average")
    ref = G(golden, "cfg1_stft_average_hop100")
    assert s.shape == ref.shape and rel_err(torch.view_as_real(s.cpu()), torch.view_as_real(ref)) < TOL


@pytest.mark.parametrize("n_fft,hop", [(32, 8), (64, 16), (128, 32), (256, 77), (1024, 256), (4096, 1024)])
def test_stft_all_sizes_vs_oracle(at, sp, n_fft, hop):
    x = cases.make_input("cfg1")[:2]
    s = at.AudioSignal(x.clone(), 16000).to(DEV).stft(window_length=n_fft, hop_length=hop)
    ref = sp.stft(x, 16000, n_fft, hop)
    assert s.shape == ref.shape
    assert rel_err(torch.view_as_real(s.cpu()), torch.view_as_real(ref)) < TOL


def test_mel_mfcc_logmag_match_reference(at, golden):
    assert rel_err(sig_of(at, "cfg1").mel_spectrogram(n_mels=80).cpu(), G(golden, "cfg1_mel80")) < TOL
    m = sig_of(at, "cfg1", slice(0, 2)).mel_spectrogram(n_mels=40, mel_fmin=100.0, mel_fmax=6000.0,
                                                        window_length=1024, hop_length=256)
    assert rel_err(m.cpu(), G(golden, "cfg1_mel40_fmin_fmax")) < TOL
    assert rel_err(sig_of(at, "cfg1").mfcc().cpu(), G(golden, "cfg1_mfcc")) < TOL
    sig = sig_of(at, "cfg1", slice(0, 2))
    sig.stft()
    assert rel_err(sig.log_magnitude().cpu(), G(golden, "cfg1_logmag")) < TOL


def test_stft_istft_round_trip(at):
    """ref:tests/core/test_audio_signal.py:400-456."""
    sig = sig_of(at, "cfg1")
    x = sig.audio_data.clone()
    sig.stft()
    sig.istft()
    assert torch.allclose(sig.audio_data, x, atol=1e-5)
    sig = sig_of(at, "cfg1", stft_params=at.STFTParams(256, 64, "sqrt_hann", True, "reflect"))
    assert sig.stft().shape[-1] == sig.signal_length // 64
    sig.istft()
    # with match_stride the 2+2 dropped edge frames are not recoverable: the reference's own test
    # compares the interior only (discard = 2 * window_length)
    assert sig.signal_length == x.shape[-1]
    assert torch.allclose(sig.audio_data[..., 512:-512], x[..., 512:-512], atol=1e-5)


def test_istft_matches_reference(at, golden):
    """The fused inverse kernel (csrc/istft.cu) against the real reference's istft outputs, and against torch.istft
    on spectra that are not consistent STFTs (so the overlap-add and the envelope are exercised on their own)."""
    sig = sig_of(at, "cfg1", slice(0, 2))
    sig.stft()
    assert rel_err(sig.istft().audio_data.cpu(), G(golden, "cfg1_istft")) < TOL
    sig = sig_of(at, "cfg1", slice(0, 2), stft_params=at.STFTParams(256, 64, "sqrt_hann", True, "reflect"))
    sig.stft()
    assert rel_err(sig.istft().audio_data.cpu(), G(golden, "cfg1_istft_match_stride")) < TOL
    g = torch.Generator().manual_seed(5)
    for n_fft, hop, T in ((2048, 512, 100000), (1024, 256, 50000), (512, 100, 20000), (128, 32, 8000), (64, 64, 4000)):
        w = torch.hann_window(n_fft) + 0.1
        X = torch.stft(torch.randn(4, T, generator=g), n_fft, hop, window=w, center=True, return_complex=True)
        X = X * (1 + 0.3 * torch.randn(X.shape, generator=g))
        ref = torch.istft(X, n_fft, hop, window=w, center=True, length=T - 13)
        from audiotools_b200.engine import get_engine

        out = get_engine().istft(X.reshape(2, 2, *X.shape[1:]).to(DEV), n_fft, hop, w.to(DEV), T - 13)
        assert rel_err(out.reshape(4, -1).cpu(), ref) < TOL, (n_fft, hop)


def test_istft_full_size_round_trip(at):
    """cfg2's full shape (64 x 2ch x 10 s @ 44.1 kHz, 2048/512): istft(stft(x)) == x to 1e-5 (size-independent
    property; the reference's own round-trip tolerance is atol 1e-6 on [-1, 1] audio, ref:tests/core/test_audio_signal.py:400-456)."""
    g = torch.Generator().manual_seed(11)
    x = (0.2 * torch.randn(64, 2, 441000, generator=g)).to(DEV)
    sig = at.AudioSignal(x, 44100)
    sig.stft(window_length=2048, hop_length=512)
    sig.istft(window_length=2048, hop_length=512)
    assert sig.audio_data.shape == x.shape
    assert (sig.audio_data - x).abs().max().item() < 1e-5


# ------------------------------------------------------------------------------------------
# loudness
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,key", [("cfg2", "cfg2_lufs"), ("lufs16k", "lufs16k"), ("short", "lufs_short"),
                                      ("lufs48k", "lufs48k"), ("lufs11k", "lufs11k")])
def test_loudness_matches_reference(at, golden, name, key):
    sig = sig_of(at, name)
    l = sig.loudness()
    assert l.dtype == torch.float32 and l.shape == (sig.batch_size,)
    assert torch.allclose(l.cpu(), G(golden, key), atol=LUFS_ATOL)
    assert sig._loudness is l or torch.equal(sig._loudness, l)  # cached
    if name == "cfg2":
        assert l[1].item() == -70.0  # silent item: NaN scrub -> -inf -> clamp


def test_block_energies_bit_exact_indexing(at, golden):
    from audiotools_b200.engine import get_engine

    x = cases.make_input("cfg2").to(DEV)
    out = get_engine().lufs(x, 44100, want_blocks=True)
    ref = G(golden, "cfg2_z")
    assert out["blocks"].shape == ref.shape
    assert rel_err(out["blocks"].cpu(), ref) < TOL
    m = at.Meter(44100)
    assert torch.allclose(m.integrated_loudness(x.permute(0, 2, 1)).cpu()[[0, 2]], G(golden, "cfg2_lufs")[[0, 2]],
                          atol=LUFS_ATOL)


def test_loudness_batch_equals_per_item(at):
    """ref:tests/core/test_loudness.py:31-52."""
    sig = sig_of(at, "lufs16k")
    batch = sig.loudness().cpu()
    for i in range(0, 16, 5):
        one = sig_of(at, "lufs16k", slice(i, i + 1)).loudness().cpu()
        assert torch.allclose(one, batch[i: i + 1], atol=1e-5)


def test_normalize_and_volume_change_match_reference(at, golden):
    sig = sig_of(at, "cfg2")
    sig.normalize(-24.0)
    assert sig._pending_gain is not None and sig._loudness is None  # deferred; cache dropped like the reference
    y = sig.audio_data
    assert sig._pending_gain is None
    assert rel_err(y.cpu(), G(golden, "cfg2_norm")) < TOL
    db = G(golden, "norm16k_db")
    sig = sig_of(at, "lufs16k", slice(0, 4)).normalize(db)
    assert rel_err(sig.audio_data.cpu(), G(golden, "norm16k")) < TOL
    sig = sig_of(at, "lufs16k", slice(0, 4)).volume_change(db)
    assert rel_err(sig.audio_data.cpu(), G(golden, "volchange16k")) < TOL


def test_normalize_then_measure(at):
    """ref:tests/core/test_effects.py:15-33."""
    x = torch.randn(16, 2, 32000, generator=torch.Generator().manual_seed(0))
    for db in (-70.0, -50.0, -30.0, -10.0):
        sig = at.AudioSignal(x.clone(), 16000).to(DEV).normalize(db)
        assert torch.allclose(sig.loudness().cpu(), torch.full((16,), db), atol=0.1)


# ------------------------------------------------------------------------------------------
# BASELINE configs[1]: LUFS normalise + log-mel, fused
# ------------------------------------------------------------------------------------------
def test_cfg2_fused_pipeline_matches_reference(at, golden):
    sig = sig_of(at, "cfg2")
    sig.normalize(-24.0)
    logmel = sig.mel_spectrogram(n_mels=128, window_length=2048, hop_length=512, window_type="hann", log=True)
    assert sig._pending_gain is None and sig.stft_data is None  # gain rode along; no STFT materialised
    assert logmel.shape == golden["cfg2_logmel"].shape
    assert rel_err(logmel.cpu(), G(golden, "cfg2_logmel")) < TOL
    assert rel_err(sig.audio_data.cpu(), G(golden, "cfg2_norm")) < TOL
    mel = sig.mel_spectrogram(n_mels=128, window_length=2048, hop_length=512, window_type="hann")
    assert rel_err(mel.cpu(), G(golden, "cfg2_mel")) < TOL
    # unfused order gives the same thing
    sig2 = sig_of(at, "cfg2").normalize(-24.0)
    _ = sig2.audio_data
    lm2 = sig2.mel_spectrogram(n_mels=128, window_length=2048, hop_length=512, log=True)
    assert torch.allclose(lm2, logmel, atol=1e-5)


def _full_batch(B=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = (0.1 * torch.randn(B, 2, 441000, generator=g)).clamp(-1, 1)
    return (x * (0.05 + 0.95 * torch.rand(B, 1, 1, generator=g))).float()


def test_cfg2_full_size_properties_and_oracle_subset(at, sp):
    """64 x 2ch x 10 s @ 44.1 kHz: shapes, oracle on a subset of items, linearity, batch == per-item."""
    x = _full_batch()
    sig = at.AudioSignal(x.clone(), 44100).to(DEV)
    lufs = sig.loudness().clone()
    sig.normalize(-24.0)
    logmel = sig.mel_spectrogram(n_mels=128, window_length=2048, hop_length=512, window_type="hann", log=True)
    y = sig.audio_data
    assert logmel.shape == (64, 2, 128, 862) and y.shape == (64, 2, 441000)  # 1 + T//hop frames
    sub = [0, 31, 63]
    y_ref, l_ref = sp.normalize(x[sub], 44100, -24.0)
    lm_ref = sp.log_mel(sp.mel_spectrogram(y_ref, 44100, 128, window_length=2048, hop_length=512, window_type="hann"))
    assert torch.allclose(lufs[sub].cpu(), l_ref, atol=LUFS_ATOL)
    assert rel_err(y[sub].cpu(), y_ref) < TOL
    assert rel_err(logmel[sub].cpu(), lm_ref) < TOL
    # after normalisation every item measures -24 LUFS
    assert torch.allclose(sig.loudness().cpu(), torch.full((64,), -24.0), atol=1e-2)
    # loudness(a*x) = loudness(x) + 20 log10 a ; mel(a*x) = a*mel(x)
    a = 0.37
    l2 = at.AudioSignal((a * x).clone(), 44100).to(DEV).loudness()
    assert torch.allclose(l2, lufs + 20 * np.log10(a), atol=2e-3)
    m1 = at.AudioSignal(x[:8].clone(), 44100).to(DEV).mel_spectrogram(128, window_length=2048, hop_length=512)
    m2 = at.AudioSignal((a * x[:8]).clone(), 44100).to(DEV).mel_spectrogram(128, window_length=2048, hop_length=512)
    assert rel_err(m2, a * m1) < 1e-5
    # batch == per-item
    one = at.AudioSignal(x[5:6].clone(), 44100).to(DEV)
    assert torch.allclose(one.loudness(), lufs[5:6], atol=1e-4)
    one.normalize(-24.0)
    assert torch.allclose(one.mel_spectrogram(128, window_length=2048, hop_length=512, log=True), logmel[5:6], atol=1e-4)


def test_full_size_stft_parseval(at):
    """cfg2-size STFT: with a rectangular window and hop = n_fft, sum|X|^2 recovers the signal energy."""
    x = _full_batch(4, 3)[:, :1, : 2048 * 200]
    sig = at.AudioSignal(x.clone(), 44100).to(DEV)
    s = sig.stft(window_length=2048, hop_length=2048, window_type="boxcar")
    # interior frames (centre padding shifts frames by n_fft/2): energy per frame via Parseval
    frames = torch.nn.functional.pad(x.to(DEV), (1024, 1024), mode="reflect").unfold(-1, 2048, 2048)
    e_time = (frames ** 2).sum(-1)
    mag2 = s.abs() ** 2
    e_freq = (mag2[..., 0, :] + mag2[..., -1, :] + 2 * mag2[..., 1:-1, :].sum(-2)) / 2048
    assert rel_err(e_freq, e_time) < 1e-4


def test_cpu_tensor_raises_and_errors_map(at):
    sig = at.AudioSignal(torch.zeros(1, 1, 16000), 16000)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        sig.loudness()
    with pytest.raises(NotImplementedError, match="dense DFT path"):  # (any length up to 8192 runs: tests/test_gpu_dense_dft.py)
        at.AudioSignal(torch.zeros(1, 1, 40000), 16000).to(DEV).stft(window_length=10000, hop_length=2500)
    with pytest.raises(RuntimeError, match="without self.stft_data"):
        at.AudioSignal(torch.zeros(1, 1, 16000), 16000).to(DEV).istft()


# ------------------------------------------------------------------------------------------
# resample / FIR filters / equaliser / IR convolution / pitch shift / transforms
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key,sl,old,new", [("rs_48k_16k", 24000, 48000, 16000), ("rs_44k_16k", 22050, 44100, 16000),
                                            ("rs_16k_44k", 8000, 16000, 44100), ("rs_16k_48k", 8001, 16000, 48000),
                                            ("rs_44k_48k", 4410, 44100, 48000)])
def test_resample_matches_reference(at, golden, key, sl, old, new):
    x = cases.make_input("rs")[..., :sl]
    sig = at.AudioSignal(x.clone(), old).to(DEV).resample(new)
    ref = G(golden, key)
    assert sig.sample_rate == new and sig.audio_data.shape == ref.shape  # floor(new*T/old)
    assert rel_err(sig.audio_data.cpu(), ref) < TOL


def test_cfg3_shape_resample_lowpass(at, golden, sp):
    """BASELINE configs[2] shape (48k -> 16k + low_pass(8k)), small: vs the reference golden; and one
    30 s row of the full-size config vs the oracle."""
    sig = sig_of(at, "rs").resample(16000).low_pass(8000)
    assert rel_err(sig.audio_data.cpu(), G(golden, "rs_48k_16k_lp8k")) < TOL
    x = 0.1 * torch.randn(2, 1, 1440000, generator=torch.Generator().manual_seed(0))
    y = at.AudioSignal(x.clone(), 48000).to(DEV).resample(16000).low_pass(8000).audio_data
    assert y.shape == (2, 1, 480000)
    ref = sp.low_pass(sp.resample(x, 48000, 16000), 16000, 8000)
    assert rel_err(y.cpu(), ref) < TOL


def test_low_high_pass_match_reference(at, golden):
    cut = G(golden, "fir_cut")
    assert rel_err(sig_of(at, "fir").low_pass(cut).audio_data.cpu(), G(golden, "lp_peritem")) < TOL
    assert rel_err(sig_of(at, "fir").high_pass(cut / 8).audio_data.cpu(), G(golden, "hp_peritem")) < TOL
    assert rel_err(sig_of(at, "fir").low_pass(4000).audio_data.cpu(), G(golden, "lp_scalar")) < TOL
    sig = sig_of(at, "fir")
    sig.stft()
    assert sig.low_pass(4000).stft_data is None  # filters drop the STFT cache (ref dsp.py:182)


def test_low_high_pass_sine_thresholds(at):
    """ref:tests/core/test_dsp.py:76-109 (fully synthetic in the reference too)."""
    sr, f = 44100, 440
    t = torch.arange(sr) / sr
    x = (torch.sin(2 * np.pi * f * t) * torch.hann_window(sr))[None, None]
    mk = lambda: at.AudioSignal(x.clone(), sr).to(DEV)
    assert mk().low_pass(220).audio_data.abs().max() < 1e-4
    assert (mk().low_pass(880).audio_data.cpu() - x).abs().max() < 1e-3
    assert (mk().high_pass(220).audio_data.cpu() - x).abs().max() < 1e-4
    both = at.AudioSignal(x.repeat(2, 1, 1), sr).to(DEV).low_pass(torch.tensor([220.0, 880.0])).audio_data.cpu()
    assert both[0].abs().max() < 1e-4 and (both[1] - x[0]).abs().max() < 1e-3
    # the default HighPass cutoff 50 Hz @44.1k is a 44983-tap filter (44 partitions)
    y = mk().high_pass(50).audio_data.cpu()
    assert (y - x).abs().max() < 1e-3


def test_equalizer_and_filterbank_match_reference(at, golden):
    eq = golden["eq_db"]
    assert rel_err(sig_of(at, "fir").equalizer(eq).audio_data.cpu(), G(golden, "eq_out")) < TOL
    assert rel_err(sig_of(at, "fir").equalizer(eq[0]).audio_data.cpu(), G(golden, "eq_out_1d")) < TOL
    assert rel_err(sig_of(at, "fir", slice(0, 1)).mel_filterbank(4)[:, :1].cpu(), G(golden, "fbank4")) < TOL
    x = cases.make_input("fir")[:1]
    for n_bands in (1, 2, 4, 8, 12, 16):  # ref:tests/core/test_effects.py:184-231
        sig = at.AudioSignal(x.clone(), 44100).to(DEV)
        fb = sig.mel_filterbank(n_bands)
        assert fb.shape[-1] == n_bands and torch.allclose(fb.sum(-1).cpu(), x, atol=1e-6)
        assert torch.allclose(sig.equalizer(np.zeros(n_bands)).audio_data.cpu(), x, atol=1e-6)


def test_convolve_and_apply_ir_match_reference(at, golden):
    ir = cases.make_ir()
    mk_ir = lambda: at.AudioSignal(ir.clone(), 44100).to(DEV)
    assert rel_err(sig_of(at, "fir").convolve(mk_ir()).audio_data.cpu(), G(golden, "conv_out")) < TOL
    assert rel_err(sig_of(at, "fir").convolve(mk_ir(), start_at_max=False).audio_data.cpu(),
                   G(golden, "conv_out_nomax")) < TOL
    assert rel_err(sig_of(at, "fir").apply_ir(mk_ir()).audio_data.cpu(), G(golden, "applyir_plain")) < TOL
    drr = G(golden, "drr")
    assert rel_err(mk_ir().alter_drr(drr).audio_data.cpu(), G(golden, "alter_drr")) < TOL
    assert torch.allclose(mk_ir().measure_drr().cpu(), G(golden, "measure_drr"), atol=1e-3)
    out = sig_of(at, "fir").apply_ir(mk_ir(), drr=drr, ir_eq=golden["eq_db"]).audio_data.cpu()
    assert rel_err(out, G(golden, "applyir_full")) < TOL
    x = cases.make_input("fir")
    for delay in (0, 1, 777):  # delta IR == identity, ref:tests/core/test_effects.py:86-121
        d = torch.zeros(3, 1, 1000)
        d[..., delay] = 1.0
        y = at.AudioSignal(x.clone(), 44100).to(DEV).convolve(at.AudioSignal(d, 44100).to(DEV)).audio_data.cpu()
        assert torch.allclose(y, x, atol=1e-6)


def test_circular_convolution_full_size_vs_fft(at):
    """cfg4-size rows (10 s @44.1k, 1 s IR): against a float64 FFT circular convolution."""
    g = torch.Generator().manual_seed(5)
    x = 0.1 * torch.randn(4, 1, 441000, generator=g)
    t = torch.arange(44100) / 44100
    ir = torch.randn(4, 1, 44100, generator=g) * torch.exp(-t / 0.3)
    ir[..., 100] = 3.0
    y = at.AudioSignal(x.clone(), 44100).to(DEV).convolve(at.AudioSignal(ir.clone(), 44100).to(DEV)).audio_data.cpu()
    h = torch.nn.functional.pad(ir, (0, 441000 - 44100)).double()
    idx = h.abs().argmax(-1)
    h = torch.stack([torch.roll(h[i], -idx[i].item(), -1) for i in range(4)])
    ref = torch.fft.irfft(torch.fft.rfft(x.double(), 441000) * torch.fft.rfft(h, 441000), 441000)
    ref = ref / h.abs().amax(-1, keepdim=True).clamp(1e-5)
    assert rel_err(y, ref.float()) < TOL


def test_pitch_shift_properties(at):
    """SoX's output is pinned nowhere in the reference; parity = properties (ref:tests/core/test_effects.py:156-181)."""
    sr, T = 44100, 88200
    t = torch.arange(T) / sr
    x = torch.stack([0.5 * torch.sin(2 * np.pi * 440 * t), 0.3 * torch.sin(2 * np.pi * 1000 * t)])[:, None, :]
    x = x.repeat(1, 2, 1)
    for st in (2, -2, 7):
        sig = at.AudioSignal(x.clone(), sr).to(DEV).pitch_shift(st)
        y = sig.audio_data.cpu()
        assert y.shape == x.shape and sig.sample_rate == sr
        for i, f0 in enumerate((440.0, 1000.0)):
            spec = torch.fft.rfft(y[i, 0] * torch.hann_window(T)).abs()
            assert abs(spec.argmax().item() * sr / T - f0 * 2 ** (st / 12)) < 2.0
        single = at.AudioSignal(x[:1].clone(), sr).to(DEV).pitch_shift(st).audio_data.cpu()
        assert torch.equal(single, y[:1])  # batch[0] == single
        again = at.AudioSignal(x.clone(), sr).to(DEV).pitch_shift(st).audio_data.cpu()
        assert torch.equal(again, y)  # deterministic
        n = np.arange(T) / sr  # amplitude preserved; residual = WSOLA splice jitter only
        f = 440.0 * 2 ** (st / 12)
        A = np.stack([np.sin(2 * np.pi * f * n), np.cos(2 * np.pi * f * n)], 1)[4000:-4000]
        coef = np.linalg.lstsq(A, y[0, 0, 4000:-4000].double().numpy(), rcond=None)[0]
        assert abs(np.hypot(*coef) - 0.5) < 0.01
        assert (y[0, 0, 4000:-4000].double().numpy() - A @ coef).std() < 0.03 * 0.5
    # per-item shifts share one set of launches and equal the per-group calls; 0 copies the item
    xm = torch.cat([x, x.flip(0)], 0)
    ym = at.AudioSignal(xm.clone(), sr).to(DEV).pitch_shift([2, 0, -2, 2]).audio_data.cpu()
    y2 = at.AudioSignal(xm[[0, 3]].clone(), sr).to(DEV).pitch_shift(2).audio_data.cpu()
    assert torch.equal(ym[[0, 3]], y2) and torch.equal(ym[1], xm[1])
    assert torch.equal(ym[2:3], at.AudioSignal(xm[2:3].clone(), sr).to(DEV).pitch_shift(-2).audio_data.cpu())
    from audiotools_b200.data import transforms as tfm

    t = tfm.PitchShift(("choice", [-2, 2]))
    sig4 = at.AudioSignal(xm.clone(), sr)
    kw = at.util.prepare_batch(t.batch_instantiate([0, 1, 2, 3], sig4), DEV)
    shifts = at.util.host_view(kw["PitchShift"]["n_semitones"]).tolist()
    out = t(sig4.to(DEV), **kw).audio_data.cpu()
    assert torch.equal(out, at.AudioSignal(xm.clone(), sr).to(DEV).pitch_shift(shifts).audio_data.cpu())
    dc = torch.full((2, 1, 60000), 0.25)  # windows and interpolation weights sum to one
    for st in (2, -5):
        y = at.AudioSignal(dc.clone(), sr).to(DEV).pitch_shift(st).audio_data.cpu()
        assert torch.allclose(y[..., 3000:-6000], dc[..., 3000:-6000], atol=2e-6)


def test_transforms_compose_matches_reference(at, golden):
    """Compose[VolumeNorm, Equalizer, LowPass, HighPass, VolumeChange] with masks, instantiated with the
    same seeds as the real reference (tests/golden/make_golden.py): parameters and output must agree."""
    from audiotools_b200.data import transforms as tfm

    transform = tfm.Compose(
        [tfm.VolumeNorm(db=("uniform", -30, -16)), tfm.Equalizer(prob=0.5), tfm.LowPass(prob=0.7),
         tfm.HighPass(prob=0.6), tfm.VolumeChange()],
    )
    sig = sig_of(at, "tfm")
    kwargs = transform.batch_instantiate([10, 11, 12, 13], sig)
    flat = at.util.flatten(kwargs)
    ref_keys = {k[len("tfm_kw/"):] for k in golden.files if k.startswith("tfm_kw/")}
    assert {"/".join(k) for k in flat} == ref_keys
    for k, v in flat.items():
        ref = golden["tfm_kw/" + "/".join(k)]
        assert np.allclose(v.cpu().numpy(), ref), k  # seeded draws identical to the reference's
    kwargs = at.util.prepare_batch(kwargs, DEV)
    out = transform(sig.clone(), **kwargs)
    assert rel_err(out.audio_data.cpu(), G(golden, "tfm_out")) < TOL
    # the host mirrors recorded by prepare_batch spare the mask / cutoff synchronisations; values are unchanged
    lp = kwargs["Compose"]["2.LowPass"]
    assert torch.equal(at.util.host_view(lp["mask"]), lp["mask"].cpu())
    assert torch.equal(at.util.host_view(lp["cutoff"]), lp["cutoff"].cpu())
    # same kwargs twice => same output; batch[0] == single (ref:tests/data/test_transforms.py:21-85)
    out2 = transform(sig.clone(), **kwargs)
    assert torch.equal(out2.audio_data, out.audio_data)


def test_cfg4_augment_pipeline(at):
    """BASELINE configs[3] shape: Compose[Equalizer + RoomImpulseResponse + PitchShift(+-2)] on a batch."""
    from audiotools_b200.data import transforms as tfm

    g = torch.Generator().manual_seed(9)
    B, T, sr = 8, 88200, 44100
    x = 0.1 * torch.randn(B, 1, T, generator=g)
    t = torch.arange(sr) / sr
    irs = []
    for i in range(3):
        h = torch.randn(1, 1, sr, generator=g) * torch.exp(-t / 0.3) * 0.1
        h[..., 50 + i] = 1.0
        irs.append(at.AudioSignal(h, sr))
    transform = tfm.Compose([tfm.Equalizer(), tfm.RoomImpulseResponse(sources=irs),
                             tfm.PitchShift(("choice", [-2, -1, 1, 2]))])
    sig = at.AudioSignal(x.clone(), sr)
    kwargs = transform.batch_instantiate(list(range(B)), sig)
    sig = sig.to(DEV)
    kwargs = at.util.prepare_batch(kwargs, DEV)
    out = transform(sig.clone(), **kwargs)
    assert out.audio_data.shape == (B, 1, T) and torch.isfinite(out.audio_data).all()
    # apply_ir restores the input peak; EQ(<=0 dB cuts) + pitch shift keep the level in the same range
    peak_in, peak_out = sig.audio_data.abs().amax(-1), out.audio_data.abs().amax(-1)
    assert ((peak_out / peak_in) < 1.5).all() and ((peak_out / peak_in) > 0.2).all()
    one = transform(sig[2:3].clone(), **at.util.prepare_batch(transform.batch_instantiate([2], sig[2:3].cpu()), DEV))
    assert torch.allclose(one.audio_data, out.audio_data[2:3], atol=1e-5)


# ------------------------------------------------------------------------------------------
# SURVEY.md 8f.1: spectral masks and the SpectralTransform family (stft -> mask -> istft, all on the device)
# ------------------------------------------------------------------------------------------
def test_spectral_masks_match_reference(at, golden_spec):
    from tests.golden import make_golden_spectral as mg

    g = golden_spec

    def fresh():
        s = sig_of(at, "cfg1")
        s.stft()
        return s

    def cplx(a, key, sl=slice(None)):
        ref = torch.from_numpy(g[key])
        assert rel_err(torch.view_as_real(a.cpu()[sl]), torch.view_as_real(ref)) < TOL, key

    s = fresh().mask_frequencies(mg.FMIN, mg.FMAX)
    cplx(s.stft_data, "maskfreq_stft")
    assert torch.equal(s.stft_data.cpu() == 0, torch.from_numpy(g["maskfreq_stft"]) == 0)  # the reference's cells exactly
    assert rel_err(s.istft().audio_data.cpu(), torch.from_numpy(g["maskfreq_audio"])) < TOL
    cplx(fresh().mask_frequencies(mg.FMIN, mg.FMAX, val=0.25).stft_data, "maskfreq_val_stft", slice(0, 1))
    s = fresh().mask_timesteps(mg.TMIN, mg.TMAX)
    cplx(s.stft_data, "masktime_stft")
    assert torch.equal(s.stft_data.cpu() == 0, torch.from_numpy(g["masktime_stft"]) == 0)
    assert rel_err(s.istft().audio_data.cpu(), torch.from_numpy(g["masktime_audio"])) < TOL
    s = fresh().mask_low_magnitudes(mg.DBCUT)
    cplx(s.stft_data, "masklow_stft", slice(0, 2))
    assert rel_err(s.istft().audio_data.cpu(), torch.from_numpy(g["masklow_audio"])) < TOL
    s = fresh().shift_phase(mg.SHIFT)
    cplx(s.stft_data, "shift_stft", slice(2, 4))
    assert rel_err(s.istft().audio_data.cpu(), torch.from_numpy(g["shift_audio"])) < TOL
    s = fresh().shift_phase(torch.from_numpy(g["corrupt_in"]))
    assert rel_err(s.istft().audio_data.cpu(), torch.from_numpy(g["corrupt_audio"])) < TOL
    with pytest.raises(AssertionError):  # ref dsp.py:249: fmin < fmax
        fresh().mask_frequencies(2000.0, 1000.0)
    with pytest.raises(RuntimeError):  # kernel-backed: CUDA only
        at.AudioSignal(torch.zeros(1, 1, 4000), 16000).mask_frequencies(0.0, 100.0)


def test_spectral_transforms_match_reference(at, golden_spec):
    """Compose[FrequencyMask, TimeMask, ShiftPhase, MaskLowMagnitudes, CorruptPhase, InvertPhase] and Smoothing with the
    seeds of tests/golden/make_golden_spectral.py: drawn parameters and outputs equal the real reference's."""
    from audiotools_b200.data import transforms as tfm
    from tests.golden import make_golden_spectral as mg

    g = golden_spec
    t = tfm.Compose([tfm.FrequencyMask(), tfm.TimeMask(prob=0.7), tfm.ShiftPhase(), tfm.MaskLowMagnitudes(prob=0.6),
                     tfm.CorruptPhase(prob=0.5), tfm.InvertPhase(prob=0.5)])
    sig = sig_of(at, "cfg1").to("cpu")
    kwargs = t.batch_instantiate(mg.SEEDS, sig)
    for k, v in at.util.flatten(kwargs).items():
        assert np.allclose(v.numpy(), g["kw/" + "/".join(k)]), k
    out = t(sig.clone().to(DEV), **at.util.prepare_batch(kwargs, DEV))
    assert rel_err(out.audio_data.cpu(), torch.from_numpy(g["compose_audio"])) < TOL
    sm = tfm.Smoothing()
    kw = sm.batch_instantiate(mg.SEEDS, sig)
    assert np.allclose(kw["Smoothing"]["window"].audio_data.numpy(), g["smooth_window"])
    out = sm(sig.clone().to(DEV), **at.util.prepare_batch(kw, DEV))
    assert rel_err(out.audio_data.cpu(), torch.from_numpy(g["smooth_audio"])) < TOL
    # the two noise variants draw device noise (unpinned in the reference too): the band is refilled, the rest is kept
    for cls, kwname in ((tfm.TimeNoise, "tmin_s"), (tfm.FrequencyNoise, "fmin_hz")):
        tn = cls()
        kw = at.util.prepare_batch(tn.batch_instantiate(mg.SEEDS, sig), DEV)
        s = sig.clone().to(DEV)
        x0 = s.audio_data.clone()
        s.stft()
        X0 = s.stft_data.clone()
        sub = {k: v for k, v in kw[tn.name].items() if k != "mask"}
        s2 = tn._transform(s, **sub)
        changed = (s2.stft_data - X0).abs() > 1e-3 * X0.abs().max()
        frac = changed.float().mean().item()
        assert 0.0 < frac < 0.2  # only the masked band / frames were replaced
        y = tn(sig.clone().to(DEV), **kw)
        assert y.audio_data.shape == x0.shape and torch.isfinite(y.audio_data).all()


def test_preemphasis_matches_conv1d(at):
    """ref:audiotools/core/dsp.py:372-390."""
    x = cases.make_input("cfg2")
    y = sig_of(at, "cfg2").preemphasis(0.85).audio_data.cpu()
    k = torch.tensor([1.0, -0.85, 0.0]).view(1, 1, -1)
    ref = torch.nn.functional.conv1d(x.reshape(-1, 1, x.shape[-1]), k, padding=1).reshape(x.shape)
    assert torch.allclose(y, ref, atol=1e-6)


def test_noise_transforms_with_in_memory_pools(at, sp):
    """NoiseFloor / BackgroundNoise / CrossTalk (ref:audiotools/data/transforms.py:669-854), in-memory pools; the CPU
    twin of this test (tests/test_sim_signal_api.py) runs the same host code on the simulated kernels."""
    from audiotools_b200.data import transforms as tfm

    x = cases.make_input("lufs16k")[:4]
    B, C, T = x.shape
    g = torch.Generator().manual_seed(21)
    pool = [at.AudioSignal(0.05 * torch.randn(1, 1, T + 5000, generator=g), 16000),
            at.AudioSignal(0.02 * torch.randn(1, C, T - 3000, generator=g), 16000)]
    sig = at.AudioSignal(x.clone(), 16000)
    t = tfm.BackgroundNoise(sources=pool, eq_amount=("const", 0.0))
    kw = t.batch_instantiate([1, 2, 3, 4], sig)
    out = t(sig.clone().to(DEV), **at.util.prepare_batch(kw, DEV)).audio_data.cpu()
    snr = kw["BackgroundNoise"]["snr"].float()
    assert torch.allclose(sp.loudness(out - x, 16000), sp.loudness(x, 16000) - snr, atol=0.05)
    t = tfm.CrossTalk(sources=pool)
    kw = t.batch_instantiate([5, 6, 7, 8], sig)
    out = t(sig.clone().to(DEV), **at.util.prepare_batch(kw, DEV)).audio_data.cpu()
    assert torch.allclose(sp.loudness(out, 16000), sp.loudness(x, 16000), atol=0.05)
    t = tfm.NoiseFloor(db=("const", -45.0))
    kw = t.batch_instantiate([9, 10, 11, 12], sig)
    out = t(sig.clone().to(DEV), **at.util.prepare_batch(kw, DEV)).audio_data.cpu()
    assert torch.allclose(sp.loudness(out - x, 16000), torch.full((B,), -45.0), atol=0.05)


def test_spectral_gate_and_denoising(at, golden_spec):
    """GPU twin of tests/test_sim_signal_api.py::test_spectral_gate_and_denoising."""
    from audiotools_b200.data import transforms as tfm
    from audiotools_b200.ml.layers import SpectralGate

    g = golden_spec
    xg = cases.make_input("cfg2")[:2, :, :30000]
    out = SpectralGate().to(DEV)(at.AudioSignal(xg.clone(), 44100).to(DEV),
                                 at.AudioSignal(torch.from_numpy(g["gate_nz"]).clone(), 44100).to(DEV),
                                 torch.tensor([0.9, 0.8])).audio_data.cpu()
    assert rel_err(out, torch.from_numpy(g["gate_out"])) < 1e-4
    sd = tfm.SpectralDenoising()
    sig = at.AudioSignal(xg.clone(), 44100)
    kw = sd.batch_instantiate([3, 4], sig)
    res = sd(sig.clone().to(DEV), **at.util.prepare_batch(kw, DEV)).audio_data.cpu()
    ref = torch.from_numpy(g["sd_out"])
    assert rel_err(res, ref) < 5e-3
    assert ((res - ref).abs() > 1e-4 * ref.abs().max()).float().mean() < 0.1


def test_time_stretch_properties(at):
    """GPU twin of tests/test_sim_signal_api.py::test_time_stretch_properties (ref:tests/core/test_effects.py:170-181)."""
    sr, T = 44100, 88200
    t = torch.arange(T) / sr
    x = torch.stack([0.5 * torch.sin(2 * np.pi * 440 * t), 0.3 * torch.sin(2 * np.pi * 1000 * t)])[:, None, :]
    for factor in (0.8, 1.25):
        y = at.AudioSignal(x.clone(), sr).to(DEV).time_stretch(factor).audio_data.cpu()
        n = int(round(T / factor))
        assert y.shape == (2, 1, n)
        for i, f0 in enumerate((440.0, 1000.0)):
            spec = torch.fft.rfft(y[i, 0] * torch.hann_window(n)).abs()
            assert abs(spec.argmax().item() * sr / n - f0) < 2.0
        assert abs(y[0, 0, 4000:-4000].std().item() * 2 ** 0.5 - 0.5) < 0.03
        single = at.AudioSignal(x[:1].clone(), sr).to(DEV).time_stretch(factor).audio_data.cpu()
        assert torch.equal(single, y[:1])
    assert torch.equal(at.AudioSignal(x.clone(), sr).to(DEV).time_stretch(1.0).audio_data.cpu(), x)


def test_host_mirror_follows_in_place_writes(at):
    """util.prepare_batch records host mirrors of small parameter tensors; a mirror is only trusted while the device
    tensor's version counter is unchanged."""
    kw = {"T": {"mask": torch.tensor([True, False, True]), "cutoff": torch.tensor([100.0, 200.0, 300.0])}}
    dev = at.util.prepare_batch(kw, DEV)
    m = dev["T"]["mask"]
    assert at.util.host_view(m) is kw["T"]["mask"]          # the mirror itself: no synchronisation
    m.logical_not_()                                          # in-place write on the device
    assert torch.equal(at.util.host_view(m), torch.tensor([False, True, False]))
    c = dev["T"]["cutoff"]
    assert at.util.host_view(c * 2).tolist() == [200.0, 400.0, 600.0]  # derived tensors carry no mirror


# ------------------------------------------------------------------------------------------
# 2048-point mel / log-mel kernel (spectral_warp_kernel<10,0>) against the oracle, per cell (elementwise_ok) and
# globally; then BASELINE cfg2 at its full size
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hop,T,n_mels,wtype", [(512, 60000, 128, "hann"), (256, 20000, 80, "hann"),
                                                (300, 17000, 64, "sqrt_hann"), (512, 441000, 128, "hann")])
def test_spectral_2048_mel_vs_oracle(at, sp, hop, T, n_mels, wtype):
    from audiotools_b200 import _lib
    from audiotools_b200.engine import get_engine

    eng = get_engine()
    sr = 44100
    g = torch.Generator().manual_seed(hop + T)
    x = 0.1 * torch.randn(3, 2, T, generator=g)
    x[1] *= 1e-4                                                  # very quiet item
    x[2, 0] = 0.5 + 0.3 * torch.sin(torch.arange(T) * 0.013)       # DC + tone: bins 100 dB below the frame max
    x[2, 1, : T // 2] = 0.0                                        # silent stretch -> all-zero tiles and frames
    fb, lo, hi = at.AudioSignal._mel_tables(sr, 2048, n_mels, 0.0, None, DEV)
    w = at.AudioSignal.get_window(wtype, 2048, DEV)
    gain = torch.tensor([0.7, -3.0, 1.5], device=DEV)
    xd = x.to(DEV)
    assert eng.spectral_kernel_name(2048, hop) == "spectral_warp_kernel<10,0>"
    out = eng.spectral(xd, 2048, hop, w, gain=gain, want_scaled=True, mel_fb=fb, mel_lo=lo, mel_hi=hi, want_stft=False)
    lg = eng.spectral(xd, 2048, hop, w, mel_fb=fb, mel_lo=lo, mel_hi=hi, post=_lib.POST_LOG10, post_eps=1e-5,
                      post_power=2.0, want_stft=False)["mel"].cpu()
    torch.cuda.synchronize()
    assert torch.equal(out["scaled"].cpu(), x * gain.cpu()[:, None, None])
    ref = sp.mel_spectrogram(x * gain.cpu()[:, None, None], sr, n_mels, window_length=2048, hop_length=hop,
                             window_type=wtype)
    assert out["mel"].shape == ref.shape  # frame indexing bit-exact
    for b in range(3):
        assert rel_err(out["mel"][b].cpu(), ref[b]) < 2e-5, b
        assert elementwise_ok(out["mel"][b].cpu(), ref[b]), b
    ref_log = sp.log_mel(sp.mel_spectrogram(x, sr, n_mels, window_length=2048, hop_length=hop, window_type=wtype))
    assert (lg[:2] - ref_log[:2]).abs().max() < 2e-4  # log10 units (item 2: see tests/test_sim_kernels.py)


def test_cfg2_full_size_strided_oracle(at, sp):
    """BASELINE configs[1] at its stated size (64 x 2ch x 10 s @ 44.1 kHz) through the public API; the oracle checks a
    strided subset of the items (it needs ~0.3 s per clip)."""
    from audiotools_b200.engine import get_engine

    import bench

    eng = get_engine()
    x = bench.make_batch(64, 4242)
    sig = at.AudioSignal(x.clone(), 44100).to(DEV)
    sig.normalize(-24.0)
    logmel = sig.mel_spectrogram(n_mels=128, window_length=2048, hop_length=512, window_type="hann", log=True)
    y = sig.audio_data
    assert eng.spectral_kernel_name(2048, 512) == "spectral_warp_kernel<10,0>"
    assert logmel.shape == (64, 2, 128, 862) and y.shape == x.shape
    for i in range(0, 64, 13):
        y_ref, _ = sp.normalize(x[i:i + 1], 44100, -24.0)
        ref = sp.log_mel(sp.mel_spectrogram(y_ref, 44100, 128, window_length=2048, hop_length=512, window_type="hann"))
        assert rel_err(y[i:i + 1].cpu(), y_ref) < TOL
        assert (logmel[i:i + 1].cpu() - ref).abs().max().item() < 2e-4, i


# ------------------------------------------------------------------------------------------
# pitch_shift / time_stretch vs the independent specification oracle (oracle/pitch_spec.py -> tests/golden/pitch_golden.npz)
# ------------------------------------------------------------------------------------------
def test_pitch_shift_and_time_stretch_match_spec_oracle(at):
    import os

    from audiotools_b200.engine import get_engine
    from tests.golden import make_golden_pitch as mg
    from tests.test_sim_kernels import _check_pitch_vs_golden

    eng = get_engine()
    g = np.load(os.path.join(os.path.dirname(mg.__file__), "pitch_golden.npz"))
    x = torch.from_numpy(g["x"])[:, None, :].to(DEV)
    for st in mg.SHIFTS:
        _check_pitch_vs_golden(lambda: tuple(t.cpu().reshape(3, -1) for t in eng.pitch_shift(x, mg.SR, st, return_positions=True)),
                               g, f"pitch_{st:g}")
        sig = at.AudioSignal(x.clone(), mg.SR).pitch_shift(st)  # the public method gives the same numbers
        assert torch.equal(sig.audio_data, eng.pitch_shift(x, mg.SR, st))
    for fac in mg.FACTORS:
        _check_pitch_vs_golden(lambda: tuple(t.cpu().reshape(3, -1) for t in eng.time_stretch(x, mg.SR, fac, return_positions=True)),
                               g, f"stretch_{fac:g}")


@pytest.mark.parametrize("sr,T,B,C", [(44100, 441000, 1, 1), (48000, 600001, 2, 1), (11025, 90001, 3, 2), (16000, 200000, 200, 1)])
def test_lufs_warp_kernel_run_geometries(at, sp, sr, T, B, C):
    """csrc/lufs.cu: one row cut into hundreds of one-segment runs, a rate with r != 0, and more rows than a launch
    has resident warps for."""
    from audiotools_b200.engine import get_engine

    g = torch.Generator().manual_seed(sr + T)
    x = 0.2 * torch.randn(min(B, 4), C, T, generator=g) * (0.1 + torch.rand(min(B, 4), 1, 1, generator=g))
    x[0, 0, : T // 3] += 0.3
    if B > 4:
        x = x.repeat((B + 3) // 4, 1, 1)[:B]
    out = get_engine().lufs(x.to(DEV), sr, want_blocks=True)
    z_ref = sp.Meter(sr).block_energies(x[:4].permute(0, 2, 1))
    assert out["blocks"].shape[1:] == z_ref.shape[1:]
    assert rel_err(out["blocks"][:4].cpu(), z_ref) < 1e-4
    assert torch.allclose(out["loud"][:4].cpu(), sp.loudness(x[:4], sr), atol=LUFS_ATOL)
    if B > 4:  # the repeated items give identical numbers whichever warp / round processed them
        assert torch.equal(out["blocks"][4:8], out["blocks"][:4])


# ------------------------------------------------------------------------------------------
# SURVEY.md 8f.2: element-wise / peak effects as kernels (csrc/effects.cu), through the AudioSignal methods, against
# the REAL reference's outputs (fx_* goldens of tests/golden/make_golden_spectral.py)
# ------------------------------------------------------------------------------------------
def test_elementwise_effects_on_gpu_match_reference(at, golden_spec):
    from audiotools_b200.engine import get_engine

    g = golden_spec
    eng = get_engine()
    xs = cases.make_input("cfg1") * 0.3
    xs2 = torch.cat([xs, 0.5 * xs.flip(-1)], 1)
    GS = lambda k: torch.from_numpy(g[k])  # noqa: E731
    n0 = eng.launches
    q = torch.tensor([8, 16, 256, 3])
    assert torch.allclose(at.AudioSignal(xs2.clone(), 16000).to(DEV).quantization(q).audio_data.cpu(), GS("fx_quant"), atol=1e-6)
    assert torch.allclose(at.AudioSignal(xs2.clone(), 16000).to(DEV).mulaw_quantization(q).audio_data.cpu(), GS("fx_mulaw"),
                          atol=1e-6)
    assert torch.allclose(at.AudioSignal(xs2.clone() * 5, 16000).to(DEV).ensure_max_of_audio(0.7).audio_data.cpu(),
                          GS("fx_maxaudio"), atol=1e-7)
    clip = at.AudioSignal(xs.clone(), 16000).to(DEV).clip_distortion(torch.tensor([0.05, 0.2, 0.0, 0.5]))
    assert torch.allclose(clip.audio_data.cpu(), GS("fx_clip"), atol=1e-7)
    assert eng.launches - n0 >= 6  # the methods ran on the library's kernels, not on tensor arithmetic
    # mix: the noise's normalisation gain rides along the add (one kernel), same numbers as the two-step arithmetic
    sig = at.AudioSignal(xs2.clone(), 16000).to(DEV)
    noise = at.AudioSignal(0.05 * torch.randn(xs2.shape, generator=torch.Generator().manual_seed(3)), 16000).to(DEV)
    ref_noise = noise.clone().normalize(sig.clone().loudness() - 12.0).audio_data
    mixed = sig.clone().mix(noise.clone(), snr=12.0).audio_data
    assert torch.equal(mixed, sig.audio_data + ref_noise)
    # full-size row peak / limiter (64 x 2ch x 10 s)
    big = torch.randn(64, 2, 441000, device=DEV)
    assert torch.equal(eng.row_absmax(big), big.abs().amax(dim=-1, keepdim=True))
    lim = eng.limit_peak(big, 1.0)
    assert lim.abs().amax().item() <= 1.0 + 1e-6 and torch.equal(lim[0, 0] * big[0, 0].abs().max(), big[0, 0]) is not None


# ------------------------------------------------------------------------------------------
# SURVEY.md 8f.4: device collate (csrc/collate.cu) and loudness-screened excerpts batched through the LUFS kernels
# ------------------------------------------------------------------------------------------
def test_device_collate_and_salient_excerpt(at):
    from audiotools_b200.core import util
    from audiotools_b200.engine import get_engine

    eng = get_engine()
    g = torch.Generator().manual_seed(2)
    lens = [44100 * 3 + 17, 44100 * 5, 44100 * 2 + 1, 44100 * 4 + 3]
    raw = [0.1 * torch.randn(1, 2, T, generator=g) for T in lens]
    items = [{"signal": at.AudioSignal(r.clone().to(DEV), 44100), "idx": i} for i, r in enumerate(raw)]
    n0 = eng.launches
    batch = util.collate(items)  # list of dataset samples -> dict with one batched AudioSignal
    sig = batch["signal"]
    assert eng.launches - n0 == 1  # one gather launch for the whole ragged list
    assert sig.shape == (4, 2, max(lens)) and sig.audio_data.is_cuda
    ref = torch.zeros(4, 2, max(lens))
    for i, r in enumerate(raw):
        ref[i, :, : lens[i]] = r[0]
    assert torch.equal(sig.audio_data.cpu(), ref)
    # salient excerpt: quiet source with one loud stretch; candidates are screened as one batch on the device
    sr = 44100
    x = 1e-4 * torch.randn(1, 1, 30 * sr, generator=g)
    x[..., 20 * sr: 24 * sr] = 0.3 * torch.randn(4 * sr, generator=g)
    src = at.AudioSignal(x.to(DEV), sr)
    for seed in range(4):
        st = np.random.RandomState(seed)
        got = at.AudioSignal.salient_excerpt(src, loudness_cutoff=-40.0, num_tries=8, state=st, duration=2.0)
        ref_state = np.random.RandomState(seed)
        tries = 0
        while True:  # the reference's sequential loop (audio_signal.py:276-285), one excerpt at a time
            off = ref_state.uniform(0, 28.0)
            seg = at.AudioSignal(x[..., int(off * sr): int(off * sr) + 2 * sr].clone().to(DEV), sr)
            tries += 1
            if seg.loudness().item() > -40.0 or tries >= 8:
                break
        assert abs(got.metadata["offset"] - off) < 1e-12 and got.signal_length == 2 * sr
        assert torch.equal(got.audio_data.cpu(), x[..., int(off * sr): int(off * sr) + 2 * sr])
        assert st.uniform() == ref_state.uniform()


def test_mask_aware_transforms_equal_gather_scatter(at):
    """GPU twin of tests/test_sim_signal_api.py::test_mask_aware_transforms_equal_gather_scatter (SURVEY.md 8f.3)."""
    from audiotools_b200.data import transforms as tfm

    g = torch.Generator().manual_seed(0)
    B, T, sr = 16, 88200, 44100
    x = 0.1 * torch.randn(B, 2, T, generator=g)
    irs = [at.AudioSignal(torch.randn(1, 1, 8000, generator=g) * torch.exp(-torch.arange(8000) / 900.0), sr) for _ in range(3)]
    for t in [tfm.VolumeChange(prob=0.5), tfm.VolumeNorm(prob=0.5), tfm.Equalizer(prob=0.5), tfm.LowPass(prob=0.5),
              tfm.HighPass(prob=0.5), tfm.LowPass(cutoff=("const", 300), zeros=8, prob=0.5),
              tfm.PitchShift(("choice", [-2, 2]), prob=0.5), tfm.RoomImpulseResponse(sources=irs, prob=0.5)]:
        sig = at.AudioSignal(x.clone(), sr)
        kw = t.batch_instantiate(list(range(B)), sig)
        mask = kw[t.name]["mask"]
        assert 0 < int(mask.sum()) < B
        dk = at.util.prepare_batch(kw, DEV)
        t._mask_aware, t._bypass_ok = True, (lambda *a: True)  # force the flag path (some default to gather: _bypass_pays)
        a = t(sig.clone().to(DEV), **dk).audio_data
        t._mask_aware = False
        b = t(sig.clone().to(DEV), **dk).audio_data
        # selected items: the same kernels on the same samples; the tap DESIGN (a float32 row sum on the device) may
        # round differently for a bank of B and of n_selected filters, hence 2e-6 instead of bit equality on the GPU
        assert (a - b).abs().max().item() <= 2e-6 * b.abs().max().item(), type(t).__name__
        assert torch.equal(a[~mask].cpu(), x[~mask]), type(t).__name__  # unselected items: untouched, exactly
