"""The AudioSignal / transforms layer driven end to end ON THE CPU: the product's host code with the engine swapped for
the CPU-simulated build of the same kernel sources (tests/cusim).  This is what the `-m gpu` tests check on an H100,
repeated here at the goldens' small sizes so that host-side regressions (argument plumbing, deferred gains, masks,
match_stride trimming, per-item grouping) show up without a GPU."""
import numpy as np
import pytest
import torch

import audiotools_b200
import audiotools_b200.engine as engine_mod
from audiotools_b200 import AudioSignal
from audiotools_b200.data import transforms as tfm
from oracle import signal_path as sp
from tests.conftest import rel_err
from tests.cusim.sim_engine import sim_engine
from tests.golden import cases

TOL = 1e-4


@pytest.fixture(autouse=True)
def _sim_engine(monkeypatch):
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    yield


def sig_of(name, sl=slice(None), **kw):
    return AudioSignal(cases.make_input(name)[sl].clone(), cases.sample_rate(name), **kw)


def G(golden, key):
    return torch.from_numpy(golden[key])


def test_stft_istft_and_match_stride(golden):
    sig = sig_of("cfg1", slice(0, 2))
    assert rel_err(torch.view_as_real(sig.stft()), torch.view_as_real(G(golden, "cfg1_stft")[:2])) < TOL
    assert rel_err(sig.istft().audio_data, G(golden, "cfg1_istft")) < TOL
    sig = sig_of("cfg1", slice(0, 2), stft_params=audiotools_b200.STFTParams(256, 64, "sqrt_hann", True, "reflect"))
    assert rel_err(torch.view_as_real(sig.stft()), torch.view_as_real(G(golden, "cfg1_stft_match_stride"))) < TOL
    assert rel_err(sig.istft().audio_data, G(golden, "cfg1_istft_match_stride")) < TOL


def test_normalize_mel_deferred_gain(golden):
    sig = sig_of("cfg2")
    sig.normalize(-24.0)
    logmel = sig.mel_spectrogram(n_mels=128, window_length=2048, hop_length=512, log=True)
    assert rel_err(logmel, G(golden, "cfg2_logmel")) < TOL
    assert rel_err(sig.audio_data, G(golden, "cfg2_norm")) < TOL


def test_mix_matches_restated_reference():
    """EffectMixin.mix (ref:audiotools/core/effects.py:27-64): pad / truncate the other signal, normalise it to
    loudness(self) - snr, add."""
    x = cases.make_input("lufs16k")            # [B, C, T] @ 16 kHz
    g = torch.Generator().manual_seed(9)
    noise = 0.05 * torch.randn(x.shape[0], x.shape[1], x.shape[2] - 1234, generator=g)
    snr = torch.tensor([5.0, 15.0, 25.0, 10.0]).repeat(x.shape[0] // 4 + 1)[: x.shape[0]]
    out = AudioSignal(x.clone(), 16000).mix(AudioSignal(noise.clone(), 16000), snr).audio_data
    other = torch.nn.functional.pad(noise, (0, 1234))
    tgt = sp.loudness(x, 16000) - snr
    ref = x + sp.normalize(other, 16000, tgt)[0]
    assert rel_err(out, ref) < TOL


def test_apply_ir_and_compose_match_reference(golden):
    ir = cases.make_ir()
    drr = G(golden, "drr")
    out = sig_of("fir").apply_ir(AudioSignal(ir.clone(), 44100), drr=drr, ir_eq=golden["eq_db"]).audio_data
    assert rel_err(out, G(golden, "applyir_full")) < TOL
    transform = tfm.Compose([tfm.VolumeNorm(db=("uniform", -30, -16)), tfm.Equalizer(prob=0.5), tfm.LowPass(prob=0.7),
                             tfm.HighPass(prob=0.6), tfm.VolumeChange()])
    sig = sig_of("tfm")
    kwargs = transform.batch_instantiate([10, 11, 12, 13], sig)
    assert rel_err(transform(sig.clone(), **kwargs).audio_data, G(golden, "tfm_out")) < TOL


def test_spectral_family_matches_reference(golden_spec):
    from tests.golden import make_golden_spectral as mg

    g = golden_spec

    def fresh():
        s = sig_of("cfg1")
        s.stft()
        return s

    assert rel_err(fresh().mask_frequencies(mg.FMIN, mg.FMAX).istft().audio_data, G(g, "maskfreq_audio")) < TOL
    assert rel_err(fresh().mask_timesteps(mg.TMIN, mg.TMAX).istft().audio_data, G(g, "masktime_audio")) < TOL
    assert rel_err(fresh().mask_low_magnitudes(mg.DBCUT).istft().audio_data, G(g, "masklow_audio")) < TOL
    assert rel_err(fresh().shift_phase(mg.SHIFT).istft().audio_data, G(g, "shift_audio")) < TOL
    assert rel_err(fresh().shift_phase(G(g, "corrupt_in")).istft().audio_data, G(g, "corrupt_audio")) < TOL
    t = tfm.Compose([tfm.FrequencyMask(), tfm.TimeMask(prob=0.7), tfm.ShiftPhase(), tfm.MaskLowMagnitudes(prob=0.6),
                     tfm.CorruptPhase(prob=0.5), tfm.InvertPhase(prob=0.5)])
    sig = sig_of("cfg1")
    kwargs = t.batch_instantiate(mg.SEEDS, sig)
    assert rel_err(t(sig.clone(), **kwargs).audio_data, G(g, "compose_audio")) < TOL
    sm = tfm.Smoothing()
    kw = sm.batch_instantiate(mg.SEEDS, sig)
    assert rel_err(sm(sig.clone(), **kw).audio_data, G(g, "smooth_audio")) < TOL


def test_preemphasis_and_pitch_transform():
    x = cases.make_input("short")  # [2, 1, 4000] @ 16 kHz
    y = AudioSignal(x.clone(), 16000).preemphasis(0.85).audio_data
    k = torch.tensor([1.0, -0.85, 0.0]).view(1, 1, -1)
    assert torch.allclose(y, torch.nn.functional.conv1d(x.reshape(-1, 1, 4000), k, padding=1).reshape(x.shape), atol=1e-7)
    xm = torch.cat([x, x.flip(0), x], 0).repeat(1, 1, 3)  # 6 items, 12000 samples
    t = tfm.PitchShift(("choice", [-2, 0, 2]))
    sig = AudioSignal(xm.clone(), 16000)
    kw = t.batch_instantiate(list(range(6)), sig)
    shifts = kw["PitchShift"]["n_semitones"].tolist()
    out = t(sig.clone(), **kw).audio_data
    for i, s in enumerate(shifts):  # one set of launches for the batch == each item on its own
        assert torch.equal(out[i:i + 1], AudioSignal(xm[i:i + 1].clone(), 16000).pitch_shift(s).audio_data)


def test_noise_transforms_with_in_memory_pools():
    """NoiseFloor / BackgroundNoise / CrossTalk (ref:audiotools/data/transforms.py:669-854) with in-memory pools: the
    same arithmetic as the reference's transforms (mix / normalize), restated with the oracle."""
    x = cases.make_input("lufs16k")[:4]  # [4, C, T] @ 16 kHz
    B, C, T = x.shape
    g = torch.Generator().manual_seed(21)
    pool = [AudioSignal(0.05 * torch.randn(1, 1, T + 5000, generator=g), 16000),
            AudioSignal(0.02 * torch.randn(1, C, T - 3000, generator=g), 16000)]
    sig = AudioSignal(x.clone(), 16000)

    t = tfm.BackgroundNoise(sources=pool, eq_amount=("const", 0.0))  # eq of 0 dB: the band filters sum to identity
    kw = t.batch_instantiate([1, 2, 3, 4], sig)
    bg = kw["BackgroundNoise"]["bg_signal"].audio_data
    assert bg.shape == x.shape
    out = t(sig.clone(), **kw).audio_data
    snr = kw["BackgroundNoise"]["snr"].float()
    noise = sp.normalize(sp.equalizer(bg, 16000, kw["BackgroundNoise"]["eq"].float()), 16000, sp.loudness(x, 16000) - snr)[0]
    assert rel_err(out, x + noise) < TOL
    assert torch.allclose(sp.loudness(out - x, 16000), sp.loudness(x, 16000) - snr, atol=0.05)

    t = tfm.CrossTalk(sources=pool)
    kw = t.batch_instantiate([5, 6, 7, 8], sig)
    out = t(sig.clone(), **kw).audio_data
    assert torch.allclose(sp.loudness(out, 16000), sp.loudness(x, 16000), atol=0.05)  # original loudness restored
    assert rel_err(out, x) > 1e-2                                                     # ... and something was mixed in

    t = tfm.NoiseFloor(db=("const", -45.0))
    kw = t.batch_instantiate([9, 10, 11, 12], sig)
    out = t(sig.clone(), **kw).audio_data
    assert torch.allclose(sp.loudness(out - x, 16000), torch.full((B,), -45.0), atol=0.05)
    # seeded: the same seeds give the same noise
    kw2 = t.batch_instantiate([9, 10, 11, 12], sig)
    assert torch.equal(kw["NoiseFloor"]["nz_signal"].audio_data, kw2["NoiseFloor"]["nz_signal"].audio_data)


def test_features_filters_and_meter_match_reference(golden):
    """The remaining AudioSignal methods of the hot path through the simulated kernels, against the real reference."""
    assert rel_err(sig_of("cfg1").mfcc(), G(golden, "cfg1_mfcc")) < TOL
    sig = sig_of("cfg1", slice(0, 2))
    sig.stft()
    assert rel_err(sig.log_magnitude(), G(golden, "cfg1_logmag")) < TOL
    lu = sig_of("lufs16k").loudness()
    assert torch.allclose(lu, G(golden, "lufs16k"), atol=1e-3)
    x = cases.make_input("lufs16k")
    meter = audiotools_b200.Meter(16000)
    raw = meter.integrated_loudness(x[:3].permute(0, 2, 1))  # [nb, nt, nch], un-clamped
    assert torch.allclose(raw.clamp(min=-70.0), lu[:3], atol=1e-3)
    cut = G(golden, "fir_cut")
    assert rel_err(sig_of("fir").low_pass(cut).audio_data, G(golden, "lp_peritem")) < TOL
    assert rel_err(sig_of("fir").high_pass(cut / 8).audio_data, G(golden, "hp_peritem")) < TOL
    assert rel_err(sig_of("fir").equalizer(golden["eq_db"]).audio_data, G(golden, "eq_out")) < TOL
    assert rel_err(sig_of("fir", slice(0, 1)).mel_filterbank(4)[:, :1], G(golden, "fbank4")) < TOL
    assert rel_err(sig_of("fir").convolve(AudioSignal(cases.make_ir().clone(), 44100)).audio_data, G(golden, "conv_out")) < TOL
    rs = AudioSignal(cases.make_input("rs")[..., :22050].clone(), 44100).resample(16000)
    assert rs.sample_rate == 16000 and rel_err(rs.audio_data, G(golden, "rs_44k_16k")) < TOL


def test_spectral_gate_and_denoising(golden_spec):
    """ml.layers.SpectralGate / transforms.SpectralDenoising (ref:audiotools/ml/layers/spectral_gate.py:10-127,
    ref:audiotools/data/transforms.py:1539-1592).  The gate is a hard threshold: with identical inputs it reproduces the
    reference to rounding; through the transform (noise normalised + equalised first) a few borderline cells flip, in
    the reference's own CPU-vs-GPU runs as well, so that output is compared loosely."""
    from audiotools_b200.ml.layers import SpectralGate

    g = golden_spec
    xg = cases.make_input("cfg2")[:2, :, :30000]
    out = SpectralGate()(AudioSignal(xg.clone(), 44100), AudioSignal(G(g, "gate_nz").clone(), 44100),
                         torch.tensor([0.9, 0.8])).audio_data
    assert rel_err(out, G(g, "gate_out")) < 1e-5
    sd = tfm.SpectralDenoising()
    sig = AudioSignal(xg.clone(), 44100)
    kw = sd.batch_instantiate([3, 4], sig)
    for kk, v in audiotools_b200.util.flatten(kw).items():
        v = v.audio_data if hasattr(v, "audio_data") else v
        assert np.allclose(v.numpy(), g["sdkw/" + "/".join(kk)]), kk
    res = sd(sig.clone(), **kw).audio_data
    ref = G(g, "sd_out")
    assert rel_err(res, ref) < 5e-3
    assert ((res - ref).abs() > 1e-4 * ref.abs().max()).float().mean() < 0.1


def test_time_stretch_properties():
    """EffectMixin.time_stretch (ref:audiotools/core/effects.py:279-309; SoX there, unpinned): duration / factor, pitch and
    level unchanged, batch == single (ref:tests/core/test_effects.py:170-181), factor 1 copies."""
    sr, T = 16000, 12000
    t = torch.arange(T) / sr
    x = torch.stack([0.5 * torch.sin(2 * np.pi * 440 * t), 0.3 * torch.sin(2 * np.pi * 1000 * t)])[:, None, :]
    for factor in (0.8, 1.25):
        y = AudioSignal(x.clone(), sr).time_stretch(factor).audio_data
        n = int(round(T / factor))
        assert y.shape == (2, 1, n)
        for i, (f0, a0) in enumerate(((440.0, 0.5), (1000.0, 0.3))):
            seg = y[i, 0, 1500:n - 1500].double().numpy()
            k = np.arange(1500, n - 1500) / sr
            A = np.stack([np.sin(2 * np.pi * f0 * k), np.cos(2 * np.pi * f0 * k)], 1)
            coef = np.linalg.lstsq(A, seg, rcond=None)[0]
            spec = torch.fft.rfft(y[i, 0] * torch.hann_window(n)).abs()
            assert abs(spec.argmax().item() * sr / n - f0) < 4.0  # the pitch did not move
            assert abs(np.hypot(*coef) - a0) < 0.05 * a0 or (seg.std() * np.sqrt(2) - a0) < 0.05 * a0
        assert torch.equal(AudioSignal(x[:1].clone(), sr).time_stretch(factor).audio_data, y[:1])
    assert torch.equal(AudioSignal(x.clone(), sr).time_stretch(1.0).audio_data, x)
    with pytest.raises(NotImplementedError):
        AudioSignal(x.clone(), sr).time_stretch(8.0)


def test_excerpt_and_salient_excerpt_semantics():
    """ref:audiotools/core/audio_signal.py:178-286 on an in-memory source: the offset is ONE uniform draw from the
    caller's state, the loudness screen keeps drawing until a window is above the cut-off (at most num_tries), and the
    state ends up where the reference's sequential loop would leave it."""
    sr = 16000
    x = torch.zeros(1, 1, 10 * sr)
    x[..., 6 * sr: 8 * sr] = 0.3 * torch.randn(2 * sr, generator=torch.Generator().manual_seed(0))  # loud only in [6 s, 8 s)
    src = AudioSignal(x, sr)
    st = np.random.RandomState(5)
    expect_off = np.random.RandomState(5).uniform(0, 10 - 1.0)
    e = AudioSignal.excerpt(src, duration=1.0, state=st)
    assert e.signal_length == sr and abs(e.metadata["offset"] - expect_off) < 1e-12
    assert torch.equal(e.audio_data[0, 0], x[0, 0, int(expect_off * sr): int(expect_off * sr) + sr])
    # sequential reference loop, re-stated: draw, measure, stop at the first window above the cut-off
    for seed in range(6):
        ref_state = np.random.RandomState(seed)
        tries, off = 0, None
        while True:
            off = ref_state.uniform(0, 9.0)
            seg = AudioSignal(x[..., int(off * sr): int(off * sr) + sr].clone(), sr)
            tries += 1
            if seg.loudness().item() > -40.0 or tries >= 8:
                break
        st = np.random.RandomState(seed)
        got = AudioSignal.salient_excerpt(src, loudness_cutoff=-40.0, num_tries=8, state=st, duration=1.0)
        assert abs(got.metadata["offset"] - off) < 1e-12, seed
        assert st.uniform() == ref_state.uniform(), seed  # both states advanced by the same number of draws
    with pytest.raises(NotImplementedError):
        AudioSignal.salient_excerpt("some/file.wav", loudness_cutoff=-40, duration=1.0)


def test_batch_collates_ragged_signals_in_one_launch():
    """AudioSignal.batch (ref:audiotools/core/audio_signal.py:380-470) on the engine: pad / truncate + concatenate is
    one gather launch, and the inputs end up padded / truncated like after the reference's in-place calls."""
    g = torch.Generator().manual_seed(2)
    mk = lambda b, T: AudioSignal(torch.randn(b, 2, T, generator=g), 16000)  # noqa: E731
    sigs = [mk(1, 900), mk(2, 1200), mk(1, 640)]
    raw = [s.audio_data.clone() for s in sigs]
    eng = engine_mod.get_engine()
    n0 = eng.launches
    out = AudioSignal.batch(sigs, pad_signals=True)
    assert eng.launches - n0 == 1 and out.shape == (4, 2, 1200)
    ref = torch.zeros(4, 2, 1200)
    ref[0, :, :900], ref[1:3], ref[3, :, :640] = raw[0][0], raw[1], raw[2][0]
    assert torch.equal(out.audio_data, ref)
    assert [s.signal_length for s in sigs] == [1200, 1200, 1200] and torch.equal(sigs[2].audio_data[0], ref[3])
    sigs = [mk(1, 900), mk(1, 640)]
    raw = [s.audio_data.clone() for s in sigs]
    out = AudioSignal.batch(sigs, truncate_signals=True)
    assert out.shape == (2, 2, 640) and torch.equal(out.audio_data, torch.cat([raw[0][..., :640], raw[1]]))
    with pytest.raises(RuntimeError):
        AudioSignal.batch([mk(1, 900), mk(1, 640)])


def test_mask_aware_transforms_equal_gather_scatter():
    """SURVEY.md 8f.3: a transform with a partial mask runs on the WHOLE batch with per-item bypass flags inside the
    kernels (no gather / scatter of the selected items, ref:audiotools/data/transforms.py:133-166) and must leave
    exactly the state the reference's ``signal[mask] = transform(signal[mask])`` leaves: selected items bit-identical
    to the gathered run, the others untouched."""
    g = torch.Generator().manual_seed(0)
    B, T, sr = 5, 6000, 16000
    x = 0.1 * torch.randn(B, 2, T, generator=g)
    irs = [AudioSignal(torch.randn(1, 1, 800, generator=g) * torch.exp(-torch.arange(800) / 100.0), sr) for _ in range(2)]
    cases_ = [tfm.VolumeChange(prob=0.5), tfm.VolumeNorm(prob=0.5), tfm.Equalizer(prob=0.5),
              tfm.LowPass(cutoff=("choice", [2000, 4000]), prob=0.5), tfm.HighPass(prob=0.5),
              tfm.LowPass(cutoff=("const", 200), zeros=8, prob=0.5),  # 641 taps: the FFT-convolution path
              tfm.PitchShift(("choice", [-2, 2]), prob=0.5), tfm.RoomImpulseResponse(sources=irs, prob=0.5)]
    for t in cases_:
        assert t._mask_aware == getattr(t, "_bypass_pays", True)
        t._mask_aware, t._bypass_ok = True, (lambda *a: True)  # force the flag path for every transform
        sig = AudioSignal(x.clone(), sr)
        kw = t.batch_instantiate(list(range(B)), sig)
        mask = kw[t.name]["mask"]
        assert 0 < int(mask.sum()) < B
        a = t(sig.clone(), **kw).audio_data
        t._mask_aware = False  # the reference's gather -> transform -> scatter
        b = t(sig.clone(), **kw).audio_data
        assert torch.equal(a, b), type(t).__name__
        assert torch.equal(a[~mask], x[~mask]), type(t).__name__


def test_arbitrary_window_lengths_match_reference():
    """stft / istft / mel_spectrogram / mfcc with windows that are not powers of two (dense-DFT kernels, csrc/dft.cu)
    against the REAL reference's outputs (tests/golden/make_golden_anywindow.py): frame counts exactly, values to 1e-4."""
    import os

    from tests.golden import make_golden_anywindow as mg

    g = np.load(os.path.join(os.path.dirname(mg.__file__), "reference_golden_anywindow.npz"))
    for key, wl, hop, wt, ms, pt in mg.STFT_CASES:
        sig = sig_of("cfg1")
        X = sig.stft(window_length=wl, hop_length=hop, window_type=wt, match_stride=ms, padding_type=pt)
        ref = torch.from_numpy(g[key + "_stft"])
        assert X.shape[1:] == ref.shape[1:] and X.shape[0] == 4, key  # frame indexing bit-exact
        assert rel_err(torch.view_as_real(X[:2]), torch.view_as_real(ref)) < TOL, key
        y = sig.istft(window_length=wl, hop_length=hop, window_type=wt, match_stride=ms).audio_data
        assert rel_err(y, torch.from_numpy(g[key + "_istft"])) < TOL, key
    mel = sig_of("cfg1").mel_spectrogram(n_mels=80, window_length=400, hop_length=160, window_type="hann")
    assert rel_err(mel, torch.from_numpy(g["w400_mel80"])) < TOL
    mf = sig_of("cfg1").mfcc(n_mfcc=20, n_mels=40, window_length=400, hop_length=160, window_type="hann")
    assert rel_err(mf, torch.from_numpy(g["w400_mfcc"])) < TOL


def test_impulse_response_augmentation_properties():
    """ref:tests/core/test_effects.py:305-329 on a synthetic room response (the reference's wav is an LFS pointer):
    solve_alpha == 1 at the measured DRR; alter_drr hits a scalar and per-item target DRRs; shapes of the split."""
    g = torch.Generator().manual_seed(11)
    sr, T, B = 16000, 8000, 6
    t = torch.arange(T) / sr
    h = 0.2 * torch.randn(1, 1, T, generator=g) * torch.exp(-t / 0.08)
    h[..., 60] = 1.0
    ir_batch = AudioSignal(h.repeat(B, 1, 1), sr)
    early, late, window = ir_batch.decompose_ir()
    assert early.shape == late.shape == window.shape
    drr = ir_batch.measure_drr()
    alpha = AudioSignal.solve_alpha(early, late, window, drr)
    assert np.allclose(alpha.numpy(), 1.0, atol=1e-5)
    out = ir_batch.deepcopy().alter_drr(5)
    assert np.allclose(out.measure_drr().numpy(), 5.0, atol=1e-4)
    target = torch.from_numpy(np.random.RandomState(0).rand(B).astype("float32") * 50)
    out = ir_batch.deepcopy().alter_drr(target)
    assert np.allclose(out.measure_drr().numpy().flatten(), target.numpy(), atol=1e-3)


@pytest.mark.parametrize("mulaw", [False, True])
def test_quantization_level_counts(mulaw):
    """ref:tests/core/test_effects.py:262-302: a signal quantised to q channels holds at most q distinct levels
    (rounded to 3 decimals, as the reference does for the straight-through residual), per item and for a scalar q."""
    g = torch.Generator().manual_seed(3)
    x = (0.2 * torch.randn(8, 1, 4000, generator=g)).clamp(-0.99, 0.99)  # (a sample at +1.0 is a (q+1)-th level in the reference too)
    q = np.random.RandomState(0).choice([2, 4, 8, 16, 32, 64, 128], size=(8,), replace=True)
    sig = AudioSignal(x.clone(), 16000)
    out = (sig.mulaw_quantization(q) if mulaw else sig.quantization(q)).audio_data
    for i, qc in enumerate(q):
        assert len(np.unique(np.around(out[i].numpy(), decimals=3))) <= qc, (i, qc)
    for qc in (2, 16, 128):
        sig = AudioSignal(x[:1].clone(), 16000)
        o = (sig.mulaw_quantization(qc) if mulaw else sig.quantization(qc)).audio_data
        assert len(np.unique(np.around(o.numpy(), decimals=3))) <= qc
