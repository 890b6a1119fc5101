"""Kernel launch counts on the CPU-simulated build of the kernels (tests/cusim).  ``b2a_kernel_launches`` is counted
inside ``B2A_LAUNCH`` in both builds, so the simulator counts what the GPU build launches.  Every engine method must
add to ``Engine.launches`` exactly what the library counted for the call, and each count is pinned here: the counts
include/b2a.h states (STOI, the LARGE / DENSE STFT with gain and mel), those of the overlap-save engine of
csrc/fftconv.cu (no frequency-domain FIR launch with one filter partition), and nothing for a rejected call."""
import pytest
import torch

from audiotools_b200 import AudioSignal, _lib
from tests.cusim.sim_engine import sim_engine

SR = 16000


@pytest.fixture(scope="module")
def eng():
    return sim_engine()


def _randn(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def _counted(eng, fn):
    """(kernels the library launched during fn(), what the engine added to ``launches``)."""
    lib0, eng0 = eng.lib.kernel_launches.value, eng.launches
    fn()
    return eng.lib.kernel_launches.value - lib0, eng.launches - eng0


def _spectral(eng, n_fft, hop, gain, mel):
    x = _randn(2, 2, 6 * n_fft, seed=n_fft)
    win = AudioSignal.get_window("hann", n_fft, "cpu")
    kw = {}
    if gain:
        kw.update(gain=torch.tensor([0.5, 2.0]), want_scaled=True)
    if mel:
        kw.update(zip(("mel_fb", "mel_lo", "mel_hi"), AudioSignal._mel_tables(SR, n_fft, 32, 0.0, None, "cpu")))
    if eng.route(n_fft, hop, 0) == _lib.ROUTE_DENSE:
        eng.dft_matrix(win, n_fft, inverse=0)  # built once per window, not part of the counted call
    return lambda: eng.spectral(x, n_fft, hop, win, **kw)


FFT, LARGE, DENSE = (512, 128), (8192, 2048), (500, 125)
SPECTRAL = {  # (geometry, gain, mel) -> launches: one fused pass on FFT; gain pass, STFT and mel on LARGE / DENSE
    (FFT, False, False): 1, (FFT, True, False): 1, (FFT, False, True): 1, (FFT, True, True): 1,
    (LARGE, False, False): 1, (LARGE, True, False): 2, (LARGE, False, True): 2, (LARGE, True, True): 3,
    (DENSE, False, False): 1, (DENSE, True, False): 2, (DENSE, False, True): 2, (DENSE, True, True): 3,
}


@pytest.mark.parametrize("geometry,gain,mel", sorted(SPECTRAL))
def test_spectral(eng, geometry, gain, mel):
    n = SPECTRAL[geometry, gain, mel]
    assert _counted(eng, _spectral(eng, *geometry, gain, mel)) == (n, n)


def test_dft_matrix_is_built_once(eng):
    win = AudioSignal.get_window("hann", 600, "cpu")
    assert _counted(eng, lambda: eng.dft_matrix(win, 600, inverse=1)) == (1, 1)
    assert _counted(eng, lambda: eng.dft_matrix(win, 600, inverse=1)) == (0, 0)


def _inverse_cases(eng, n_fft, hop):
    """The inverse STFT and the three backward passes of one geometry (matrices built up front on DENSE)."""
    x = _randn(1, 2, 6 * n_fft, seed=hop)
    win = AudioSignal.get_window("hann", n_fft, "cpu")
    fb, lo, hi = AudioSignal._mel_tables(SR, n_fft, 32, 0.0, None, "cpu")
    if eng.route(n_fft, hop, 1) == _lib.ROUTE_DENSE:
        for inverse in (0, 1, 2):
            eng.dft_matrix(win, n_fft, inverse=inverse)
    X = eng.spectral(x, n_fft, hop, win)["stft"]
    N, T = X.shape[-1], x.shape[-1]
    gm = _randn(1, 2, 32, N, seed=1)
    return {
        "istft": lambda: eng.istft(X, n_fft, hop, win, T),
        "stft_backward": lambda: eng.stft_backward(X, T, n_fft, hop, win),
        "istft_backward": lambda: eng.istft_backward(x, N, n_fft, hop, win),
        "mel_backward": lambda: eng.mel_backward(X, gm, fb, lo, hi),
    }


INVERSE = {  # (geometry, method) -> launches
    (FFT, "istft"): 1, (FFT, "stft_backward"): 2, (FFT, "istft_backward"): 3, (FFT, "mel_backward"): 1,
    (LARGE, "istft"): 2, (LARGE, "stft_backward"): 3, (LARGE, "istft_backward"): 3, (LARGE, "mel_backward"): 1,
    (DENSE, "istft"): 2, (DENSE, "stft_backward"): 3, (DENSE, "istft_backward"): 3, (DENSE, "mel_backward"): 1,
}


@pytest.mark.parametrize("geometry,method", sorted(INVERSE))
def test_inverse_and_backward(eng, geometry, method):
    n = INVERSE[geometry, method]
    assert _counted(eng, _inverse_cases(eng, *geometry)[method]) == (n, n)


def _spec(seed=0, shape=(2, 1, 33, 20)):
    return torch.complex(_randn(*shape, seed=seed), _randn(*shape, seed=seed + 1))


LAUNCHES = {  # method (and variant) -> launches
    "spectral_loss": 2, "spectral_loss_mel": 2,
    "spec_band_mask": 1, "spec_band_mask_out": 1, "spec_band_mask_backward": 1, "spec_rotate": 1,
    "spec_mask_low": 2, "spec_mask_low_out": 2, "spec_mask_low_backward": 1,  # global maximum, then the mask
    "spec_gate": 2, "spec_gate_backward": 1,
    "lufs": 2, "loudness_stats": 3,
    "gain": 1, "row_absmax": 1, "limit_peak": 2, "limit_peak_given_peak": 1, "peak_scale_backward": 1, "mix": 1,
    "quantize": 1, "quantize_mulaw": 1, "quantile": 1, "clamp_items": 1, "mel_dct": 1,
    "pack_rows": 1, "fir_direct": 1, "fir_pad_fold": 2,
    # fill, filter FFT, then per chunk of rows: origins, block FFT, (the FIR over partitions when P > 1,) inverse FFT
    "fftconv_P1": 5, "fftconv_P2": 6,
    # + the IR's peak (and, backward, the tap reversal)
    "circular_convolve_P1": 6, "circular_convolve_P2": 7,
    "circular_convolve_backward_P1": 7, "circular_convolve_backward_P2": 8,
    "resample": 1, "resample_decimating": 1, "resample_backward": 2, "resample_backward_T2": 1,
    "pitch_shift": 4, "pitch_shift_per_item": 4, "pitch_shift_zero": 0,
    "time_stretch_1": 1, "time_stretch": 4,
    "stoi": 4, "stoi_one_frame": 3, "stoi_backward": 4, "stoi_backward_one_frame": 3,  # n10 <= 384: no band launch
    "alter_drr": 1,
}


@pytest.fixture(scope="module")
def calls(eng):
    """method (and variant) -> a call of it on small inputs; what the calls need is computed up front."""
    x, y = _randn(2, 1, 4000, seed=1), _randn(2, 1, 4000, seed=2)
    X, G = _spec(3), _spec(5)
    fvals, tvals = torch.linspace(0, SR / 2, 33), torch.linspace(0, 0.1, 20)
    lo, hi, cut = torch.tensor([100.0, 2000.0]), torch.tensor([900.0, 5000.0]), torch.tensor([-30.0])
    win = AudioSignal.get_window("hann", 256, "cpu")
    mel = AudioSignal._mel_tables(SR, 256, 32, 0.0, None, "cpu")
    ws_low = eng.spec_mask_low_out(X, cut)[1]
    nz, smooth = _spec(7, (1, 1, 33, 12)), [0.5, 1.0, 0.5]
    thresh = eng.spec_gate(X, nz, 1.5, 0.5, smooth, smooth)[1]
    peak = eng.row_absmax(x)
    taps = _randn(1, 31, seed=9)
    short_ir, long_ir = _randn(1, 1, 500, seed=10), _randn(1, 1, 1500, seed=11)
    est, ref = _randn(1, 1, 16000, seed=12), _randn(1, 1, 16000, seed=13)
    est10, ref10 = _randn(1, 1, 300, seed=14), _randn(1, 1, 300, seed=15)
    ws16 = eng.stoi(est, ref, 16000, return_workspace=True)[3]
    ws10 = eng.stoi(est10, ref10, 10000, return_workspace=True)[3]
    one = torch.ones(1, dtype=torch.float64)
    return {
        "spectral_loss": lambda: eng.spectral_loss(x, y, 256, 64, win),
        "spectral_loss_mel": lambda: eng.spectral_loss(x, y, 256, 64, win, mel=mel, want_grad_x=True),
        "spec_band_mask": lambda: eng.spec_band_mask(X.clone(), fvals, lo, hi, 0),
        "spec_band_mask_out": lambda: eng.spec_band_mask_out(X, tvals, lo / 1e4, hi / 1e4, 1),
        "spec_band_mask_backward": lambda: eng.spec_band_mask_backward(G, X, fvals, lo, hi, 0),
        "spec_rotate": lambda: eng.spec_rotate(X.clone(), torch.tensor([0.3, -1.0])),
        "spec_mask_low": lambda: eng.spec_mask_low(X.clone(), cut),
        "spec_mask_low_out": lambda: eng.spec_mask_low_out(X, cut),
        "spec_mask_low_backward": lambda: eng.spec_mask_low_backward(G, X, cut, 0.0, ws_low),
        "spec_gate": lambda: eng.spec_gate(X, nz, 1.5, 0.5, smooth, smooth),
        "spec_gate_backward": lambda: eng.spec_gate_backward(G, X, thresh, 0.5, smooth, smooth),
        "lufs": lambda: eng.lufs(x, SR, target_db=torch.tensor([-24.0]), want_blocks=True),
        "loudness_stats": lambda: eng.loudness_stats(_randn(1, 2, 4 * SR, seed=16), SR, want_series=True),
        "gain": lambda: eng.gain(x, torch.tensor([0.5, 2.0])),
        "row_absmax": lambda: eng.row_absmax(x),
        "limit_peak": lambda: eng.limit_peak(x, 0.5),
        "limit_peak_given_peak": lambda: eng.limit_peak(x, 0.5, peak),
        "peak_scale_backward": lambda: eng.peak_scale_backward(y, x, x_ref=y),
        "mix": lambda: eng.mix(x, y, torch.tensor([0.5, 2.0])),
        "quantize": lambda: eng.quantize(x, torch.tensor([8.0])),
        "quantize_mulaw": lambda: eng.quantize(x, torch.tensor([16.0, 256.0]), mulaw=True),
        "quantile": lambda: eng.quantile(x.reshape(-1), torch.tensor([0.1, 0.9])),
        "clamp_items": lambda: eng.clamp_items(x, torch.tensor([-0.5, -1.0]), torch.tensor([0.5, 1.0])),
        "mel_dct": lambda: eng.mel_dct(_randn(1, 2, 32, 10, seed=17), _randn(32, 13, seed=18)),
        "pack_rows": lambda: eng.pack_rows([x[0], y[:, :, :900], x[1, :, :100]], 1000),
        "fir_direct": lambda: eng.fir_direct(x, taps, rows_per_filt=2, left0=15),
        "fir_pad_fold": lambda: eng.fir_pad_fold(y, taps, rows_per_filt=2, left0=15, grad_x=torch.zeros_like(y)),
        "fftconv_P1": lambda: eng.fftconv(x, _randn(1, 1024, seed=19), rows_per_filt=2),
        "fftconv_P2": lambda: eng.fftconv(x, _randn(1, 1025, seed=20), rows_per_filt=2),
        "circular_convolve_P1": lambda: eng.circular_convolve(x, short_ir),
        "circular_convolve_P2": lambda: eng.circular_convolve(x, long_ir),
        "circular_convolve_backward_P1": lambda: eng.circular_convolve_backward(y, short_ir),
        "circular_convolve_backward_P2": lambda: eng.circular_convolve_backward(y, long_ir),
        "resample": lambda: eng.resample(x, 16000, 24000),
        "resample_decimating": lambda: eng.resample(x, 48000, 16000),  # the decimating fir_direct
        "resample_backward": lambda: eng.resample_backward(_randn(2, 1, 6000, seed=21), 4000, 16000, 24000),
        "resample_backward_T2": lambda: eng.resample_backward(_randn(2, 1, 3, seed=22), 2, 16000, 24000),
        "pitch_shift": lambda: eng.pitch_shift(x, SR, 2.0),
        "pitch_shift_per_item": lambda: eng.pitch_shift(x, SR, [2.0, -3.0]),
        "pitch_shift_zero": lambda: eng.pitch_shift(x, SR, 0.0),  # a copy
        "time_stretch_1": lambda: eng.time_stretch(x, SR, 1.0),
        "time_stretch": lambda: eng.time_stretch(x, SR, 1.25),
        "stoi": lambda: eng.stoi(est, ref, 16000),
        "stoi_one_frame": lambda: eng.stoi(est10, ref10, 10000),
        "stoi_backward": lambda: eng.stoi_backward(one, ws16, est.shape, 16000),
        "stoi_backward_one_frame": lambda: eng.stoi_backward(one, ws10, est10.shape, 10000),
        "alter_drr": lambda: eng.alter_drr(_randn(2, 1, 4000, seed=23), 44100, torch.tensor([5.0])),
    }


@pytest.mark.parametrize("name", sorted(LAUNCHES))
def test_method(eng, calls, name):
    n = LAUNCHES[name]
    assert _counted(eng, calls[name]) == (n, n)


def test_rejected_call_launches_nothing(eng):
    """Argument validation runs before the first launch: the library counts nothing, and neither does the engine."""
    x = _randn(2, 1, 4000, seed=1)
    lib0, eng0 = eng.lib.kernel_launches.value, eng.launches
    with pytest.raises(_lib.B2AError, match="per filter need more than"):
        eng.fftconv(x, _randn(1, 100, seed=2), rows_per_filt=1)  # 2 rows, 1 row per filter, 1 filter
    with pytest.raises(_lib.B2AError, match="null pointer"):
        eng._call(eng.lib.b2a_stoi_f32, None, None, 1, 1, 16000, 0, None, 1, 1, 1, None, None, None, None, 0, None)
    assert (eng.lib.kernel_launches.value - lib0, eng.launches - eng0) == (0, 0)
