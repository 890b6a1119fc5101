"""The spectral accuracy checks of tests/test_gpu_spectral_accuracy.py at small shapes on the CPU-simulated build of
the kernels (tests/cusim), with the same module and budgets (tests/spectral64.py).  The simulator evaluates
sqrt.approx / lg2.approx as sqrtf / log2f and sincospif in double, and g++ does not contract a*b + c into FMAs: a
route that passes here and fails on the H100 differs in one of those instructions."""
import pytest

import tests.test_gpu_spectral_accuracy as G
from tests import spectral64 as s64
from tests.cusim.sim_engine import sim_engine


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    return sim_engine()


def _ours(eng):
    return lambda x, n, hop, w, **kw: eng.spectral(x, n, hop, w, **kw)["stft"]


@pytest.mark.parametrize("n_fft,n_off", [(32, 32), (64, 64), (128, 128), (256, 256), (512, 128), (1024, 64),
                                         (2048, 64), (4096, 32), (8192, 8), (16384, 4), (32768, 4),
                                         (2, 2), (3, 3), (400, 400), (1001, 64), (4095, 16), (8191, 4)])
def test_dft_matrix_by_impulses(eng, n_fft, n_off):
    """Impulses at every offset (small windows) or sampled offsets, against the closed form."""
    offs = s64.impulse_offsets(n_fft, n_off)
    err = s64.impulse_error(_ours(eng), n_fft, offs, "cpu")
    assert err <= s64.impulse_budget(n_fft), (n_fft, err / s64.impulse_budget(n_fft))
    err1 = s64.impulse_error(_ours(eng), n_fft, [1], "cpu")  # the untangle twiddles themselves
    assert err1 <= s64.untangle_budget(n_fft), (n_fft, err1 / s64.U)


@pytest.mark.parametrize("n_fft", [32, 64, 256, 2048, 4096, 3, 400])
def test_forward_per_bin_against_float64(eng, n_fft):
    G.test_forward_per_bin_against_float64(eng, n_fft)


def test_forward_large_window_per_bin(eng):
    """8192 .. 32768 on six frames: noise and the sparse signals within the large route's budget."""
    for n_fft in (8192, 32768):
        hop = n_fft // 4
        sig = s64.signals(n_fft, hop, 6)
        w = s64.windows(n_fft, "cpu")["hann"]
        for name in ("noise", "tones_120dB", "dc"):
            fr, be = s64.frame_errors(eng.spectral(sig[name], n_fft, hop, w)["stft"],
                                      s64.stft_ref(sig[name], n_fft, hop, w))
            err = be.max().item() if name == "noise" else fr.max().item()
            assert err <= s64.budget(n_fft), (n_fft, name, err / s64.budget(n_fft))


@pytest.mark.parametrize("n_fft", [32, 256, 2048, 400])
@pytest.mark.parametrize("pad_mode", ["reflect", "constant", "replicate"])
def test_padding_modes_per_bin(eng, n_fft, pad_mode):
    G.test_padding_modes_per_bin(eng, n_fft, pad_mode)


@pytest.mark.parametrize("n_fft,n_mels,sr", [(2048, 320, 44100), (32, 5, 44100), (400, 40, 44100),
                                             (512, 160, 44100)])
def test_mel_and_log_mel_per_band(eng, n_fft, n_mels, sr):
    G.test_mel_and_log_mel_per_band(eng, n_fft, n_mels, sr)


@pytest.mark.parametrize("n_fft", [32, 64, 2048, 4096, 400])
def test_inverse_per_sample_against_float64(eng, n_fft):
    G.test_inverse_per_sample_against_float64(eng, n_fft)


@pytest.mark.parametrize("n_fft", [32, 256, 4096, 400])
def test_backward_per_element(eng, n_fft):
    G.test_backward_per_element(eng, n_fft)


@pytest.mark.parametrize("n_fft", [32, 256, 2048, 4096, 400])
def test_power_of_two_scaling_is_exact(eng, n_fft):
    G.test_power_of_two_scaling_is_exact(eng, n_fft)


@pytest.mark.parametrize("n_fft", [32, 256, 400])
def test_rows_are_independent(eng, n_fft):
    G.test_rows_are_independent(eng, n_fft)


@pytest.mark.parametrize("n_fft", [32, 256, 2048, 4096, 400])
def test_frame_shift_is_exact(eng, n_fft):
    G.test_frame_shift_is_exact(eng, n_fft)


@pytest.mark.parametrize("n_fft", [64, 256, 512, 2048])
def test_warp_kernel_modes_agree(eng, n_fft):
    G.test_warp_kernel_modes_agree(eng, n_fft)
