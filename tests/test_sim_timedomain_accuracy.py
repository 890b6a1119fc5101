"""The time-domain accuracy checks of tests/test_gpu_timedomain_accuracy.py at small shapes on the CPU-simulated build
of the kernels (tests/cusim), with the same module and budgets (tests/timedomain64.py).  g++ does not contract
a * b + c into FMAs, so a check that fails only on the H100 names an FMA contraction."""
import pytest

import tests.test_gpu_timedomain_accuracy as G
from tests import timedomain64 as td
from tests.cusim.sim_engine import sim_engine


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    return sim_engine()


@pytest.mark.parametrize("K,stride", [(1, 1), (8, 1), (9, 2), (103, 3), (320, 1), (319, 6)])
def test_fir_direct_per_sample(eng, K, stride):
    for T in sorted({1, max(1, K - 1), 2047, 2049}):
        if eng.lib.b2a_fir_direct_supported(T, K, stride):
            c = G.check_fir_direct(eng, T, K, stride)
            assert c <= td.BUDGET_C["fir_direct"], (T, K, stride, c)


@pytest.mark.parametrize("pad_mode", ["replicate", "constant"])
@pytest.mark.parametrize("subtract", [False, True])
def test_fir_direct_pad_subtract_bypass(eng, pad_mode, subtract):
    c = G.check_fir_direct(eng, 3000, 103, 1, pad_mode=pad_mode, subtract=subtract, left0=140, rows=4,
                           bypass=[0, 1, 0, 1])
    assert c <= td.BUDGET_C["fir_direct"], c


def test_fir_direct_largest_stride(eng):
    G.test_fir_direct_largest_stride(eng)


@pytest.mark.parametrize("L", [1, 1023, 1025, 2049, 4097])
def test_fftconv_per_block(eng, L):
    for T in (1, 1024, 1025, 5000):
        c = G.check_fftconv(eng, T, L, offset0=L // 2)
        assert c <= td.BUDGET_C["fftconv"], (T, L, c)


@pytest.mark.parametrize("pad_mode", ["replicate", "constant", "circular"])
def test_fftconv_modes_offsets_scale(eng, pad_mode):
    G.test_fftconv_modes_offsets_scale(eng, pad_mode)


@pytest.mark.parametrize("T,L", [(3000, 3000), (5000, 1200), (2000, 4500), (1, 1)])
def test_circconv_per_block(eng, T, L):
    for roll in (True, False):
        G.test_circconv_per_block(eng, T, L, roll)


def test_circconv_tied_and_tiny_peaks(eng):
    G.test_circconv_tied_and_tiny_peaks(eng)


@pytest.mark.parametrize("old_sr,new_sr", [(48000, 16000), (44100, 22050), (44100, 16000), (16000, 44100),
                                           (8000, 44100), (44100, 8000)])
def test_resample_per_sample(eng, old_sr, new_sr):
    for T in (1, 2, 50, 3000):
        if new_sr * T // old_sr >= 1:
            c = G.check_resample(eng, old_sr, new_sr, T)
            rt = td.resample_route(eng.lib, T, old_sr, new_sr)
            assert c <= td.BUDGET_C[rt], (old_sr, new_sr, T, rt, c)


def test_power_of_two_scaling_is_exact(eng):
    G.test_power_of_two_scaling_is_exact(eng)


@pytest.mark.parametrize("n_rows", [1, 7])
def test_rows_are_independent(eng, n_rows):
    G.test_rows_are_independent(eng, n_rows)


def test_tile_shift_is_exact(eng):
    G.test_tile_shift_is_exact(eng)


@pytest.mark.parametrize("sr", [8000, 22050, 44100, 48000, 192000])
def test_kweight_per_block_against_float64(eng, sr):
    b, v, e = G.check_kweight(eng, sr, int(1.2 * sr), names=["noise", "noise_1e-6", "dc_step", "sin20+noise",
                                                              "sin45+noise", "loud_then_-100dB"])
    assert b <= 1.0, (sr, e.max())
    assert v <= td.KW_VS_SEQ32, (sr, v)


def test_kweight_channels(eng):
    b, v, e = G.check_kweight(eng, 16000, 16000, C=5, names=["noise", "sin30+noise"])
    assert b <= 1.0 and v <= td.KW_VS_SEQ32, (e.max(), v)


@pytest.mark.parametrize("T", [100, 2048, 6401])
def test_kweight_short_rows(eng, T):
    G.test_kweight_short_rows(eng, T)


def test_integrated_loudness_against_float64(eng):
    G.test_integrated_loudness_against_float64(eng, 44100)


@pytest.mark.parametrize("old_sr,new_sr", [(48000, 16000), (44100, 16000), (11025, 96000)])
def test_resample_backward_per_sample(eng, old_sr, new_sr):
    G.test_resample_backward_per_sample(eng, old_sr, new_sr)


def test_equalizer_backward_per_sample(eng):
    G.test_equalizer_backward_per_sample(eng)


@pytest.mark.parametrize("T,L", [(3000, 3000), (2000, 4500)])
def test_circconv_backward_per_block(eng, T, L):
    G.test_circconv_backward_per_block(eng, T, L)
