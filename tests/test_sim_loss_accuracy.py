"""The loss accuracy checks of tests/test_gpu_loss_accuracy.py at small shapes on the CPU-simulated build of the
kernels (tests/cusim), with the same model and budgets (tests/loss64.py): rows of at most 4000 samples, four rows per
case, every window and both modes, the partial tiles and the exact properties.  The simulator's log10f / powf / sqrtf
are the host's libm, so the same budgets hold; a check that fails on one platform only names one of those."""
import pytest

import tests.test_gpu_loss_accuracy as G
from tests import loss64 as L
from tests import spectral64 as s64
from tests.cusim.sim_engine import sim_engine
from tests.test_sim_metrics import ENGINE_GEOMETRIES, _x

# four rows per case, every kind in turn
SIM_KINDS = [("noise", "tones_120dB", "gap", "same"), ("noise_1e-3", "dc", "x_zero", "nyquist"),
             ("noise", "noise_1e-6", "y_zero", "same"), ("noise", "gap", "dc", "tones_120dB"),
             ("noise_1e-3", "x_zero", "y_zero", "gap")]


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(G, "MAX_T", 4000)
    monkeypatch.setattr(G, "SIM_KINDS", SIM_KINDS)
    return sim_engine()


@pytest.mark.parametrize("mode", ["stft", "mel"])
@pytest.mark.parametrize("n_fft", G.WINDOWS)
def test_cells_and_terms_against_float64(eng, n_fft, mode):
    G.test_cells_and_terms_against_float64(eng, n_fft, mode)


@pytest.mark.parametrize("wl,hop,mel,ms,pt,wt,kw", ENGINE_GEOMETRIES)
def test_engine_geometries_per_cell(eng, wl, hop, mel, ms, pt, wt, kw):
    """The geometries of test_sim_metrics' engine test (T = 3000, 2 x 2 rows of noise), per cell."""
    x, y = _x((2, 2, 3000), wl), _x((2, 2, 3000), wl + 1)
    right_pad, pad = s64.padding(3000, wl, hop, ms)
    w = s64.windows(wl, "cpu")[wt]
    out = L.check(eng, x.reshape(4, 1, -1), y.reshape(4, 1, -1), wl, hop, w, (pad, right_pad, pt, 2 if ms else 0), mel,
                  kinds=["noise"] * 4, **kw)
    L.assert_within(out, "mel" if mel else "stft", (wl, hop, mel))


@pytest.mark.parametrize("mode", ["stft", "mel"])
@pytest.mark.parametrize("n_fft", G.WINDOWS)
def test_swap_symmetry(eng, n_fft, mode):
    G.test_swap_symmetry(eng, n_fft, mode)


@pytest.mark.parametrize("mode", ["stft", "mel"])
@pytest.mark.parametrize("n_fft", G.WINDOWS)
def test_rows_are_independent(eng, n_fft, mode):
    G.test_rows_are_independent(eng, n_fft, mode, R=4)


@pytest.mark.parametrize("mode", ["stft", "mel"])
@pytest.mark.parametrize("n_fft", G.WINDOWS)
def test_tile_phase_is_exact(eng, n_fft, mode):
    G.test_tile_phase_is_exact(eng, n_fft, mode)


@pytest.mark.parametrize("mode", ["stft", "mel"])
@pytest.mark.parametrize("n_fft", [64, 2048])
def test_requests_are_independent(eng, n_fft, mode):
    G.test_requests_are_independent(eng, n_fft, mode)


@pytest.mark.parametrize("mode", ["stft", "mel"])
@pytest.mark.parametrize("n_fft", [64, 512, 2048])
def test_magnitude_only_scaling_is_exact(eng, n_fft, mode):
    G.test_magnitude_only_scaling_is_exact(eng, n_fft, mode)
