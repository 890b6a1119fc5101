"""The spectral-mask accuracy checks of tests/test_gpu_specmask_accuracy.py on the CPU-simulated build of
csrc/specmask.cu (tests/cusim), with the same module and budgets (tests/specmask64.py), at the sizes a CPU can run:
every tile edge up to 65 frames and 33 bins (257 frames for the band masks' block sizes), one case past the
grid-stride cap, and every non-finite case."""
import pytest
import torch

import tests.test_gpu_specmask_accuracy as G
from tests.cusim.sim_engine import sim_engine

F_SIM = [1, 15, 16, 17, 33]
N_SIM = [1, 63, 64, 65, 255, 256, 257]


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    return sim_engine()


@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("F", F_SIM)
def test_band_masks_bit_for_bit(eng, F, axis):
    for N in N_SIM:
        G.check_band(eng, F, N, axis)


@pytest.mark.parametrize("shape,per_cell,smax", [((3, 2, 33, 70), True, 3.0), ((4, 1, 17, 65), False, 1e4),
                                                  ((3, 1, 513, 400), True, 1e4)])
def test_rotate_per_cell(eng, shape, per_cell, smax):
    G.check_rotate(eng, shape, per_cell, smax)


@pytest.mark.parametrize("val", [0.0, 0.5])
def test_mask_low_random(eng, val):
    G.check_mask_low(eng, G.ramped((3, 2, 17, 65), 66), torch.linspace(-60.0, -20.0, 3), val, val)


def test_mask_low_past_the_grid_cap(eng):
    G.check_mask_low(eng, G.ramped((3, 1, 513, 400), 401), torch.tensor([-60.0, -40.0, -20.0]), 0.5, "cap")


@pytest.mark.parametrize("val", [0.0, 0.5])
def test_mask_low_near_the_cutoff(eng, val):
    G.test_mask_low_near_the_cutoff(eng, val)


def test_mask_low_floor_silence_and_infinite_cutoffs(eng):
    G.test_mask_low_loud_item_sets_the_floor_of_a_quiet_one(eng)
    G.test_mask_low_all_silent(eng)
    G.test_mask_low_infinite_cutoffs(eng, float("inf"))
    G.test_mask_low_infinite_cutoffs(eng, float("-inf"))


@pytest.mark.parametrize("F", [1, 15, 16, 17, 33])
def test_gate_tiles(eng, F):
    for N in [1, 63, 64, 65, 130]:
        G.gate_case(eng, 2, 2, F, N, (1, 1, F, 50), F + N, hf=3, ht=5)


@pytest.mark.parametrize("hf", G.HALVES)
def test_gate_smoothing_widths(eng, hf):
    for ht in G.HALVES:
        G.gate_case(eng, 2, 1, 17, 65, (1, 1, 17, 50), 3 * hf + ht + 17, hf=hf, ht=ht)


@pytest.mark.parametrize("F,N", [(33, 130), (17, 65)])
def test_gate_asymmetric_smoothing_orientation(eng, F, N):
    G.test_gate_asymmetric_smoothing_orientation(eng, F, N)


@pytest.mark.parametrize("nz_shape", [(1, 1), (3, 1), (1, 2), (3, 2)])
def test_gate_noise_shapes(eng, nz_shape):
    G.gate_case(eng, 3, 2, 17, 65, nz_shape + (17, 50), 31, amount=(1.0, 0.3, 0.8))


@pytest.mark.parametrize("nz_N", G.NZ_FRAMES)
def test_gate_noise_frames(eng, nz_N):
    G.test_gate_noise_frames(eng, nz_N)


@pytest.mark.parametrize("amount", [(0.0,), (1.0,), (0.25, 1.0)])
def test_gate_amounts(eng, amount):
    G.test_gate_amounts(eng, amount)


def test_gate_silent_noise_and_signal(eng):
    G.test_gate_silent_noise_and_signal(eng)


@pytest.mark.parametrize("where,value", G.NONFINITE)
def test_gate_nonfinite(eng, where, value):
    G.check_gate_nonfinite(eng, where, value)


@pytest.mark.parametrize("imag", [False, True])
@pytest.mark.parametrize("value", G.MASK_LOW_NONFINITE, ids=["nan", "-nan", "inf", "-inf"])
def test_mask_low_nonfinite(eng, value, imag):
    G.check_mask_low_nonfinite(eng, value, imag)


def test_refusals_before_any_launch(eng):
    G.check_refusals(eng)


def test_reruns_bit_identical(eng):
    G.check_reruns(eng)
