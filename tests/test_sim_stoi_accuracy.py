"""The STOI per-stage accuracy checks of tests/test_gpu_stoi_accuracy.py on the CPU-simulated build of csrc/stoi.cu
(tests/cusim), with the same module and budgets (tests/stoi64.py): rows of at most about 1 s except where M needs more,
and a subset of the rates; plus the workspace layouts against the library, which need no kernel."""
import numpy as np
import pytest

import audiotools_b200.engine as engine_mod
import tests.test_gpu_stoi_accuracy as G
from tests import stoi64 as s
from tests.cusim.sim_engine import sim_engine


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    return sim_engine()


def test_workspace_layouts_match_the_library():
    lib = sim_engine().lib
    for B, T, sr in ((1, 257, 10000), (3, 16000, 16000), (2, 44101, 44100), (5, 99999, 7999), (7, 12345, 12345),
                     (4, 310_000_000, 10000)):
        up, down = s.Engine.stoi_ratio(sr)
        L = s.Layout(B, T, up, down)
        assert lib.b2a_stoi_workspace_bytes(B, T, up, down) == L.bytes
        assert lib.b2a_stoi_backward_workspace_bytes(B, T, up, down) == L.bwd_bytes


@pytest.mark.parametrize("sr", [8000, 10000, 12345, 22050, 44100, 96000])
def test_every_stage_at_every_rate(eng, sr):
    G.check_rate(eng, sr, 0.8)


@pytest.mark.parametrize("sr", [8000, 10000, 7999])
def test_resampler_tiles(eng, sr):
    G.check_resampler_tiles(eng, sr)


def test_gradient_input_tiles(eng):
    G.check_input_tiles(eng, 8000)


@pytest.mark.parametrize("n_fr", [1, 2, 255, 256, 257, 513])
def test_mask_scan_chunks(eng, n_fr):
    G.check_mask_chunks(eng, n_fr)


@pytest.mark.parametrize("M", [0, 1, 29, 30, 31, 32, 33, 46, 47, 36, 38, 64, 65])
def test_band_tiles_and_score_shapes(eng, M):
    G.check_m(eng, M)


@pytest.mark.parametrize("sr,bad,value", G.NONFINITE)
def test_nonfinite_inputs(eng, sr, bad, value):
    G.check_nonfinite(eng, sr, bad, value)


def test_batch_rows_equal_single_items(eng):
    G.check_batch_rows(eng, [0, 1, 29, 30, 31, 200, 47])


def test_power_of_two_scaling(eng):
    G.check_power_of_two_scaling(eng, 10000, 9000)
    G.check_power_of_two_scaling(eng, 44100, 30000)


def test_restatement_resampler_sends_no_gradient_through_padding():
    """The float64 restatement's gather gives a NaN in the 10 kHz gradient to the input samples its taps reach and
    to no other: in particular not to sample 0 through the zero-padding slots."""
    import torch
    from tests import stoi_grad_cases as sg

    x = torch.zeros(4000, dtype=torch.float64, requires_grad=True)
    y = sg.resample(x, 16000)
    g = torch.zeros_like(y)
    g[1000] = float("nan")
    (gx,) = torch.autograd.grad(y, x, g)
    bad = np.nonzero(~np.isfinite(gx.numpy()))[0]
    assert bad.size > 0 and 0 not in bad and bad.min() > 1000
