"""The effect-kernel accuracy checks of tests/test_gpu_effects_accuracy.py on the CPU-simulated build of csrc/effects.cu,
dft.cu and collate.cu (tests/cusim), with the same module and budgets (tests/effects64.py), at the sizes a CPU can run:
every stride edge, the NaN and overflow cases and the refusals.  Host libm stands in for libdevice here, so mu-law
samples are classified rather than compared bit for bit."""
import numpy as np
import pytest
import torch

import tests.test_gpu_effects_accuracy as G
from tests import effects64 as o
from tests.cusim.sim_engine import sim_engine


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    return sim_engine()


@pytest.mark.parametrize("T", G.OS_T)
def test_order_stats_exact(eng, T):
    G.test_order_stats_exact(eng, T)


@pytest.mark.parametrize("T", [1, 2, 1025, 4096])
@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("sign", [1, -1])
def test_order_stats_and_quantile_nan(eng, T, where, sign):
    G.check_nan_rows(eng, T, where, sign)


def test_order_stats_k_count_limit(eng):
    G.test_order_stats_k_count_limit(eng)


@pytest.mark.parametrize("T", [1, 2, 1023, 1024, 1025, 10 ** 5])
def test_quantile(eng, T):
    G.test_quantile(eng, T)


@pytest.mark.parametrize("nan_row", [0, 2])
def test_clip_distortion_nan(eng, nan_row):
    """clip_distortion's engine path (quantiles of row 0, then the clamp) against the reference's expressions."""
    x = torch.from_numpy(G.rng(9).standard_normal((3, 1, 4000)).astype(np.float32)) * 0.3
    x[nan_row, 0, 17] = float("nan")
    q = torch.tensor([0.1, 0.2, 0.05])
    thr = eng.quantile(x[0, 0], torch.cat([q / 2, 1 - q / 2]))
    got = eng.clamp_items(x, thr[:3], thr[3:])
    want = x.clamp(torch.quantile(x, q / 2, dim=-1)[:, :1, :], torch.quantile(x, 1 - q / 2, dim=-1)[:, :1, :])
    assert torch.equal(got.isnan(), want.isnan())
    assert torch.equal(got.nan_to_num(), want.nan_to_num())


@pytest.mark.parametrize("T", G.DRR_T)
def test_alter_drr_strides(eng, T):
    G.test_alter_drr_strides(eng, T)


@pytest.mark.parametrize("where", ["0", "t0", "T-1-t0", "T-1"])
def test_alter_drr_direct_path_at_row_ends(eng, where):
    G.test_alter_drr_direct_path_at_row_ends(eng, where)


def test_alter_drr_edges(eng):
    G.test_alter_drr_t0_zero_and_short_rows(eng)
    G.test_alter_drr_tied_maxima_and_negative_response(eng)
    G.test_alter_drr_second_channel_beyond_t0(eng)
    G.test_alter_drr_target_edges(eng)


@pytest.mark.parametrize("C", [1, 2, 5])
def test_alter_drr_channels(eng, C):
    G.test_alter_drr_channels(eng, C)


@pytest.mark.parametrize("where", ["window", "early", "late", "channel0"])
def test_alter_drr_nan(eng, where):
    G.test_alter_drr_nan(eng, where)


@pytest.mark.parametrize("mulaw", [True, False])
@pytest.mark.parametrize("q", G.Q_LEVELS)
def test_quantize_level_boundaries(eng, q, mulaw):
    G.test_quantize_level_boundaries(eng, q, mulaw)


@pytest.mark.parametrize("mulaw", [True, False])
def test_quantize_per_item_and_q1(eng, mulaw):
    G.test_quantize_per_item_and_q1(eng, mulaw)


@pytest.mark.parametrize("mulaw", [True, False])
@pytest.mark.parametrize("n", [4096, 4097, 4098, 4099])
def test_quantize_walks(eng, n, mulaw):
    G.test_quantize_walks(eng, n, mulaw)


@pytest.mark.parametrize("T", G.PS_T)
def test_peak_scale_strides(eng, T):
    G.test_peak_scale_strides(eng, T)


def test_peak_scale_edges(eng):
    G.test_peak_scale_ties_and_row_ends(eng)
    G.test_peak_scale_limit_edges(eng)


def test_peak_scale_bypass_and_many_rows(eng):
    G.test_peak_scale_bypass_and_many_rows(eng)


@pytest.mark.parametrize("where", [0, 137, 299])
@pytest.mark.parametrize("restore", [False, True])
def test_peak_scale_nan(eng, where, restore):
    G.test_peak_scale_nan(eng, where, restore)


def test_limit_peak_with_nan(eng):
    """ensure_max_of_audio's engine path with a NaN sample: the peak is NaN, so the gain is 1, as in the reference."""
    x = torch.from_numpy(G.rng(34).standard_normal((2, 1, 500)).astype(np.float32)) * 2
    x[1, 0, 77] = float("nan")
    got = eng.limit_peak(x, 1.0)
    peak = x.abs().max(dim=-1, keepdim=True)[0]
    gain = torch.ones_like(peak)
    gain[peak > 1] = 1 / peak[peak > 1]
    assert torch.equal(got.nan_to_num(), (x * gain).nan_to_num()) and torch.equal(got.isnan(), (x * gain).isnan())


@pytest.mark.parametrize("n_mfcc", G.MFCC)
def test_mel_dct_coefficient_chunks(eng, n_mfcc):
    for n_mels in G.MELS:
        for N in [1, 127, 128, 129]:
            G.check_dct(eng, 1, n_mels, n_mfcc, N, n_mfcc * 1000 + n_mels + N)


@pytest.mark.parametrize("n_mfcc,n_mels", [(80, 40), (33, 128)])
def test_mel_dct_transposed_basis(eng, n_mfcc, n_mels):
    G.test_mel_dct_transposed_basis(eng, n_mfcc, n_mels)


def test_mel_dct_largest_basis_and_refusals(eng):
    G.test_mel_dct_largest_basis_and_refusals(eng)


@pytest.mark.parametrize("T_out", [4, 1024, 1021, 1022, 1023])
def test_pack_rows_tails_offsets_strides(eng, T_out):
    G.test_pack_rows_tails_offsets_strides(eng, T_out)


def test_pack_rows_row_limit(eng):
    G.test_pack_rows_row_limit(eng)


def test_refusals_through_the_c_abi(eng):
    G.test_refusals_through_the_c_abi(eng)


def test_reruns_bit_identical(eng):
    G.test_reruns_bit_identical(eng)


def test_batch_equals_single_items(eng):
    G.test_batch_equals_single_items(eng)


def test_power_of_two_scaling_is_exact(eng):
    G.test_power_of_two_scaling_is_exact(eng)


def test_oracle_sanity():
    """The oracles against torch on finite data."""
    row = G.rng(1).standard_normal(999).astype(np.float32)
    q = [0.0, 0.1, 0.5, 0.77, 1.0]
    v, *_ = o.quantile(row, q)
    assert np.allclose(v, torch.quantile(torch.from_numpy(row), torch.tensor(q)).double().numpy(), rtol=1e-6)
    assert o.same_values(o.order_stats(np.array([np.nan, -0.0, 0.0, -np.inf], np.float32), [0, 1, 2, 3]),
                         [-np.inf, 0.0, 0.0, np.nan])
