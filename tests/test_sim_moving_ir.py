"""The moving impulse response checks of tests/test_gpu_moving_ir.py on the CPU-simulated build of the kernels
(tests/cusim), with the same oracle and budget (tests/moving_ir64.py), plus the oracle's own check and the transform
(``SyntheticRoomImpulseResponse(source_speed=...)``).  The workspace-chunk and at-size cases run on the H100 only."""
import numpy as np
import pytest
import torch

import audiotools_b200.engine as engine_mod
import tests.test_gpu_moving_ir as G
from tests import moving_ir64 as M
from tests import timedomain64 as td
from tests.cusim.sim_engine import sim_engine


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    return sim_engine()


def test_oracle_identical_waypoints_are_convolve():
    g = torch.Generator().manual_seed(0)
    for C, n_ch, T, L, hop in ((2, 2, 5000, 1500, 1024), (3, 1, 5000, 7000, 1500), (1, 1, 900, 300, 1024)):
        x = torch.randn(2, C, T, generator=g)
        ir = torch.randn(2, 1, n_ch, L, generator=g)
        K = (T - 1) // hop + 1
        y, scale = M.moving_ir64(x, ir.expand(2, K, n_ch, L), hop)
        y0, scale0 = td.circconv64(x, ir[:, 0].reshape(2 * n_ch, L), 1 if n_ch == C else C)
        assert np.abs(y - y0).max() <= 1e-12 * np.abs(y0).max()
        if K == 1:
            assert np.allclose(scale, scale0, rtol=1e-12)


def test_oracle_weights_sum_to_one():
    for T, hop in ((1, 1024), (5000, 1024), (7001, 3001), (4000, 4000)):
        v = M.path_weights(T, (T - 1) // hop + 1, hop)
        assert (v >= 0).all() and np.allclose(v.sum(0), 1.0, atol=1e-15)


@pytest.mark.parametrize("shape", G.SHAPES)
def test_path_per_block(eng, shape):
    assert G.check_path(eng, *shape) <= 1.0, shape


def test_path_bypass(eng):
    assert G.check_path(eng, 3, 2, 2, 6000, 2000, 1300, bypass=[False, True, False]) <= 1.0


@pytest.mark.parametrize("shape", [(2, 2, 2, 6144, 1500, 1024), (1, 2, 1, 3000, 2500, 4000),
                                   (1, 1, 1, 3000, 700, 4000), (2, 5, 1, 7001, 1024, 3001)])
def test_identical_waypoints_are_convolve(eng, shape):
    assert G.check_identical_waypoints(eng, *shape) <= 1.0, shape


def test_batch_equals_items_and_reruns(eng):
    G.check_batch_equals_items(eng, 3, 2, 1, 9000, 2500, 1100)
    G.check_batch_equals_items(eng, 3, 2, 2, 9000, 700, 2048)


def test_apply_moving_ir(eng):
    G.check_apply_moving_ir(4, 2, 1, 6000, 2500, 1536)
    G.check_apply_moving_ir(2, 2, 2, 6000, 2500, 1536, use_original_phase=True)


def test_refusals(eng):
    G.check_refusals(eng)


def test_launch_counts(eng):
    G.check_launches(eng)


def test_bad_arguments_launch_nothing_in_the_real_library(eng):
    lib = eng.lib
    x = torch.zeros(2, 3000)
    ir = torch.zeros(2, 3, 1000)
    out = torch.zeros(2, 3000)
    ws = torch.zeros(lib.b2a_circconv_path_workspace_bytes(2, 3000, 3, 1000, 1, 1, 1024), dtype=torch.uint8)
    p = lambda t: t.data_ptr()  # noqa: E731
    bad = [
        dict(hop=1023), dict(K=2), dict(K=4), dict(L=3001), dict(rows_per_ir=2, rows=3), dict(ir_channels=3),
        dict(ir_channels=0), dict(ws_bytes=16),
    ]
    for b in bad:
        a = dict(rows=2, K=3, L=1000, rows_per_ir=1, ir_channels=1, hop=1024, ws_bytes=ws.numel())
        a.update(b)
        lib0 = lib.kernel_launches.value
        rc = lib.b2a_circconv_path_f32(p(x), a["rows"], 3000, p(ir), a["K"], a["L"], a["rows_per_ir"],
                                       a["ir_channels"], a["hop"], 1,
                                       None, p(out), p(ws), a["ws_bytes"], None)
        assert rc != 0, b
        assert lib.kernel_launches.value == lib0, b


def test_transform_static_unchanged(eng):
    G.check_static_unchanged(G._speech(3, 2, 8000), 16000)


def test_transform_paths(eng):
    G.check_paths(G._speech(6, 2, 12000), 16000)


@pytest.mark.parametrize("kw", [{}, {"diffuse_after": 0.02}, {"bands": 3}])
def test_transform_batch_equals_instantiate(eng, kw):
    G.check_batch_equals_instantiate(G._speech(3, 2, 8000), 16000, **kw)


def test_transform_default_hop_at_16k(eng):
    G.check_default_hop_low_rate(G._speech(2, 2, 8000), 16000)


def test_transform_bad_speed_and_hop(eng):
    G.check_bad_speed_and_hop(G._speech(1, 2, 8000), 16000)


def test_transform_shared_tail_seed(eng, monkeypatch):
    G.check_shared_tail_seed(G._speech(2, 2, 8000), 16000, monkeypatch)


def test_transform_bands_chunked(eng, monkeypatch):
    # MAX_ROWS lowered to 100: 2 items x 2 microphones x 8 bands x 8 waypoints = 256 rows
    G.check_bands_chunked(G._speech(2, 2, 8000), 16000, monkeypatch, max_rows=100)
