"""The moving impulse response (``Engine.circular_convolve_moving``, ``AudioSignal.apply_moving_ir``,
``SyntheticRoomImpulseResponse(source_speed=...)``; csrc/fftconv.cu ``path_fir_kernel`` + ``path_ifft_kernel``,
DESIGN.md K22) on the H100 (``-m gpu``) against the float64 oracle of tests/moving_ir64.py, per 1024-sample output
block within ``timedomain64.fft_budget("circconv", min(L, T))``.  The checks are functions of the engine so that
tests/test_sim_moving_ir.py runs them on the CPU-simulated build at small shapes."""
import numpy as np
import pytest
import torch

from tests import moving_ir64 as M
from tests import timedomain64 as td

pytestmark = pytest.mark.gpu

DEV = "cuda:0"

# (B, C, IR channels, T, L, hop): waypoints on block edges (hop 1024, 2048), mid-block (1536), one sample off an edge
# (1025, 2047), a hop that is no multiple of 1024 and a T that is no multiple of the hop (1500, 3001), one waypoint
# (T <= hop), L = 1, L > T (truncated), L over many partitions, 1 / 2 / 5 channels with per-channel and shared IRs
SHAPES = [
    (2, 2, 2, 6144, 1500, 1024),
    (1, 1, 1, 7000, 3000, 2048),
    (2, 2, 1, 6000, 2500, 1536),
    (1, 2, 2, 5000, 700, 1025),
    (1, 1, 1, 9000, 4100, 2047),
    (2, 5, 5, 8000, 2100, 1500),
    (1, 5, 1, 7001, 1024, 3001),
    (2, 2, 2, 3000, 1800, 4000),
    (1, 1, 1, 1024, 1025, 1024),
    (1, 2, 1, 5000, 1, 1100),
    (2, 1, 1, 4000, 6000, 1200),
    (1, 2, 2, 20000, 11000, 1024),
]


def case(B, C, n_ch, T, L, hop, seed=0, identical=False):
    """x [B, C, T] and decaying random IRs [B, K, n_ch, L], on DEV."""
    g = torch.Generator().manual_seed(seed)
    K = (T - 1) // hop + 1
    x = torch.randn(B, C, T, generator=g)
    irs = torch.randn(B, K, n_ch, L, generator=g) * torch.exp(-torch.arange(L) / max(L / 4.0, 1.0))
    if identical:
        irs = irs[:, :1].expand(B, K, n_ch, L).contiguous()
    return x.to(DEV), irs.to(DEV)


def check_path(eng, B, C, n_ch, T, L, hop, seed=0, bypass=None):
    """The worst block error over the budget; bypassed items must come back bit for bit."""
    x, irs = case(B, C, n_ch, T, L, hop, seed)
    y = eng.circular_convolve_moving(x, irs, hop, bypass=None if bypass is None else torch.tensor(bypass, device=DEV))
    ref, scale = M.moving_ir64(x, irs, hop, bypass=bypass)
    if bypass is not None:
        for b, skip in enumerate(bypass):
            if skip:
                assert torch.equal(y[b], x[b])
    return td.block_errors(y, ref, scale).max() / td.fft_budget("circconv", min(L, T))


def check_identical_waypoints(eng, B, C, n_ch, T, L, hop):
    """K copies of one IR give the static circular convolution: within budget, and bit for bit with K = 1 when the IR
    spans more than one partition (the FIR then sums in the static engine's order)."""
    x, irs = case(B, C, n_ch, T, L, hop, seed=3, identical=True)
    y = eng.circular_convolve_moving(x, irs, hop)
    y0 = eng.circular_convolve(x, irs[:, 0])
    ref, scale = td.circconv64(x, irs[:, 0].reshape(B * n_ch, -1), 1 if n_ch == C else C)
    err = td.block_errors(y, ref, scale).max() / td.fft_budget("circconv", min(L, T))
    if irs.shape[1] == 1 and min(L, T) > td.FFT_BLOCK:
        assert torch.equal(y, y0)
    return err


def check_batch_equals_items(eng, B, C, n_ch, T, L, hop):
    x, irs = case(B, C, n_ch, T, L, hop, seed=5)
    y = eng.circular_convolve_moving(x, irs, hop)
    assert torch.equal(y, eng.circular_convolve_moving(x, irs, hop))
    for b in range(B):
        assert torch.equal(y[b:b + 1], eng.circular_convolve_moving(x[b:b + 1].contiguous(), irs[b:b + 1].contiguous(),
                                                                    hop))


def check_apply_moving_ir(B, C, n_ch, T, L, hop, use_original_phase=False):
    """AudioSignal.apply_moving_ir: the path convolution, then every row back at its input peak (apply_ir's rule)."""
    from audiotools_b200 import AudioSignal

    x, irs = case(B, C, n_ch, T, L, hop, seed=7)
    bypass = torch.tensor([i % 2 == 1 for i in range(B)], device=x.device)
    y = AudioSignal(x.clone(), 16000).apply_moving_ir(irs, hop, use_original_phase=use_original_phase,
                                                      _bypass=bypass).audio_data
    if not use_original_phase:  # the phase round trip (stft, istft) runs on every item, as in apply_ir
        for b in range(1, B, 2):
            assert torch.equal(y[b], x[b])
    ref, scale = M.moving_ir64(x, irs, hop, bypass=bypass.cpu().numpy())
    want = M.keep_peak64(x, ref)
    got = y.reshape(B * C, T).cpu().double().numpy()
    rows = ~np.repeat(bypass.cpu().numpy(), C)
    if not use_original_phase:
        gain = np.abs(want).max(-1, keepdims=True) / np.maximum(np.abs(ref).max(-1, keepdims=True), 1e-300)
        err = td.block_errors(got[rows], want[rows], gain[rows] * scale[rows]).max()
        assert err / td.fft_budget("circconv", min(L, T)) <= 2.0, err
    return got


def check_refusals(eng):
    x, irs = case(1, 2, 2, 5000, 600, 1024)
    with pytest.raises(ValueError, match="hop"):
        eng.circular_convolve_moving(x, irs[:, :5], 1000)
    for K in (4, 6):
        with pytest.raises(ValueError, match="waypoints"):
            eng.circular_convolve_moving(x, irs[:, :1].expand(1, K, 2, 600).contiguous(), 1024)
    with pytest.raises(ValueError, match="irs must be"):
        eng.circular_convolve_moving(x, irs[:, :, :1].expand(1, 5, 3, 600).contiguous(), 1024)
    for hop in (1024.0, 1024.5, True):
        with pytest.raises(ValueError, match="an int"):
            eng.circular_convolve_moving(x, irs, hop)
    from audiotools_b200 import AudioSignal

    with pytest.raises(NotImplementedError, match="gradient"):
        AudioSignal(x.clone().requires_grad_(), 16000).apply_moving_ir(irs, 1024)
    with pytest.raises(NotImplementedError, match="gradient"):
        AudioSignal(x.clone(), 16000).apply_moving_ir(irs.clone().requires_grad_(), 1024)


# the library's own launch count for one call: ir_peak + fill_windows, then per chunk of rows: the filter partitions,
# row origins, signal blocks, path FIR and the inverse
def expected_launches(chunks: int) -> int:
    return 2 + 5 * chunks


def check_launches(eng):
    x, irs = case(2, 2, 1, 6000, 2500, 1536)
    lib0, eng0 = eng.lib.kernel_launches.value, eng.launches
    eng.circular_convolve_moving(x, irs, 1536)
    assert (eng.lib.kernel_launches.value - lib0, eng.launches - eng0) == (expected_launches(1),) * 2
    lib0, eng0 = eng.lib.kernel_launches.value, eng.launches
    with pytest.raises(ValueError):
        eng.circular_convolve_moving(x, irs, 1000)
    assert (eng.lib.kernel_launches.value - lib0, eng.launches - eng0) == (0, 0)


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


@pytest.mark.parametrize("shape", SHAPES)
def test_path_per_block(eng, shape):
    assert check_path(eng, *shape) <= 1.0, shape


def test_path_bypass(eng):
    assert check_path(eng, 3, 2, 2, 6000, 2000, 1300, bypass=[False, True, False]) <= 1.0


@pytest.mark.parametrize("shape", [(2, 2, 2, 6144, 1500, 1024), (1, 2, 1, 3000, 2500, 4000),
                                   (1, 1, 1, 3000, 700, 4000), (2, 5, 1, 7001, 1024, 3001)])
def test_identical_waypoints_are_convolve(eng, shape):
    assert check_identical_waypoints(eng, *shape) <= 1.0, shape


def test_batch_equals_items_and_reruns(eng):
    check_batch_equals_items(eng, 3, 2, 1, 9000, 2500, 1100)
    check_batch_equals_items(eng, 3, 2, 2, 9000, 700, 2048)


def test_rows_straddle_workspace_chunks(eng):
    """Per IR the path's spectra take ~114 MB here, so the 256 MB budget holds two IRs: 5 items run in 3 chunks."""
    B, C, n_ch, T, L, hop = 5, 1, 1, 120000, 120000, 1024
    lib0 = eng.lib.kernel_launches.value
    assert check_path(eng, B, C, n_ch, T, L, hop, seed=11) <= 1.0
    assert eng.lib.kernel_launches.value - lib0 == expected_launches(3)
    check_batch_equals_items(eng, 3, 1, 1, T, L, hop)


def test_apply_moving_ir(eng):
    check_apply_moving_ir(4, 2, 1, 6000, 2500, 1536)
    check_apply_moving_ir(2, 2, 2, 6000, 2500, 1536, use_original_phase=True)


def test_refusals(eng):
    check_refusals(eng)


def test_launch_counts(eng):
    check_launches(eng)


def test_at_size_strided_rows(eng):
    """64 items x 2 channels x 10 s at 44.1 kHz, 1 s IRs, hop 0.05 s: every 9th row against the oracle."""
    B, C, T, L, hop = 64, 2, 441000, 44100, 2205
    K = (T - 1) // hop + 1
    g = torch.Generator(device=DEV).manual_seed(0)
    x = torch.randn(B, C, T, generator=g, device=DEV)
    irs = torch.randn(B, K, C, L, generator=g, device=DEV) * torch.exp(-torch.arange(L, device=DEV) / 8000.0)
    y = eng.circular_convolve_moving(x, irs, hop)
    for r in range(0, B * C, 9):
        b, c = divmod(r, C)
        ref, scale = M.moving_ir64(x[b:b + 1, c:c + 1], irs[b:b + 1, :, c:c + 1], hop)
        err = td.block_errors(y[b, c], ref, scale).max() / td.fft_budget("circconv", L)
        assert err <= 1.0, (r, err)


# ------------------------------------------------------------------ SyntheticRoomImpulseResponse(source_speed=...)
def _room_tfm(**kw):
    from audiotools_b200.data import transforms as tfm

    return tfm.SyntheticRoomImpulseResponse(duration=0.05, **kw)


def _run(t, x, sr, states):
    from audiotools_b200 import AudioSignal

    sig = AudioSignal(x.clone(), sr)
    params = t.batch_instantiate(states, sig)
    return t(sig, **params).audio_data, params[t.name]


def check_static_unchanged(x, sr):
    """source_speed=None draws nothing new and gives the static transform's output; speed 0 gives it within 1e-5."""
    y0, p0 = _run(_room_tfm(diffuse_after=0.02), x, sr, [1, 2, 3])
    y1, p1 = _run(_room_tfm(diffuse_after=0.02, source_speed=None), x, sr, [1, 2, 3])
    assert sorted(p0) == sorted(p1) and "end" not in p1 and "speed" not in p1
    assert torch.equal(y0, y1)
    y2, p2 = _run(_room_tfm(diffuse_after=0.02, source_speed=("const", 0.0), waypoint_hop=0.07), x, sr, [1, 2, 3])
    for k in p0:
        if k != "mask":
            assert torch.equal(torch.as_tensor(p0[k]), torch.as_tensor(p2[k])), k
    assert (y2 - y0).abs().max() <= 1e-5 * y0.abs().max()


def check_paths(x, sr):
    t = _room_tfm(source_speed=("uniform", 0.5, 20.0), waypoint_hop=0.07)
    _, p = _run(t, x, sr, list(range(6)))
    src, end, speed = (p[k].cpu().double().numpy() for k in ("source", "end", "speed"))
    room = p["room"].cpu().double().numpy()
    hop = round(0.07 * sr)
    K = (x.shape[-1] - 1) // hop + 1
    path = t.path(src, end, speed, K, hop / sr)
    assert path.shape == (6, K, 3)
    assert (path >= t.margin - 1e-9).all() and (path <= room[:, None] - t.margin + 1e-9).all()
    dist = np.linalg.norm(end - src, axis=-1)
    travelled = np.linalg.norm(path - src[:, None], axis=-1)
    want = np.minimum(speed[:, None] * np.arange(K)[None] * hop / sr, dist[:, None])
    assert np.allclose(travelled, want, atol=1e-9)
    assert (path[want >= dist[:, None]] == np.repeat(end[:, None], K, 1)[want >= dist[:, None]]).all()


def check_batch_equals_instantiate(x, sr, **kw):
    from audiotools_b200 import AudioSignal

    t = _room_tfm(source_speed=("uniform", 1.0, 5.0), waypoint_hop=0.07, **kw)
    y, _ = _run(t, x, sr, [4, 5, 6])
    for b, state in enumerate([4, 5, 6]):
        sig = AudioSignal(x[b:b + 1].clone(), sr)
        yb = t(sig, **t.instantiate(state, sig)).audio_data
        assert torch.equal(yb[0], y[b]), b


def check_default_hop_low_rate(x, sr):
    """Below 20.48 kHz the default waypoint_hop (0.05 s) is under the convolution's 1024-sample minimum: the transform
    raises the hop to 1024 samples.  At speed 0 the result is the static transform's."""
    t = _room_tfm(source_speed=("const", 0.0))
    assert t.waypoint_hop == 0.05 and round(0.05 * sr) < 1024
    y, p = _run(t, x, sr, [1, 2])
    y0, _ = _run(_room_tfm(), x, sr, [1, 2])
    assert (y - y0).abs().max() <= 1e-5 * y0.abs().max()
    seen = []
    from audiotools_b200.engine import get_engine

    eng = get_engine()
    real = eng.circular_convolve_moving
    eng.circular_convolve_moving = lambda *a, **kw: seen.append(a[2]) or real(*a, **kw)
    try:
        _run(_room_tfm(source_speed=("uniform", 0.5, 2.0)), x, sr, [3, 4])
    finally:
        del eng.circular_convolve_moving
    assert seen == [1024]


def check_bad_speed_and_hop(x, sr):
    with pytest.raises(ValueError, match="speeds must be"):
        _run(_room_tfm(source_speed=("const", -1.0)), x, sr, [1])
    for hop in (0.0, -0.05, float("nan")):
        with pytest.raises(ValueError, match="waypoint_hop"):
            _room_tfm(source_speed=("const", 1.0), waypoint_hop=hop)


def check_shared_tail_seed(x, sr, monkeypatch):
    from audiotools_b200.core import room

    seeds = []
    real = room.image_source_ir

    def spy(*a, **kw):
        seeds.append(np.asarray(kw["seed"]))
        return real(*a, **kw)

    monkeypatch.setattr(room, "image_source_ir", spy)
    t = _room_tfm(diffuse_after=0.02, source_speed=("const", 3.0), waypoint_hop=0.07)
    _, p = _run(t, x, sr, [7, 8])
    K = (x.shape[-1] - 1) // round(0.07 * sr) + 1
    assert np.array_equal(np.concatenate(seeds), np.repeat(p["seed"].cpu().numpy(), K))


def check_bands_chunked(x, sr, monkeypatch, max_rows=None):
    """Bands make items x microphones x bands exceed MAX_ROWS over the B K waypoint items: image_source_ir is called in
    chunks, each within MAX_ROWS (it raises otherwise), and the result is the items' one at a time."""
    from audiotools_b200.core import room

    if max_rows is not None:
        monkeypatch.setattr(room, "MAX_ROWS", max_rows)
    calls = []
    real = room.image_source_ir

    def spy(room_, *a, **kw):
        calls.append(len(room_))
        return real(room_, *a, **kw)

    monkeypatch.setattr(room, "image_source_ir", spy)
    B, C = x.shape[:2]
    K = (x.shape[-1] - 1) // round(0.07 * sr) + 1
    t = _room_tfm(bands=8, source_speed=("uniform", 1.0, 5.0), waypoint_hop=0.07)
    y, _ = _run(t, x, sr, list(range(B)))
    assert B * K * C * 8 > room.MAX_ROWS and len(calls) > 1 and sum(calls) == B * K
    assert max(calls) * C * 8 <= room.MAX_ROWS
    from audiotools_b200 import AudioSignal

    for b in range(B):
        sig = AudioSignal(x[b:b + 1].clone(), sr)
        assert torch.equal(t(sig, **t.instantiate(b, sig)).audio_data[0], y[b]), b


def _speech(B, C, T, seed=0):
    return (0.1 * torch.randn(B, C, T, generator=torch.Generator().manual_seed(seed))).to(DEV)


def test_transform_static_unchanged():
    check_static_unchanged(_speech(3, 2, 16000), 16000)


def test_transform_paths():
    check_paths(_speech(6, 2, 24000), 16000)


@pytest.mark.parametrize("kw", [{}, {"diffuse_after": 0.02}, {"bands": 3}])
def test_transform_batch_equals_instantiate(kw):
    check_batch_equals_instantiate(_speech(3, 2, 16000), 16000, **kw)


def test_transform_default_hop_at_16k():
    check_default_hop_low_rate(_speech(2, 2, 16000), 16000)


def test_transform_bad_speed_and_hop():
    check_bad_speed_and_hop(_speech(1, 2, 16000), 16000)


def test_transform_shared_tail_seed(monkeypatch):
    check_shared_tail_seed(_speech(2, 2, 16000), 16000, monkeypatch)


def test_transform_bands_chunked(monkeypatch):
    # 150 s at 16 kHz, a waypoint every 1120 samples: 2 items x 2143 waypoints x 2 microphones x 8 bands = 68 576 rows
    check_bands_chunked(_speech(2, 2, 2_400_000), 16000, monkeypatch)
