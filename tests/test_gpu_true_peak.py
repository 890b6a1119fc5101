"""``Engine.true_peak`` / ``AudioSignal.true_peak`` and ``normalize(true_peak_limit=...)`` on the H100 (``-m gpu``):
the true-peak level of csrc/truepeak.cu against the float64 restatement of tests/truepeak64.py.

* row peaks within 2e-6 max |x_row| and dBTP within 1e-4 of the oracle run with the library's float taps: 16 k to
  192 kHz, 1, 2 and 5 channels, T = 1, 2, 11, 12, 13 and the kernel's chunk length +- 1, noise, chirps, clipped sines,
  silence; a row with a NaN or inf reads NaN or +inf;
* exactness: row peak >= row_absmax bit for bit (equal at 192 kHz), bit-identical reruns, row b of a batch equal to a
  single-item call;
* scale: 70 000 rows, and a [4, 2, 300 000 000] batch with a clipped burst past flat index 2^31;
* the API: ``loudness_stats(true_peak=True)``, ``normalize(-14, true_peak_limit=-1)`` (cap, untouched items, bypass,
  gradient), ``VolumeNorm(true_peak_limit=...)`` with a partial mask, no host sync, launch counts against the profiler.
tests/test_sim_true_peak.py runs the same checks at smaller sizes on the CPU simulator."""
import numpy as np
import pytest
import torch

from tests import truepeak64 as tp

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CHUNK = 4096  # samples of a row per CTA work item in csrc/truepeak.cu
LENGTHS = (1, 2, 11, 12, 13, CHUNK - 1, CHUNK, CHUNK + 1)
GF = float(np.float32(np.log(10) / 20))


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


def _np(t):
    return t.detach().cpu().double().numpy()


def make_batch(sr: float, C: int, T: int, seed: int = 0) -> np.ndarray:
    """[5, C, T] float32: noise, a chirp over 0.01 .. 0.49 fs, a 1.5-amplitude sine clipped at +-1, silence, and noise
    with a clipped sine on alternate channels; channels differ in level and seed."""
    rng = np.random.default_rng(seed)
    n = np.arange(T)
    items = []
    for kind in ("noise", "chirp", "clipped", "silent", "mixed"):
        rows = []
        for c in range(C):
            s = 1.0 - 0.15 * c
            if kind == "noise":
                r = 0.3 * s * rng.standard_normal(T)
            elif kind == "chirp":
                f = 0.01 + 0.48 * n / max(T, 1)
                r = 0.8 * s * np.sin(2 * np.pi * np.cumsum(f) + rng.uniform(0, 6.3))
            elif kind == "clipped":
                r = np.clip(1.5 * s * np.sin(2 * np.pi * (0.21 + 0.01 * c) * n + rng.uniform(0, 6.3)), -1, 1)
            elif kind == "silent":
                r = np.zeros(T)
            else:
                r = 0.2 * rng.standard_normal(T) if c % 2 == 0 else np.clip(1.3 * np.sin(2 * np.pi * 0.3 * n), -1, 1)
            rows.append(r)
        items.append(np.stack(rows))
    return np.stack(items).astype(np.float32)


def check_against_oracle(eng, sr, C, T, seed=0):
    x = make_batch(sr, C, T, seed)
    out = eng.true_peak(torch.from_numpy(x).to(DEV), sr)
    taps = eng.true_peak_taps(sr)
    assert taps.shape == (tp.factor(sr) - 1, 12)
    ref = tp.row_peaks(x, taps)
    rows = _np(out["rows"])
    assert out["rows"].shape == (x.shape[0], C) and out["db"].shape == (x.shape[0],)
    assert out["rows"].dtype == torch.float32 and out["db"].dtype == torch.float32
    amax = np.abs(x.astype(np.float64)).max(axis=-1)
    err = np.abs(rows - ref)
    assert (err <= 2e-6 * amax).all(), (sr, C, T, float((err / np.maximum(amax, 1e-30)).max()))
    db, db_ref = _np(out["db"]), tp.item_db(ref)
    silent = np.isneginf(db_ref)
    assert (np.isneginf(db) == silent).all() and silent[3]
    assert np.abs(db[~silent] - db_ref[~silent]).max() <= 1e-4, (sr, C, T)
    assert (rows[3] == 0).all()


def check_nonfinite(eng, sr):
    x = make_batch(sr, 2, 300, seed=3)
    x[0, 1, 100] = np.nan
    x[1, 0, 0] = np.inf
    x[2, 1, 299] = -np.inf
    x[4, 0, 150:152] = [np.inf, -np.inf]
    out = eng.true_peak(torch.from_numpy(x).to(DEV), sr)
    rows, db = _np(out["rows"]), _np(out["db"])
    bad = np.zeros(rows.shape, bool)
    bad[0, 1] = bad[1, 0] = bad[2, 1] = bad[4, 0] = True
    assert (np.isnan(rows[bad]) | np.isposinf(rows[bad])).all()
    assert np.isnan(rows[0, 1])
    assert (np.isnan(db[[0, 1, 2, 4]]) | np.isposinf(db[[0, 1, 2, 4]])).all()
    ref = tp.row_peaks(x, eng.true_peak_taps(sr))
    good = ~bad & np.isfinite(ref)
    assert (np.abs(rows[good] - ref[good]) <= 2e-6 * np.abs(x).max(axis=-1)[good]).all()


def check_exact(eng, sr, T=CHUNK + 700):
    x = torch.from_numpy(make_batch(sr, 2, T, seed=5)).to(DEV)
    a, b = eng.true_peak(x, sr), eng.true_peak(x, sr)
    assert torch.equal(a["rows"], b["rows"]) and torch.equal(a["db"], b["db"])
    absmax = eng.row_absmax(x).squeeze(-1)
    assert bool((a["rows"] >= absmax).all())
    if tp.factor(sr) == 1:
        assert torch.equal(a["rows"], absmax)
    for i in range(x.shape[0]):
        one = eng.true_peak(x[i:i + 1].clone(), sr)
        assert torch.equal(one["rows"][0], a["rows"][i]) and torch.equal(one["db"][0], a["db"][i])


def check_launches(eng):
    x = torch.zeros(2, 2, 100, device=DEV)
    n0 = eng.launches
    eng.true_peak(x, 48000)
    assert eng.launches - n0 == 2
    lib = eng.lib
    k0 = lib.kernel_launches.value
    p = x.data_ptr()
    assert lib.b2a_true_peak_f32(p, 2, 2, 100, 3, p, p, None) == -1 and b"factor must be 1, 2 or 4" in lib.b2a_last_error()
    assert lib.b2a_true_peak_f32(p, 0, 2, 100, 4, p, p, None) == -1 and b"bad shape" in lib.b2a_last_error()
    assert lib.b2a_true_peak_f32(None, 2, 2, 100, 4, p, p, None) == -1 and b"null pointer" in lib.b2a_last_error()
    assert lib.b2a_true_peak_f32(p, 2, 2, 1 << 62, 4, p, p, None) == -1 and b"overflows" in lib.b2a_last_error()
    assert lib.kernel_launches.value == k0


def check_api(eng, sr=48000):
    """loudness_stats(true_peak=True), true_peak(), normalize(-14, true_peak_limit=-1) with and without a bypass."""
    from audiotools_b200 import AudioSignal

    g = torch.Generator().manual_seed(0)
    T = sr
    n = torch.arange(T)
    x = torch.zeros(5, 2, T)
    x[0] = 0.05 * torch.sin(2 * np.pi * 1000 / sr * n)                      # crest 3 dB: cap not binding
    x[1] = 0.01 * torch.randn(2, T, generator=g)
    x[1, :, :: sr // 4] = 0.9                                                # clicks: the cap binds
    x[2] = torch.clamp(1.5 * torch.sin(2 * np.pi * 0.21 * n), -1, 1)
    x[3] = 0.2 * torch.randn(2, T, generator=g)
    x[3, 1, 1000:1010] = 0.95                                                # a burst on one channel
    # x[4] silent
    x = x.to(DEV)
    sig = AudioSignal(x.clone(), sr)
    base = sig.loudness_stats()
    with_tp = sig.loudness_stats(true_peak=True)
    peak = sig.true_peak()
    assert list(with_tp) == list(base) + ["True Peak"]
    for k in base:
        assert torch.equal(with_tp[k], base[k]), k
    assert torch.equal(with_tp["True Peak"], peak)
    assert torch.equal(peak, eng.true_peak(x, sr)["db"]) and bool(torch.isneginf(peak[4]))
    series = sig.loudness_stats(series=True, true_peak=True)
    assert list(series) == list(base) + ["True Peak", "momentary", "short_term"]

    plain = AudioSignal(x.clone(), sr).normalize(-14.0)
    capped = AudioSignal(x.clone(), sr).normalize(-14.0, true_peak_limit=-1.0)
    p_plain, p_capped = plain.true_peak(), capped.true_peak()
    finite = torch.isfinite(p_capped)
    assert bool((p_capped[finite] <= -1 + 1e-4).all()), p_capped
    binding = p_plain > -1.0
    assert bool(binding[1]) and not bool(binding[0]) and not bool(binding[4])
    assert bool(((p_capped[binding] - (-1.0)).abs() <= 1e-3).all())
    for i in range(5):
        if not bool(binding[i]):
            assert torch.equal(capped.audio_data[i], plain.audio_data[i]), i
    per_item = AudioSignal(x.clone(), sr).normalize(-14.0, true_peak_limit=torch.full((5,), -1.0))
    assert torch.equal(per_item.audio_data, capped.audio_data)
    bypass = torch.tensor([False, True, False, True, False], device=DEV)
    byp = AudioSignal(x.clone(), sr).normalize(-14.0, _bypass=bypass, true_peak_limit=-1.0)
    assert torch.equal(byp.audio_data[bypass], x[bypass])
    assert torch.equal(byp.audio_data[~bypass], capped.audio_data[~bypass])

    # gradient: the gain is a constant
    leaf = x.clone().requires_grad_(True)
    y = AudioSignal(leaf, sr).normalize(-14.0, true_peak_limit=-1.0).audio_data
    cot = torch.randn(x.shape, generator=g).to(DEV)
    (y * cot).sum().backward()
    gain = torch.minimum(eng.lufs(x, sr, target_db=torch.tensor([-14.0], device=DEV))["gain"],
                         torch.exp((-1.0 - eng.true_peak(x, sr)["db"]) * GF))
    assert torch.equal(leaf.grad, cot * gain[:, None, None])
    assert torch.equal(y.detach(), capped.audio_data)


def check_volume_norm_mask(sr=16000):
    """VolumeNorm(true_peak_limit=-1) in a Compose with prob < 1: the bypass-flag path equals the reference's gather /
    scatter path bit for bit, and leaves the unselected items untouched."""
    from audiotools_b200 import AudioSignal
    from audiotools_b200.data import transforms as tfm

    g = torch.Generator().manual_seed(1)
    B, T = 6, sr
    x = 0.02 * torch.randn(B, 2, T, generator=g)
    x[:, :, :: sr // 8] = 0.8  # high crest: the cap binds at -10 LUFS
    x = x.to(DEV)
    t = tfm.VolumeNorm(db=("uniform", -20, -10), prob=0.5, true_peak_limit=-1.0)
    comp = tfm.Compose([t, tfm.VolumeChange(db=("const", 0.0))])
    sig = AudioSignal(x.clone(), sr)
    kw = comp.batch_instantiate(list(range(B)), sig)
    mask = kw[comp.name][t.name]["mask"]
    assert 0 < int(mask.sum()) < B
    assert t._mask_aware
    a = comp(sig.clone(), **kw).audio_data
    t._mask_aware = False  # the reference's gather -> transform -> scatter
    b = comp(sig.clone(), **kw).audio_data
    t._mask_aware = True
    assert torch.equal(a, b)
    m = mask.to(a.device)
    assert torch.equal(a[~m], x[~m])
    assert bool((AudioSignal(a[m].clone(), sr).true_peak() <= -1 + 1e-4).all())
    # parameter draws unchanged by the limit
    kw0 = tfm.Compose([tfm.VolumeNorm(db=("uniform", -20, -10), prob=0.5), tfm.VolumeChange(db=("const", 0.0))]) \
        .batch_instantiate(list(range(B)), sig)
    assert torch.equal(kw0["Compose"]["0.VolumeNorm"]["db"], kw[comp.name][t.name]["db"])
    assert torch.equal(kw0["Compose"]["0.VolumeNorm"]["mask"], mask)


# --------------------------------------------------------------------------- tests
@pytest.mark.parametrize("sr", [16000, 22050, 44100, 48000, 96000, 192000])
@pytest.mark.parametrize("C", [1, 2, 5])
def test_against_float64(eng, sr, C):
    for T in LENGTHS:
        check_against_oracle(eng, sr, C, T, seed=T)


def test_long_rows_against_float64(eng):
    check_against_oracle(eng, 44100, 2, 10 * CHUNK + 123)


@pytest.mark.parametrize("sr", [16000, 44100, 96000, 192000])
def test_nonfinite_rows(eng, sr):
    check_nonfinite(eng, sr)


@pytest.mark.parametrize("sr", [44100, 96000, 192000])
def test_exactness(eng, sr):
    check_exact(eng, sr)


def test_launches_and_rejected_calls(eng):
    check_launches(eng)


def test_api(eng):
    check_api(eng)


def test_volume_norm_partial_mask(eng):
    check_volume_norm_mask()


def test_many_short_rows(eng):
    """70 000 rows: more than the 65535 rows of row_absmax's grid."""
    g = torch.Generator(device=DEV).manual_seed(0)
    x = torch.randn(35000, 2, 37, device=DEV, generator=g)
    out = eng.true_peak(x, 44100)
    ref = tp.row_peaks(_np(x), eng.true_peak_taps(44100))
    assert np.abs(_np(out["rows"]) - ref).max() <= 2e-6 * float(x.abs().max())
    assert np.abs(_np(out["db"]) - tp.item_db(ref)).max() <= 1e-4


def test_more_than_2_31_elements(eng):
    """[4, 2, 300e6] zeros with a clipped burst past flat index 2^31: only the burst's row is non-zero, and it matches
    the oracle on the burst."""
    B, C, T = 4, 2, 300_000_000
    x = torch.zeros(B, C, T, device=DEV)
    start = (1 << 31) + 12345
    row, off = divmod(start, T)
    n = torch.arange(3000, device=DEV, dtype=torch.float64)
    burst = torch.clamp(1.4 * torch.sin(2 * np.pi * 0.23 * n + 0.4), -1, 1).float()
    x.view(-1)[start:start + 3000] = burst
    out = eng.true_peak(x, 48000)
    rows = _np(out["rows"]).reshape(-1)
    ref = tp.row_peaks(np.pad(_np(burst), 6)[None], eng.true_peak_taps(48000))[0]  # zeros around, as in the row
    assert row == 7 and off + 3000 < T
    assert (rows[:row] == 0).all() and abs(rows[row] - ref) <= 2e-6
    assert rows[row] > 1.0
    db = _np(out["db"])
    assert np.isneginf(db[:3]).all() and abs(db[3] - 20 * np.log10(ref)) <= 1e-4
    del x
    torch.cuda.empty_cache()


def test_no_host_sync(eng):
    from audiotools_b200 import AudioSignal

    x = 0.1 * torch.randn(4, 2, 48000, device=DEV)
    sig = AudioSignal(x.clone(), 48000)
    db = torch.tensor(-14.0, device=DEV)  # a host number would be copied to the device (a sync) by normalize itself
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        sig.true_peak()
        sig.normalize(db, true_peak_limit=-1.0)
        sig.normalize(db, true_peak_limit=torch.full((4,), -1.0, device=DEV))
        eng.true_peak(x, 48000)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_launches_match_the_profiler(eng):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    x = 0.1 * torch.randn(64, 2, 441000, device=DEV)
    eng.true_peak(x, 44100)
    torch.cuda.synchronize()
    n0 = eng.launches
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        eng.true_peak(x, 44100)
        torch.cuda.synchronize()
    added = eng.launches - n0
    gpu = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    if not gpu:
        pytest.skip("the profiler recorded no GPU activity")
    names = [e.name for e in gpu]
    assert (sum("b2a::" in n for n in names), added) == (2, 2), names
