"""``Engine.limit`` / ``AudioSignal.limit`` / ``transforms.Limiter`` on the H100 (``-m gpu``): the look-ahead true-peak
limiter of csrc/limiter.cu against the float64 restatement of tests/limiter64.py.

* per sample: the reduction within 2e-6 and the output within 2e-6 max |x| of the oracle: 16 k to 192 kHz (factors 4, 2,
  1), 1, 2 and 5 channels, T = 1, A, 2 A + 1, the chunk length +- 1, several chunks and one row of 330 chunks at a 2 s
  release, A = 0, 1, the default and 1024, releases of 1 ms, 50 ms and 2 s, scalar and per-item ceilings, with and
  without a gain, in place and out of place; overs in the first and last sample of a row and on both sides of a chunk
  boundary; a NaN or inf sample;
* properties: no sample passes the ceiling, ``true_peak()`` of the output stays within TP_TOL of it, items under the
  ceiling and samples away from every over come back bit for bit, batch == single items, reruns identical;
* the point: ``normalize(-16).limit(-1)`` ends at least 6 LU nearer to -16 LUFS than ``normalize(-16,
  true_peak_limit=-1)`` on clicks over quiet noise;
* the API: the pending gain is consumed, launch counts, refused arguments, ``Limiter`` under a partial mask, no host
  sync, the profiler's launch count.
tests/test_sim_limiter.py runs the same checks at smaller sizes on the CPU simulator."""
import numpy as np
import pytest
import torch

from tests import limiter64 as lim
from tests import truepeak64 as tp

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CHUNK = lim.CHUNK
LAUNCHES = 3   # b2a_limiter_f32 (DESIGN.md K18)
TP_TOL = 0.02  # dB: true peak of the output over the ceiling (the oracle study in DESIGN.md K18 found < 0.004)


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


def _np(t):
    return t.detach().cpu().double().numpy()


def make_batch(sr: float, C: int, T: int, seed: int = 0) -> np.ndarray:
    """[7, C, T] float32: quiet noise (never over -1 dBTP), a faded 1.6-amplitude sine at 0.01 .. 0.45 fs, an unfaded
    fs/4 sine at 45 degrees (full level at both ends), a 1.5-amplitude sine clipped at +-1, clicks on quiet noise (in
    the first and the last sample and on both sides of every chunk boundary), amplitude-modulated noise, silence."""
    rng = np.random.default_rng(seed)
    n = np.arange(T)
    items = []
    for kind in ("quiet", "sine", "quarter", "clipped", "clicks", "am", "silent"):
        rows = []
        for c in range(C):
            s = 1.0 - 0.12 * c
            if kind == "quiet":
                r = 0.02 * s * rng.standard_normal(T)
            elif kind == "sine":
                r = 1.6 * s * np.sin(2 * np.pi * rng.uniform(0.01, 0.45) * n + rng.uniform(0, 6.3))
                nf = T // 8
                if nf:
                    ramp = 0.5 * (1 - np.cos(np.pi * np.arange(nf) / nf))
                    r[:nf] *= ramp
                    r[T - nf:] *= ramp[::-1]
            elif kind == "quarter":
                r = lim.quarter_rate_sine(T, 1.3 * s)
            elif kind == "clipped":
                r = lim.clipped_sine(T, 0.21 + 0.01 * c, rng.uniform(0, 6.3), 1.5) * s
            elif kind == "clicks":
                r = 0.03 * rng.standard_normal(T)
                if c == 0:
                    pos = [0, T - 1] + [k * CHUNK + o for k in range(1, T // CHUNK + 1) for o in (-3, 2)]
                    pos = [p for p in pos if 0 <= p < T]
                    r[pos] = 1.2 * np.where(np.arange(len(pos)) % 2 == 0, 1.0, -1.0)
            elif kind == "am":
                r = s * rng.standard_normal(T) * (1 + 0.8 * np.sin(2 * np.pi * 40.0 * n / sr + c)) / 2.5
            else:
                r = np.zeros(T)
            rows.append(r)
        items.append(np.stack(rows))
    return np.stack(items).astype(np.float32)


def check_against_oracle(eng, sr, C, T, A=None, release=0.05, per_item=False, gain=False, inplace=False, seed=0,
                         x=None):
    lookahead = 0.0015 if A is None else A / sr
    x = make_batch(sr, C, T, seed) if x is None else x
    B = x.shape[0]
    rng = np.random.default_rng(seed + 1)
    cdb = torch.tensor(rng.uniform(-9, -0.5, B), dtype=torch.float32, device=DEV) if per_item else -1.0
    g = rng.uniform(0.5, 1.8, B).astype(np.float32) if gain else None
    xt = torch.from_numpy(x.copy()).to(DEV)
    out, red = eng.limit(xt, sr, cdb, lookahead, release, gain=None if g is None else torch.from_numpy(g).to(DEV),
                         want_reduction=True, out=xt if inplace else None)
    assert (out.data_ptr() == xt.data_ptr()) == inplace
    assert out.shape == x.shape and red.shape == (B, T) and red.dtype == torch.float32
    L, c, A_used, a = eng.limiter_params(sr, cdb, lookahead, release, B, DEV)
    assert L == tp.factor(sr) and (A is None or A_used == A)
    want, r = lim.limit(x, eng.true_peak_taps(sr), _np(c), A_used, a, g)
    where = (sr, C, T, A_used, release, per_item, gain, inplace)
    err_r = np.abs(_np(red) - r).max()
    assert err_r <= 2e-6, (where, err_r)
    scale = float(np.abs(x if g is None else x * g[:, None, None]).max())
    err_o = np.abs(_np(out) - want).max()
    assert err_o <= 2e-6 * max(scale, 1e-30), (where, err_o / max(scale, 1e-30))
    if B == 7 and not gain and not per_item:
        assert (r[0] == 0).all() and (r[6] == 0).all() and (T < CHUNK - 1 or r[1:6].max(axis=1).min() > 0.01)
    return _np(red), r


def check_nonfinite(eng, sr, A=20):
    """The oracle's rule: r is NaN from the first non-finite value of e less 2 A to the end of the row, the whole item
    with it; other items as without the bad sample."""
    T = CHUNK + 900
    x = make_batch(sr, 2, T, seed=3)
    clean = x.copy()
    x[1, 1, 2000] = np.nan
    x[3, 0, 3000] = np.inf
    x[5, 1, CHUNK + 100] = -np.inf
    out, red = eng.limit(torch.from_numpy(x).to(DEV), sr, -1.0, A / sr, 0.001, want_reduction=True)
    out0, red0 = eng.limit(torch.from_numpy(clean).to(DEV), sr, -1.0, A / sr, 0.001, want_reduction=True)
    L, c, _, a = eng.limiter_params(sr, -1.0, A / sr, 0.001, 7, DEV)
    _, r = lim.limit(x, eng.true_peak_taps(sr), _np(c), A, a)
    red, out = _np(red), _np(out)
    assert (np.isnan(red) == np.isnan(r)).all()
    reach = 6 if L > 1 else 0
    for b, p in ((1, 2000), (3, 3000), (5, CHUNK + 100)):
        first = int(np.argmax(np.isnan(red[b])))
        assert p - reach - 2 * A - 1 <= first <= p - 2 * A and np.isnan(red[b, first:]).all()
        assert np.isnan(out[b, :, first:]).all() and not np.isnan(out[b, :, :first]).any()
    ok = ~np.isnan(r)
    assert np.abs(red[ok] - r[ok]).max() <= 2e-6
    for b in (0, 2, 4, 6):
        assert torch.equal(torch.from_numpy(out[b]), out0[b].cpu().double()) and (red[b] == _np(red0[b])).all()


def check_properties(eng, sr=44100, T=2 * CHUNK + 1500, release=0.001):
    from audiotools_b200 import AudioSignal

    A = int(round(0.0015 * sr))
    x = make_batch(sr, 2, T, seed=7)
    rng = np.random.default_rng(8)
    x[4] = (0.01 * rng.standard_normal((2, T))).astype(np.float32)  # one click only, on channel 1
    p = CHUNK + 40
    x[4, 1, p] = 1.4
    g = np.array([1.0, 0.8, 1.0, 1.1, 1.0, 0.9, 1.0], np.float32)
    xt, gt = torch.from_numpy(x).to(DEV), torch.from_numpy(g).to(DEV)
    out, red = eng.limit(xt, sr, -1.0, 0.0015, release, gain=gt, want_reduction=True)
    c = np.float32(10 ** (-1 / 20))
    assert float(out.abs().max()) <= float(c) * (1 + 2.0 ** -21)  # a few float32 roundings
    peak = AudioSignal(out.clone(), sr).true_peak()
    assert bool((peak[:6] <= -1 + TP_TOL).all()) and bool(torch.isneginf(peak[6])), peak
    assert float(peak[:6].max()) > -1.2  # and the limiter did not simply turn everything down
    xg = eng.gain(xt, gt)
    for b in (0, 6):  # never over the ceiling
        assert torch.equal(out[b], xg[b]) and not bool(red[b].any())
    far = np.ones(T, bool)
    far[p - 7 - 2 * A:p + 7 + 2 * A + int(19 * release * sr) + 1] = False
    far_t = torch.from_numpy(far).to(DEV)
    assert torch.equal(out[4][:, far_t], xg[4][:, far_t]) and not bool(red[4][far_t].any())
    assert float(red[4].max()) > 0.3 and not torch.equal(out[4, 0], xg[4, 0])  # channel 0 follows channel 1's click
    out2, red2 = eng.limit(xt, sr, -1.0, 0.0015, release, gain=gt, want_reduction=True)
    assert torch.equal(out, out2) and torch.equal(red, red2)
    for b in range(x.shape[0]):
        o1, r1 = eng.limit(xt[b:b + 1].clone(), sr, -1.0, 0.0015, release, gain=gt[b:b + 1], want_reduction=True)
        assert torch.equal(o1[0], out[b]) and torch.equal(r1[0], red[b]), b
    assert torch.equal(eng.limit(xt, sr, -1.0, 0.0015, release, gain=gt), out)  # without the reduction output


def check_full_level_start(eng, sr=44100):
    """A signal that starts and ends at full level: a mean over 2 A + 1 at the row ends (instead of over the samples
    inside the row) overshot by 1.8 dB here."""
    from audiotools_b200 import AudioSignal

    x = np.stack([lim.quarter_rate_sine(6000, 1.3), lim.clipped_sine(6000)])[:, None].astype(np.float32)
    sig = AudioSignal(torch.from_numpy(x).to(DEV), sr).limit(-1.0)
    assert bool((sig.true_peak() <= -1 + TP_TOL).all()), sig.true_peak()
    assert float(sig.audio_data[:, :, :100].abs().max()) <= 10 ** (-1 / 20) * (1 + 2.0 ** -21)


def point_batch(sr, seconds, B=3):
    x = np.stack([lim.clicks_on_noise(sr, seconds, int(3 * seconds), seed=b, noise_db=-34.0) for b in range(B)])
    return np.stack([x, x[:, ::-1]], axis=1).astype(np.float32)


def check_point_of_the_feature(eng, sr=44100, seconds=3.0):
    from audiotools_b200 import AudioSignal

    x = torch.from_numpy(point_batch(sr, seconds)).to(DEV)
    limited = AudioSignal(x.clone(), sr).normalize(-16.0).limit(-1.0)
    capped = AudioSignal(x.clone(), sr).normalize(-16.0, true_peak_limit=-1.0)
    assert bool((limited.true_peak() <= -1 + TP_TOL).all()) and bool((capped.true_peak() <= -1 + 1e-3).all())
    l_lim, l_cap = limited.loudness(), capped.loudness()
    assert bool(((l_lim + 16).abs() + 6 <= (l_cap + 16).abs()).all()), (l_lim, l_cap)
    # amplitude-modulated noise whose true peak is 2.2 dB over the ceiling at the target loudness (the limiter costs
    # 0.32 .. 0.41 LU there, 0.43 .. 0.50 at 2.5 dB over and 0.63 .. 0.68 at 3 dB over: DESIGN.md K18)
    am = np.stack([lim.am_noise(sr, seconds, seed=10 + b) for b in range(2)])[:, None].astype(np.float32)
    sig = AudioSignal(torch.from_numpy(am).to(DEV), sr)
    target = sig.loudness() + (-1.0 + 2.2 - sig.true_peak())
    sig = sig.normalize(target)
    over = sig.true_peak() + 1.0
    assert bool(((over > 2) & (over < 3)).all()), over
    sig.limit(-1.0)
    assert bool((sig.true_peak() <= -1 + TP_TOL).all())
    assert bool(((sig.loudness() - target).abs() <= 0.5).all()), (sig.loudness(), target)


def check_api(eng, sr=44100):
    from audiotools_b200 import AudioSignal
    from audiotools_b200.data import transforms as tfm

    x = torch.from_numpy(make_batch(sr, 2, sr // 2, seed=11)[:6]).to(DEV)
    lib = eng.lib
    # launches: limit() costs its own three; after normalize() the gain rides along
    n0, k0 = eng.launches, lib.kernel_launches.value
    eng.lufs(x, sr, target_db=torch.tensor([-16.0], device=DEV))
    n_lufs = eng.launches - n0
    n0 = eng.launches
    out = eng.limit(x, sr, -1.0)
    assert eng.launches - n0 == LAUNCHES
    n0 = eng.launches
    sig = AudioSignal(x.clone(), sr).normalize(-16.0)
    sig._stft_data = torch.zeros(1)
    sig.limit(-1.0)
    assert eng.launches - n0 == n_lufs + LAUNCHES
    assert lib.kernel_launches.value - k0 == 2 * (n_lufs + LAUNCHES)
    assert sig._pending_gain is None and sig._loudness is None and sig.stft_data is None
    ref = AudioSignal(x.clone(), sr).normalize(-16.0)
    assert torch.equal(sig.audio_data, eng.limit(ref.audio_data, sr, -1.0))  # == materialise, then limit
    assert AudioSignal(x.clone(), sr).limit(-1.0) is not None
    assert torch.equal(AudioSignal(x.clone(), sr).limit().audio_data, out)
    per_item = torch.tensor([-1.0, -2.0, -3.0, -4.0, -5.0, -6.0])
    a = AudioSignal(x.clone(), sr).limit(per_item, lookahead=0.001, release=0.02).audio_data
    for b in range(6):
        one = AudioSignal(x[b:b + 1].clone(), sr).limit(per_item[b:b + 1], lookahead=0.001, release=0.02).audio_data
        assert torch.equal(one[0], a[b])
    # no backward
    with pytest.raises(NotImplementedError, match="limit"):
        AudioSignal(x.clone().requires_grad_(True), sr).limit(-1.0)
    with pytest.raises(NotImplementedError, match="limit"):
        eng.limit(x.clone().requires_grad_(True), sr, -1.0)
    # refused arguments launch nothing
    k0 = lib.kernel_launches.value
    with pytest.raises(ValueError, match="lookahead"):
        eng.limit(x, sr, -1.0, lookahead=1025 / sr)
    with pytest.raises(ValueError, match="release"):
        eng.limit(x, sr, -1.0, release=0.0)
    p, (B, C, T) = x.data_ptr(), x.shape
    bad = [((p, None, B, C, T, 4, p, 1025, 0.5, p, None, p, None), b"lookahead"),
           ((p, None, B, C, T, 4, p, -1, 0.5, p, None, p, None), b"lookahead"),
           ((p, None, B, C, T, 4, p, 66, 1.0, p, None, p, None), b"release"),
           ((p, None, B, C, T, 4, p, 66, -0.1, p, None, p, None), b"release"),
           ((p, None, B, C, T, 3, p, 66, 0.5, p, None, p, None), b"factor must be 1, 2 or 4"),
           ((None, None, B, C, T, 4, p, 66, 0.5, p, None, p, None), b"null pointer"),
           ((p, None, B, C, T, 4, None, 66, 0.5, p, None, p, None), b"null pointer"),
           ((p, None, B, C, T, 4, p, 66, 0.5, None, None, p, None), b"null pointer"),
           ((p, None, B, C, T, 4, p, 66, 0.5, p, None, None, None), b"null pointer"),
           ((p, None, B, 0, T, 4, p, 66, 0.5, p, None, p, None), b"bad shape"),
           ((p, None, B, C, 1 << 62, 4, p, 66, 0.5, p, None, p, None), b"overflows")]
    for args, msg in bad:
        assert lib.b2a_limiter_f32(*args) == -1 and msg in lib.b2a_last_error(), msg
    assert lib.b2a_limiter_workspace_bytes(B, C, 1 << 62) == 0 and lib.b2a_limiter_workspace_bytes(0, C, T) == 0
    assert lib.b2a_limiter_workspace_bytes(2, 2, CHUNK + 1) == 4 * (2 * (CHUNK + 1) + 3 * 2 * 2)
    assert lib.kernel_launches.value == k0
    # the transform, under a partial mask: the selected items are limited, the others untouched
    t = tfm.Limiter(ceiling=("uniform", -6.0, -1.0), lookahead=0.001, release=0.02, prob=0.5)
    comp = tfm.Compose([t])
    sig = AudioSignal(x.clone(), sr)
    kw = comp.batch_instantiate(list(range(6)), sig)
    mask = kw[comp.name][t.name]["mask"]
    assert 0 < int(mask.sum()) < 6
    y = comp(sig.clone(), **kw).audio_data
    m = mask.to(y.device)
    want = AudioSignal(x[m].clone(), sr).limit(kw[comp.name][t.name]["ceiling"][mask], lookahead=0.001,
                                                release=0.02).audio_data
    assert torch.equal(y[m], want) and torch.equal(y[~m], x[~m]) and not torch.equal(y[m], x[m])


# --------------------------------------------------------------------------- tests
LENGTHS = (1, 2, 66, 133, CHUNK - 1, CHUNK, CHUNK + 1, 3 * CHUNK + 17)


@pytest.mark.parametrize("C", [1, 2, 5])
@pytest.mark.parametrize("sr", [16000, 44100, 48000, 96000, 192000])
def test_against_float64(eng, sr, C):
    for T in LENGTHS:
        check_against_oracle(eng, sr, C, T, seed=T, inplace=T % 2 == 0)


@pytest.mark.parametrize("release", [0.001, 0.05, 2.0])
@pytest.mark.parametrize("A", [0, 1, 1024])
def test_lookaheads_and_releases(eng, A, release):
    for sr, C in ((44100, 2), (192000, 1)):
        for T in sorted({1, max(A, 1), 2 * A + 1, CHUNK - 1, CHUNK + 1, 3 * CHUNK + 17}):
            check_against_oracle(eng, sr, C, T, A=A, release=release, seed=T + A, per_item=T % 2 == 1, gain=T % 3 == 0,
                                 inplace=T % 4 == 1)


@pytest.mark.parametrize("gain,per_item,inplace", [(True, False, False), (False, True, True), (True, True, True)])
def test_gain_ceilings_and_in_place(eng, gain, per_item, inplace):
    for sr in (16000, 48000):
        check_against_oracle(eng, sr, 2, 2 * CHUNK + 123, release=0.02, gain=gain, per_item=per_item, inplace=inplace)


def test_a_row_of_330_chunks_at_a_2_s_release(eng):
    """a^4096 = 0.95: the carry of a burst is above 2^-26 for some 350 chunks, so a wrong or truncated carry shows."""
    sr, T = 44100, 330 * CHUNK + 77
    rng = np.random.default_rng(5)
    x = (0.02 * rng.standard_normal((2, 2, T))).astype(np.float32)
    x[0, 0, 5000:5040] = 1.5
    x[0, 1, 200 * CHUNK - 2] = -1.1
    x[1, :, 40 * CHUNK + 7:40 * CHUNK + 300] *= 60
    got, want = check_against_oracle(eng, sr, 2, T, release=2.0, x=x)
    assert want[0, 150 * CHUNK] > 1e-4 and want[0, -1] > 1e-4  # the release is still running 145 and 325 chunks on
    check_against_oracle(eng, sr, 2, T, A=1024, release=2.0, x=x, inplace=True)


@pytest.mark.parametrize("sr", [44100, 96000, 192000])
def test_nonfinite_samples(eng, sr):
    check_nonfinite(eng, sr)


def test_properties(eng):
    check_properties(eng)
    check_properties(eng, sr=96000, release=0.0005)


def test_signal_at_full_level_from_the_first_sample(eng):
    check_full_level_start(eng)


def test_the_point_of_the_feature(eng):
    check_point_of_the_feature(eng)


def test_api(eng):
    check_api(eng)


def test_more_than_2_31_elements(eng):
    """[3, 2, 400e6]: 2.4e9 samples, zeros with a burst past flat index 2^31; only the burst's item
    changes, in place."""
    B, C, T = 3, 2, 400_000_000
    x = torch.zeros(B, C, T, device=DEV)
    p = T - 15000
    n = torch.arange(3000, device=DEV, dtype=torch.float64)
    burst = (1.4 * torch.sin(2 * np.pi * 0.23 * n + 0.4)).float()
    x[2, 1, p:p + 3000] = burst
    x[1, 0, 123] = 0.5
    small = torch.zeros(1, C, 20000, device=DEV)
    small[0, 1, 10000:13000] = burst
    want = eng.limit(small, 48000, -1.0)
    out = eng.limit(x, 48000, -1.0, out=x)
    # the burst sits elsewhere in its chunk than in the small signal: the same values up to the scan's rounding
    assert float((out[2, :, p - 10000:p + 10000] - want[0]).abs().max()) <= 2e-6 and float(want[0].abs().max()) > 0.8
    assert float(out[2, :, :p - 10000].abs().max()) == 0 and float(out[0].abs().max()) == 0
    assert float(out[1].abs().sum()) == 0.5
    del x, out
    torch.cuda.empty_cache()


def test_no_host_sync(eng):
    from audiotools_b200 import AudioSignal

    x = 0.5 * torch.randn(4, 2, 48000, device=DEV)
    sig = AudioSignal(x.clone(), 48000)
    db = torch.tensor(-16.0, device=DEV)
    per_item = torch.full((4,), -2.0, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        sig.normalize(db).limit(-1.0)
        sig.limit(per_item, lookahead=0.003, release=0.2)
        eng.limit(x, 48000, -1.0, want_reduction=True)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_launches_match_the_profiler(eng):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    x = 0.5 * torch.randn(64, 2, 441000, device=DEV)
    eng.limit(x, 44100, -1.0)
    torch.cuda.synchronize()
    n0, k0 = eng.launches, eng.lib.kernel_launches.value
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        eng.limit(x, 44100, -1.0)
        torch.cuda.synchronize()
    added = eng.launches - n0
    assert eng.lib.kernel_launches.value - k0 == added
    gpu = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    if not gpu:
        pytest.skip("the profiler recorded no GPU activity")
    names = [e.name for e in gpu]
    assert (sum("b2a::limiter" in n for n in names), added) == (LAUNCHES, LAUNCHES), names
