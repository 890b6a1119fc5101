"""``Engine.sos_filter`` / ``AudioSignal.sos_filter`` / ``parametric_eq`` / ``transforms.ParametricEQ`` on the H100
(``-m gpu``): the biquad cascades of csrc/iir.cu against the float64 oracle of tests/iir64.py.

* per sample: the worst 1024-sample block of every row within RATIO times the sequential float32 cascade's worst block
  on the same input, or FLOOR_U u, whichever is larger: 16 k to 192 kHz, 1, 2 and 5 channels, S = 1 .. 8, shared and
  per-item sections, every cookbook kind with freq 10 Hz .. 0.45 sr, Q 0.1 .. 20 and gains of +-24 dB, T = 1, 2, the
  chunk length +- 1, several chunks and a long row; noise, DC steps, 20 .. 60 Hz tones, impulses, silence and a
  100 dB drop; forward and reverse, with and without a gain, in place and out of place;
* properties: identity sections, an unstable section, a NaN sample, batch == single items, reruns identical, the gain
  of a peak at its centre;
* the gradient against the float64 adjoint, the dot-product test, refused parameter gradients;
* the API: the pending gain is consumed, launch counts, refused arguments, ``ParametricEQ`` under a partial mask and
  inside ``Compose``, no host sync, the profiler's launch count, a batch past 2^31 elements.
tests/test_sim_iir.py runs the same checks at smaller sizes on the CPU simulator."""
import numpy as np
import pytest
import torch

from tests import iir64

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CHUNK = 1024     # csrc/iir.cu
LAUNCHES = 3     # b2a_sos_filter_f32 (DESIGN.md K19)
RATIO = 2.0      # worst block of the kernel / worst block of the sequential float32 cascade
FLOOR_U = 64.0   # u: the absolute floor for rows where the float32 cascade is nearly exact
KINDS = ("peaking", "low_shelf", "high_shelf", "low_pass", "high_pass", "band_pass", "notch", "all_pass")
SIGNALS = ("noise", "dc_steps", "low_tone", "impulses", "silence", "drop")


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


def _np(t):
    return t.detach().cpu().double().numpy()


def random_sos(rng, sr: float, S: int, items: int) -> np.ndarray:
    """[items, S, 6] float64 cookbook sections: every kind, freq log-uniform in 10 Hz .. 0.45 sr, Q log-uniform in
    0.1 .. 20, gains uniform in +-24 dB."""
    out = np.empty((items, S, 6))
    for i in range(items):
        for s in range(S):
            kind = KINDS[rng.integers(len(KINDS))]
            f = float(np.exp(rng.uniform(np.log(10.0), np.log(0.45 * sr))))
            q = float(np.exp(rng.uniform(np.log(0.1), np.log(20.0))))
            out[i, s] = iir64.cookbook(kind, f, float(rng.uniform(-24, 24)), q, sr)
    return out


def make_signal(kind: str, rng, sr: float, C: int, T: int) -> np.ndarray:
    n = np.arange(T)
    if kind == "noise":
        x = rng.standard_normal((C, T))
    elif kind == "dc_steps":
        x = np.repeat(rng.uniform(-1, 1, (C, 1 + T // 700)), 700, axis=1)[:, :T]
    elif kind == "low_tone":
        x = np.stack([np.sin(2 * np.pi * rng.uniform(20, 60) / sr * n + rng.uniform(0, 6.3)) for _ in range(C)])
    elif kind == "impulses":
        x = np.zeros((C, T))
        x[:, rng.integers(0, T, max(1, T // 3000))] = 1.0
        x[:, 0] = -0.5
    elif kind == "silence":
        x = np.zeros((C, T))
    else:  # a 100 dB drop half way
        x = rng.standard_normal((C, T))
        x[:, T // 2:] *= 1e-5
    return x.astype(np.float32)


def make_batch(rng, sr, C, T, B=len(SIGNALS)) -> np.ndarray:
    return np.stack([make_signal(SIGNALS[b % len(SIGNALS)], rng, sr, C, T) for b in range(B)])


def check_accuracy(eng, sr, C, T, S, per_item=False, seed=0, gain=False, inplace=False, reverse=False, x=None,
                   sos=None):
    """The kernel against float64, per row and per block, relative to the sequential float32 cascade."""
    rng = np.random.default_rng(seed)
    if x is None:
        x = make_batch(rng, sr, C, T)
    B = x.shape[0]
    if sos is None:
        sos = random_sos(rng, sr, S, B if per_item else 1)
    g = rng.uniform(0.25, 4.0, B).astype(np.float32) if gain else None
    xt = torch.from_numpy(x.copy()).to(DEV)  # a copy: in place on the simulator would overwrite x
    gt = None if g is None else torch.from_numpy(g).to(DEV)
    sos_arg = sos[0] if sos.shape[0] == 1 and seed % 2 else sos
    y = eng.sos_filter(xt, torch.from_numpy(sos_arg), gain=gt, reverse=reverse, out=xt if inplace else None)
    s32 = iir64.coefficients(sos, B)
    ref = iir64.reference(x, s32, gain=g, reverse=reverse)
    base = iir64.baseline(x, s32, gain=g, reverse=reverse)
    got = _np(y)
    finite = np.isfinite(ref).all(axis=-1).reshape(-1)
    assert (np.isfinite(got).all(axis=-1).reshape(-1) == finite).all()
    e_k = iir64.block_error(got, ref)[finite]
    e_b = iir64.block_error(base, ref)[finite]
    bound = np.maximum(RATIO * e_b, FLOOR_U)
    where = (sr, C, T, S, per_item, gain, inplace, reverse, seed)
    assert (e_k <= bound).all(), (where, e_k.tolist(), e_b.tolist())
    return e_k, e_b


def check_properties(eng, sr=48000, T=3 * CHUNK + 77):
    rng = np.random.default_rng(21)
    x = make_batch(rng, sr, 2, T)
    xt = torch.from_numpy(x).to(DEV)
    B = x.shape[0]
    # identity sections return the input
    ident = np.tile(np.array([1.0, 0, 0, 1, 0, 0]), (3, 1))
    assert torch.equal(eng.sos_filter(xt, ident), xt)
    # an unstable section: its item is NaN, the others are untouched
    sos = random_sos(rng, sr, 3, B)
    bad = sos.copy()
    bad[2, 1] = [1.0, 0.5, 0.2, 1.0, -1.2, 1.0]  # a2 = 1: a pole on the unit circle
    y_ok = eng.sos_filter(xt, sos)
    y_bad = eng.sos_filter(xt, bad)
    assert bool(torch.isnan(y_bad[2]).all())
    keep = [b for b in range(B) if b != 2]
    assert torch.equal(y_bad[keep], y_ok[keep])
    bad[2, 1] = [1.0, 0.5, 0.2, 1.0, -1.9, 0.9]  # |a1| = 1 + a2: a pole at z = 1
    assert bool(torch.isnan(eng.sos_filter(xt, bad)[2]).all())
    # a NaN sample stays in its row, from that sample on
    xn = x.copy()
    p = CHUNK + 300
    xn[0, 1, p] = np.nan
    xn[3, 0, 17] = np.inf
    yn = _np(eng.sos_filter(torch.from_numpy(xn).to(DEV), sos))
    y0 = _np(y_ok)
    for b, c, q in ((0, 1, p), (3, 0, 17)):
        assert not np.isfinite(yn[b, c, q:]).any() and np.array_equal(yn[b, c, :q], y0[b, c, :q])
        assert np.array_equal(yn[b, 1 - c], y0[b, 1 - c])
    assert np.array_equal(np.delete(yn, (0, 3), axis=0), np.delete(y0, (0, 3), axis=0))
    # batch == single items, reruns identical, shared == the same set per item
    assert torch.equal(eng.sos_filter(xt, sos), y_ok)
    for b in range(B):
        assert torch.equal(eng.sos_filter(xt[b:b + 1].clone(), sos[b:b + 1])[0], y_ok[b]), b
    assert torch.equal(eng.sos_filter(xt, sos[1]), eng.sos_filter(xt, np.repeat(sos[1:2], B, axis=0)))


def check_peak_gain(eng, sr=48000):
    """A steady sine at a peak's centre comes out gain_db louder, within 0.05 dB."""
    from audiotools_b200 import AudioSignal

    T = sr
    n = np.arange(T)
    for f0, g, q in ((1000.0, 12.0, 2.0), (50.0, -9.0, 0.7), (0.4 * sr, 6.0, 8.0), (200.0, 24.0, 20.0)):
        x = np.sin(2 * np.pi * f0 / sr * n)[None, None].astype(np.float32)
        sig = AudioSignal(torch.from_numpy(x).to(DEV), sr).parametric_eq("peaking", f0, g, q)
        y = _np(sig.audio_data)[0, 0, T // 2:]
        level = 20 * np.log10(np.sqrt(np.mean(y ** 2)) / np.sqrt(0.5))
        assert abs(level - g) <= 0.05, (f0, g, q, level)


def check_gradient(eng, sr=44100, T=2 * CHUNK + 300):
    from audiotools_b200 import AudioSignal

    rng = np.random.default_rng(31)
    x = make_batch(rng, sr, 2, T, B=3)
    sos = random_sos(rng, sr, 4, 3)
    gy = rng.standard_normal(x.shape).astype(np.float32)
    xt = torch.from_numpy(x).to(DEV).requires_grad_(True)
    sig = AudioSignal(xt, sr)
    sig.sos_filter(torch.from_numpy(sos))
    sig.audio_data.backward(torch.from_numpy(gy).to(DEV))
    s32 = iir64.coefficients(sos, 3)
    want = iir64.reference(gy, s32, reverse=True)  # the adjoint: the flipped upstream gradient, filtered, flipped back
    base = iir64.baseline(gy, s32, reverse=True)
    e_k, e_b = iir64.block_error(_np(xt.grad), want), iir64.block_error(base, want)
    assert (e_k <= np.maximum(RATIO * e_b, FLOOR_U)).all(), (e_k, e_b)
    # the dot-product test in float64: <H x, g> = <x, H^T g>
    y64 = iir64.reference(x, s32)
    assert np.isclose((y64 * gy).sum(), (x.astype(np.float64) * want).sum(), rtol=1e-9, atol=0)
    # with a pending gain: d/dx of H(g x) is g H^T
    g = torch.tensor([0.5, 2.0, 1.5], device=DEV)
    xt2 = torch.from_numpy(x).to(DEV).requires_grad_(True)
    sig = AudioSignal(xt2, sr)
    sig._pending_gain = g  # as normalize() leaves it when grad mode was off
    sig.sos_filter(sos)
    sig.audio_data.backward(torch.from_numpy(gy).to(DEV))
    want_g = want * _np(g)[:, None, None]
    e_k = iir64.block_error(_np(xt2.grad), want_g)
    assert (e_k <= np.maximum(RATIO * iir64.block_error(base * _np(g)[:, None, None], want_g), FLOOR_U)).all()
    # parameters that require a gradient are refused
    for kw in ({"freq": torch.tensor([1000.0], requires_grad=True)}, {"gain_db": torch.tensor([3.0], requires_grad=True)},
               {"q": torch.tensor([1.0], requires_grad=True)}):
        args = dict(freq=1000.0, gain_db=3.0, q=1.0)
        args.update(kw)
        with pytest.raises(NotImplementedError, match="requires a gradient"):
            AudioSignal(torch.from_numpy(x).to(DEV).requires_grad_(True), sr).parametric_eq("peaking", **args)
    with pytest.raises(NotImplementedError, match="requires a gradient"):
        AudioSignal(torch.from_numpy(x).to(DEV), sr).sos_filter(torch.from_numpy(sos).requires_grad_(True))


def check_api(eng, sr=16000):
    from audiotools_b200 import AudioSignal
    from audiotools_b200.data import transforms as tfm

    rng = np.random.default_rng(41)
    x = torch.from_numpy(make_batch(rng, sr, 2, sr // 2)).to(DEV)
    B = x.shape[0]
    lib = eng.lib
    sos = random_sos(rng, sr, 2, B)
    n0, k0 = eng.launches, lib.kernel_launches.value
    out = eng.sos_filter(x, sos)
    assert eng.launches - n0 == LAUNCHES and lib.kernel_launches.value - k0 == LAUNCHES
    # a pending gain is consumed by the filter's own passes
    n0 = eng.launches
    eng.lufs(x, sr, target_db=torch.tensor([-16.0], device=DEV))
    n_lufs = eng.launches - n0
    n0 = eng.launches
    sig = AudioSignal(x.clone(), sr).normalize(-16.0)
    sig._stft_data = torch.zeros(1)
    sig.sos_filter(sos)
    assert eng.launches - n0 == n_lufs + LAUNCHES
    assert sig._pending_gain is None and sig._loudness is None and sig.stft_data is None
    ref = AudioSignal(x.clone(), sr).normalize(-16.0)
    assert torch.equal(sig.audio_data, eng.sos_filter(ref.audio_data, sos))  # == materialise, then filter
    assert torch.equal(AudioSignal(x.clone(), sr).sos_filter(sos).audio_data, out)
    # parametric_eq == the cookbook's sections through sos_filter
    kinds = ["low_shelf", "peaking", "notch"]
    freq = np.array([100.0, 1000.0, 3000.0])
    gdb = np.array([[6.0, -3.0, 0.0]] * B)
    q = np.array([0.7, 2.0, 5.0])
    y = AudioSignal(x.clone(), sr).parametric_eq(kinds, freq, gdb, q).audio_data
    want = np.stack([np.stack([iir64.cookbook(k, freq[i], gdb[b, i], q[i], sr) for i, k in enumerate(kinds)])
                     for b in range(B)])
    assert float((y - eng.sos_filter(x, want)).abs().max()) <= 1e-4 * float(y.abs().max())
    # refusals: a bad kind / freq / q / S, and the C entry point's argument checks launch nothing
    k0 = lib.kernel_launches.value
    sig = AudioSignal(x.clone(), sr)
    with pytest.raises(ValueError, match="kind"):
        sig.parametric_eq("shelf", 100.0)
    with pytest.raises(ValueError, match="freq"):
        sig.parametric_eq("peaking", sr / 2)
    with pytest.raises(ValueError, match="freq"):
        sig.parametric_eq("peaking", 0.0)
    with pytest.raises(ValueError, match="q must be positive"):
        sig.parametric_eq("peaking", 100.0, q=0.0)
    with pytest.raises(ValueError, match="sections"):
        eng.sos_filter(x, np.tile(np.array([1.0, 0, 0, 1, 0, 0]), (9, 1)))
    with pytest.raises(ValueError, match="sos must be"):
        eng.sos_filter(x, np.ones((2, 3, 6)))
    p, (Bx, C, T) = x.data_ptr(), x.shape
    bad = [((None, None, Bx, C, T, p, 1, 2, 0, p, p, None), b"null pointer"),
           ((p, None, Bx, C, T, None, 1, 2, 0, p, p, None), b"null pointer"),
           ((p, None, Bx, C, T, p, 1, 2, 0, None, p, None), b"null pointer"),
           ((p, None, Bx, C, T, p, 1, 2, 0, p, None, None), b"null pointer"),
           ((p, None, Bx, 0, T, p, 1, 2, 0, p, p, None), b"bad shape"),
           ((p, None, Bx, C, 0, p, 1, 2, 0, p, p, None), b"bad shape"),
           ((p, None, Bx, C, 1 << 62, p, 1, 2, 0, p, p, None), b"overflows"),
           ((p, None, Bx, C, T, p, 1, 0, 0, p, p, None), b"sections"),
           ((p, None, Bx, C, T, p, 1, 9, 0, p, p, None), b"sections"),
           ((p, None, Bx, C, T, p, 2, 2, 0, p, p, None), b"sos_items")]
    for args, msg in bad:
        assert lib.b2a_sos_filter_f32(*args) == -1 and msg in lib.b2a_last_error(), msg
    assert lib.b2a_sos_filter_workspace_bytes(Bx, C, 1 << 62, 2) == 0
    assert lib.b2a_sos_filter_workspace_bytes(Bx, C, T, 9) == 0
    assert lib.b2a_sos_filter_workspace_bytes(2, 3, CHUNK + 1, 4) == 8 * 2 * (2 * 3 * 2 * 8)  # e and s in double
    assert lib.kernel_launches.value == k0
    # the transform under a partial mask and inside Compose: unselected items come back unchanged
    t = tfm.ParametricEQ(prob=0.5)
    comp = tfm.Compose([t])
    sig = AudioSignal(x.clone(), sr)
    kw = comp.batch_instantiate(list(range(B)), sig)
    sub = kw[comp.name][t.name]
    mask = sub["mask"]
    assert 0 < int(mask.sum()) < B
    assert float(sub["freq"].max()) <= 0.45 * sr
    y = comp(sig.clone(), **kw).audio_data
    m = mask.to(y.device)
    kinds = [b[0] for b in t.bands]
    want = AudioSignal(x[m].clone(), sr).parametric_eq(kinds, sub["freq"][mask], sub["gain_db"][mask],
                                                       sub["q"][mask]).audio_data
    assert torch.equal(y[~m], x[~m]) and not torch.equal(y[m], x[m])
    assert float((y[m] - want).abs().max()) == 0.0
    kw1 = t.instantiate(3, sig)
    assert kw1[t.name]["freq"].shape == (len(kinds),)


# --------------------------------------------------------------------------- tests
LENGTHS = (1, 2, 700, CHUNK - 1, CHUNK, CHUNK + 1, 5 * CHUNK + 17, 40 * CHUNK + 3)


@pytest.mark.parametrize("C", [1, 2, 5])
@pytest.mark.parametrize("sr", [16000, 44100, 48000, 192000])
def test_against_float64(eng, sr, C):
    for i, T in enumerate(LENGTHS):
        check_accuracy(eng, sr, C, T, S=1 + (i + C) % 8, per_item=i % 2 == 1, seed=100 * i + C,
                       gain=i % 3 == 0, inplace=i % 4 == 1, reverse=i % 3 == 2)


@pytest.mark.parametrize("S", list(range(1, 9)))
def test_sections(eng, S):
    for per_item in (False, True):
        for reverse in (False, True):
            check_accuracy(eng, 48000, 2, 7 * CHUNK + 5, S, per_item=per_item, seed=S, reverse=reverse)


@pytest.mark.parametrize("kind", KINDS)
def test_every_kind_at_the_edges_of_its_parameters(eng, kind):
    sr = 48000
    rows = []
    for f in (10.0, 20.0, 100.0, 0.45 * sr):
        for q in (0.1, 0.7071, 20.0):
            for g in (-24.0, 24.0):
                rows.append(iir64.cookbook(kind, f, g, q, sr))
    sos = np.stack(rows)[:, None]
    rng = np.random.default_rng(3)
    x = np.stack([make_signal(SIGNALS[i % len(SIGNALS)], rng, sr, 1, 9 * CHUNK + 11) for i in range(len(rows))])
    check_accuracy(eng, sr, 1, x.shape[-1], 1, x=x, sos=sos)
    check_accuracy(eng, sr, 1, x.shape[-1], 1, x=x, sos=sos, reverse=True)


def test_a_long_row(eng):
    """A row of 1000 chunks: 32 batches of the carry kernel's warp scan, with a 20 Hz Q 8 +12 dB peak."""
    sr = 48000
    sos = np.stack([iir64.cookbook("peaking", 20.0, 12.0, 8.0, sr), iir64.cookbook("low_shelf", 30.0, 12.0, 0.7, sr),
                    iir64.cookbook("high_pass", 10.0, 0.0, 0.7071, sr)])[None]
    rng = np.random.default_rng(9)
    x = np.stack([make_signal(s, rng, sr, 1, 1000 * CHUNK + 9) for s in ("noise", "low_tone", "drop")])
    check_accuracy(eng, sr, 1, x.shape[-1], 3, x=x, sos=sos)


def test_properties(eng):
    check_properties(eng)


def test_peak_gain_at_its_centre(eng):
    check_peak_gain(eng)


def test_gradient(eng):
    check_gradient(eng)


def test_api(eng):
    check_api(eng)


def test_more_than_2_31_elements(eng):
    """[3, 2, 400e6]: 2.4e9 samples, zeros with a burst past flat index 2^31; only the burst's row changes, in place."""
    B, C, T = 3, 2, 400_000_000
    x = torch.zeros(B, C, T, device=DEV)
    p = T - 20000
    rng = np.random.default_rng(4)
    burst = torch.from_numpy(rng.standard_normal(3000).astype(np.float32)).to(DEV)
    x[2, 1, p:p + 3000] = burst
    sos = iir64.cookbook("peaking", 1000.0, 6.0, 2.0, 48000)[None]
    small = torch.zeros(1, 1, 20000, device=DEV)
    small[0, 0, 0:3000] = burst
    want = eng.sos_filter(small, sos)
    out = eng.sos_filter(x, sos, out=x)
    got = out[2, 1, p:]
    assert float((got - want[0, 0]).abs().max()) <= 1e-5 * float(want.abs().max())
    assert float(out[2, 1, :p].abs().max()) == 0 and float(out[:2].abs().max()) == 0 and float(out[2, 0].abs().max()) == 0
    del x, out
    torch.cuda.empty_cache()


def test_no_host_sync(eng):
    from audiotools_b200 import AudioSignal
    from audiotools_b200.core import util
    from audiotools_b200.data import transforms as tfm

    x = 0.5 * torch.randn(4, 2, 48000, device=DEV)
    sos = torch.from_numpy(random_sos(np.random.default_rng(0), 48000, 3, 4)).to(DEV)
    t = tfm.ParametricEQ(prob=0.5)
    sig = AudioSignal(x.clone(), 48000)
    kw = util.prepare_batch(t.batch_instantiate(list(range(4)), sig), DEV)
    db = torch.tensor(-16.0, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        sig.normalize(db).sos_filter(sos)
        sig.parametric_eq("peaking", 1000.0, 6.0, 2.0)
        t(sig, **kw)
        eng.sos_filter(x, sos, reverse=True)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_launches_match_the_profiler(eng):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    x = 0.5 * torch.randn(64, 2, 441000, device=DEV)
    sos = random_sos(np.random.default_rng(1), 44100, 4, 1)
    eng.sos_filter(x, sos)
    torch.cuda.synchronize()
    n0, k0 = eng.launches, eng.lib.kernel_launches.value
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        eng.sos_filter(x, sos)
        torch.cuda.synchronize()
    added = eng.launches - n0
    assert eng.lib.kernel_launches.value - k0 == added
    gpu = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    if not gpu:
        pytest.skip("the profiler recorded no GPU activity")
    names = [e.name for e in gpu]
    assert (sum("b2a::iir" in n for n in names), added) == (LAUNCHES, LAUNCHES), names
