"""``core.iir.sosfilt(..., zi)`` / ``sosfiltfilt`` / ``AudioSignal.sos_filter(zero_phase=True)`` on the H100
(``-m gpu``): the stateful and zero-phase cascades of csrc/iir.cu against the float64 oracle of tests/iirfilt64.py,
with the bound of tests/test_gpu_iir.py (the worst 1024-sample block within RATIO times the float32 baseline's, or
FLOOR_U u).

* zero phase, per sample: S = 1 .. 8, shared and per-item sections, cookbook kinds and odd-order butter / cheby1
  designs (sections with b2 = a2 = 0), every padtype, the default padlen, 0 and an explicit one, T just above the
  padding, the chunk length +- 1, 32 chunks +- 1 and several chunks, noise, DC steps, low tones and a 100 dB drop,
  with and without a gain;
* streaming: rows split at random points (pieces of 1 sample, pieces across chunk and 32-chunk boundaries), zf
  chained into zi, against one float64 pass; zi = 0 against ``sos_filter`` bit for bit;
* properties: a symmetric impulse response, unstable items, NaN samples, batch == single items, reruns, bypassed
  items, the pending gain;
* the gradient against the float64 Jacobian, a dot-product test, refusals;
* the API: refused arguments, launch counts, no host sync, the profiler's launch count.
tests/test_sim_iir_state.py runs the same checks at smaller sizes on the CPU simulator."""
import numpy as np
import pytest
import torch
from scipy import signal as sps

import tests.test_gpu_iir as G
from tests import iir64, iirfilt64

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CHUNK = G.CHUNK
RATIO, FLOOR_U = G.RATIO, G.FLOOR_U
LAUNCHES_ZI, LAUNCHES_FILTFILT, LAUNCHES_BACKWARD = 3, 6, 7  # DESIGN.md K19
PADTYPES = ("odd", "even", "constant", None)
SIGNALS = ("noise", "dc_steps", "low_tone", "drop")


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


def _np(t):
    return t.detach().cpu().double().numpy()


def designed_sos(rng, sr, S, items):
    """[items, S, 6]: cookbook sections, with a butter or cheby1 design of odd order (b2 = a2 = 0 in its first-order
    section) in some items."""
    sos = G.random_sos(rng, sr, S, items)
    for i in range(items):
        if S >= 2 and i % 2 == 1:
            order = 2 * int(rng.integers(1, S)) - 1 if S > 1 else 1
            f = float(np.exp(rng.uniform(np.log(20.0), np.log(0.4 * sr))))
            btype = ("lowpass", "highpass")[int(rng.integers(2))]
            d = sps.butter(order, f, btype, fs=sr, output="sos") if i % 4 == 1 else \
                sps.cheby1(order, 1.0, f, btype, fs=sr, output="sos")
            sos[i, :d.shape[0]] = d
    return sos


def bound_ok(got, ref, base, where):
    finite = np.isfinite(ref).all(axis=-1).reshape(-1)
    assert (np.isfinite(got).all(axis=-1).reshape(-1) == finite).all(), where
    e_k = iir64.block_error(got, ref)[finite]
    e_b = iir64.block_error(base, ref)[finite]
    assert (e_k <= np.maximum(RATIO * e_b, FLOOR_U)).all(), (where, e_k.tolist(), e_b.tolist())
    return e_k, e_b


def check_filtfilt(eng, sr, C, T, S, per_item=False, seed=0, gain=False, padtype="odd", padlen=None, x=None,
                   sos=None):
    from audiotools_b200.core import iir

    rng = np.random.default_rng(seed)
    if x is None:
        x = np.stack([G.make_signal(SIGNALS[b % len(SIGNALS)], rng, sr, C, T) for b in range(len(SIGNALS))])
    B = x.shape[0]
    if sos is None:
        sos = designed_sos(rng, sr, S, B if per_item else 1)
    g = rng.uniform(0.25, 4.0, B).astype(np.float32) if gain else None
    xt = torch.from_numpy(x.copy()).to(DEV)
    if g is None and seed % 2 == 0:
        y = iir.sosfiltfilt(torch.from_numpy(sos[0] if sos.shape[0] == 1 else sos), xt, padtype, padlen)
    else:
        y = eng.sos_filtfilt(xt, sos, padtype, padlen, gain=None if g is None else torch.from_numpy(g).to(DEV))
    s32 = iir64.coefficients(sos, B)
    ref = iirfilt64.reference_filtfilt(x, s32, g, padtype, padlen)
    base = iirfilt64.baseline_filtfilt(x, s32, g, padtype, padlen)
    return bound_ok(_np(y), ref, base, (sr, C, T, S, per_item, gain, padtype, padlen, seed))


def check_streaming(eng, sr, C, T, S, seed=0, cuts=None):
    """One row split into pieces, zf chained into zi: y against one float64 pass, every zf against scipy's."""
    from audiotools_b200.core import iir

    rng = np.random.default_rng(seed)
    x = np.stack([G.make_signal(SIGNALS[b % len(SIGNALS)], rng, sr, C, T) for b in range(len(SIGNALS))])
    B = x.shape[0]
    sos = designed_sos(rng, sr, S, B)
    s32 = iir64.coefficients(sos, B)
    if cuts is None:
        cuts = np.unique(np.concatenate([rng.integers(1, T, 6), [1, 2, CHUNK + 3, CHUNK + 4, 32 * CHUNK - 5]]))
    cuts = [0] + [int(c) for c in cuts if 0 < c < T] + [T]
    zi = torch.zeros(S, B, C, 2, dtype=torch.float64, device=DEV)
    zi_b = np.zeros((S, B, C, 2))  # the float32 baseline's chain
    zi_r = np.zeros((S, B, C, 2))  # float64
    ys, yb = [], []
    xt = torch.from_numpy(x).to(DEV)
    for a, e in zip(cuts[:-1], cuts[1:]):
        y, zf = iir.sosfilt(torch.from_numpy(sos), xt[..., a:e].contiguous(), zi=zi)
        _, zf_r = iirfilt64.reference_state(x[..., a:e], s32, zi_r)
        y_b, zf_b = iirfilt64.baseline_state(x[..., a:e], s32, zi_b)
        got = _np(zf)
        scale = np.abs(zf_r).max(axis=(0, 3))[None, :, :, None]  # the row's largest |zf| component
        e_k = (np.abs(got - zf_r) / np.where(scale > 0, scale, 1)).max(axis=(0, 3))
        e_b = (np.abs(zf_b - zf_r) / np.where(scale > 0, scale, 1)).max(axis=(0, 3))
        assert ((e_k <= FLOOR_U * iir64.U) | (e_k <= RATIO * e_b)).all(), (a, e, e_k.max(), e_b.max())
        ys.append(_np(y))
        yb.append(y_b)
        zi, zi_r, zi_b = zf, zf_r, zf_b.astype(np.float32)
    ref = iir64.reference(x, s32)
    base = iir64.baseline(x, s32)
    return bound_ok(np.concatenate(ys, axis=-1), ref, base, ("stream", sr, C, T, S, seed, cuts))


def check_zero_state_equals_sos_filter(eng, T=2 * CHUNK + 9):
    from audiotools_b200.core import iir

    rng = np.random.default_rng(5)
    for S in range(1, 9):
        x = torch.from_numpy(G.make_batch(rng, 48000, 2, T)).to(DEV)
        sos = G.random_sos(rng, 48000, S, x.shape[0])
        y, zf = iir.sosfilt(sos, x, zi=torch.zeros(S, x.shape[0], 2, 2, device=DEV))
        assert torch.equal(y, eng.sos_filter(x, sos)), S
        assert torch.equal(iir.sosfilt(sos, x), eng.sos_filter(x, sos)), S


def check_properties(eng, sr=48000, T=3 * CHUNK + 77):
    from audiotools_b200 import AudioSignal

    rng = np.random.default_rng(21)
    x = np.stack([G.make_signal(SIGNALS[b % len(SIGNALS)], rng, sr, 2, T) for b in range(len(SIGNALS))])
    xt = torch.from_numpy(x).to(DEV)
    B = x.shape[0]
    sos = designed_sos(rng, sr, 3, B)
    y_ok = eng.sos_filtfilt(xt, sos)
    # an impulse far from the edges: a symmetric response
    imp = np.zeros((1, 1, T), np.float32)
    c = T // 2
    imp[0, 0, c] = 1.0
    peak = G.random_sos(np.random.default_rng(2), sr, 2, 1)
    h = _np(eng.sos_filtfilt(torch.from_numpy(imp).to(DEV), peak))[0, 0]
    ref = iirfilt64.reference_filtfilt(imp, iir64.coefficients(peak, 1))[0, 0]
    n = min(c, T - 1 - c)
    assert np.abs(h[c - n:c + 1][::-1] - h[c:c + n + 1]).max() <= FLOOR_U * iir64.U * np.abs(ref).max() + \
        np.abs(ref[c - n:c + 1][::-1] - ref[c:c + n + 1]).max()
    # an unstable item is NaN, the others are untouched
    bad = sos.copy()
    bad[2, 1] = [1.0, 0.5, 0.2, 1.0, -1.2, 1.0]
    y_bad = eng.sos_filtfilt(xt, bad)
    assert bool(torch.isnan(y_bad[2]).all())
    keep = [b for b in range(B) if b != 2]
    assert torch.equal(y_bad[keep], y_ok[keep])
    zi = torch.ones(3, B, 2, 2, dtype=torch.float64, device=DEV)
    y_s, zf = eng.sos_filter_zi(xt, bad, zi)
    assert bool(torch.isnan(y_s[2]).all()) and bool(torch.isnan(zf[:, 2]).all()) and bool(torch.isfinite(zf[:, 0]).all())
    # a NaN or inf sample makes its whole row non-finite under zero phase; other rows are unaffected
    xn = x.copy()
    xn[0, 1, CHUNK + 300] = np.nan
    xn[3, 0, 17] = np.inf
    yn = _np(eng.sos_filtfilt(torch.from_numpy(xn).to(DEV), sos))
    y0 = _np(y_ok)
    for b, ch in ((0, 1), (3, 0)):
        assert not np.isfinite(yn[b, ch]).any()
        assert np.array_equal(yn[b, 1 - ch], y0[b, 1 - ch])
    assert np.array_equal(np.delete(yn, (0, 3), axis=0), np.delete(y0, (0, 3), axis=0))
    # batch == single items, reruns identical
    assert torch.equal(eng.sos_filtfilt(xt, sos), y_ok)
    for b in range(B):
        assert torch.equal(eng.sos_filtfilt(xt[b:b + 1].clone(), sos[b:b + 1])[0], y_ok[b]), b
    # AudioSignal: bypassed items come back bit for bit, the pending gain is consumed in the passes
    byp = torch.tensor([True, False, True, False], device=DEV)
    sig = AudioSignal(xt.clone(), sr).sos_filter(sos, zero_phase=True, _bypass=byp)
    assert torch.equal(sig.audio_data[byp], xt[byp]) and torch.equal(sig.audio_data[~byp], y_ok[~byp])
    n0 = eng.launches
    sig = AudioSignal(xt.clone(), sr).normalize(-16.0)
    n_norm = eng.launches - n0
    sig._stft_data = torch.zeros(1)
    n0 = eng.launches
    sig.sos_filter(sos, zero_phase=True)
    assert eng.launches - n0 == LAUNCHES_FILTFILT
    assert sig._pending_gain is None and sig._loudness is None and sig.stft_data is None
    ref_sig = AudioSignal(xt.clone(), sr).normalize(-16.0)
    assert torch.equal(sig.audio_data, eng.sos_filtfilt(ref_sig.audio_data, sos))
    assert n_norm > 0


def check_gradient(eng, sr=44100, T=257):
    """Per sample against the float64 Jacobian of scipy's sosfiltfilt (columns from unit impulses); a dot-product
    test at about 40 k samples; the refusals."""
    from audiotools_b200 import AudioSignal
    from audiotools_b200.core import iir

    rng = np.random.default_rng(31)
    for padtype, padlen, S in (("odd", None, 3), ("even", 40, 2), ("constant", None, 4), (None, None, 1),
                               ("odd", 0, 2)):
        B = 3
        x = np.stack([G.make_signal(SIGNALS[b], rng, sr, 2, T) for b in range(B)])
        sos = designed_sos(rng, sr, S, B)
        gy = rng.standard_normal(x.shape).astype(np.float32)
        xt = torch.from_numpy(x).to(DEV).requires_grad_(True)
        iir.sosfiltfilt(torch.from_numpy(sos), xt, padtype, padlen).backward(torch.from_numpy(gy).to(DEV))
        s32 = iir64.coefficients(sos, B)
        want = np.empty(x.shape)
        for b in range(B):
            J = sps.sosfiltfilt(s32[b].astype(np.float64), np.eye(T), axis=-1, padtype=padtype, padlen=padlen)
            want[b] = gy[b].astype(np.float64) @ J.T  # row i of J: the response to an impulse at i
        e = iir64.block_error(_np(xt.grad), want)
        assert (e <= FLOOR_U).all(), (padtype, padlen, S, e)
    # with a pending gain, through AudioSignal: d/dx of F(g x) is g F^T
    x = np.stack([G.make_signal(SIGNALS[b], rng, sr, 1, T) for b in range(2)])
    sos = designed_sos(rng, sr, 2, 2)
    gy = rng.standard_normal(x.shape).astype(np.float32)
    xt = torch.from_numpy(x).to(DEV).requires_grad_(True)
    sig = AudioSignal(xt, sr)
    g = torch.tensor([0.5, 2.0], device=DEV)
    sig._pending_gain = g
    sig.sos_filter(sos, zero_phase=True)
    sig.audio_data.backward(torch.from_numpy(gy).to(DEV))
    s32 = iir64.coefficients(sos, 2)
    want = np.stack([_np(g)[b] * gy[b].astype(np.float64) @ sps.sosfiltfilt(s32[b].astype(np.float64), np.eye(T),
                                                                            axis=-1).T for b in range(2)])
    assert (iir64.block_error(_np(xt.grad), want) <= FLOOR_U).all()
    # the dot-product test: <F x, g> = <x, F^T g>, F^T g from the kernels, F x from scipy in float64
    T2 = 40_000
    x = np.stack([G.make_signal(s, rng, 48000, 2, T2) for s in ("noise", "low_tone")])
    sos = np.concatenate([sps.butter(3, 2000.0, fs=48000, output="sos"),
                          iir64.cookbook("peaking", 100.0, 6.0, 2.0, 48000)[None]])  # passes most of both rows
    gy = rng.standard_normal(x.shape).astype(np.float32)
    gx = _np(eng.sos_filtfilt_backward(torch.from_numpy(gy).to(DEV), sos))
    y64 = iirfilt64.reference_filtfilt(x, iir64.coefficients(sos, 2))
    lhs, rhs = (y64 * gy).sum(), (x.astype(np.float64) * gx).sum()
    scale = np.linalg.norm(y64) * np.linalg.norm(gy) + np.linalg.norm(x) * np.linalg.norm(gx)
    assert abs(lhs - rhs) <= 1e-6 * scale, (lhs, rhs, scale)
    # refusals: sosfilt with zi has no backward, sos is a constant
    xg = torch.from_numpy(x[:, :, :100].copy()).to(DEV)
    zi = torch.zeros(4, 2, 2, 2, dtype=torch.float64, device=DEV)
    with pytest.raises(NotImplementedError, match="requires a gradient"):
        iir.sosfilt(sos, xg.clone().requires_grad_(True), zi=zi)
    with pytest.raises(NotImplementedError, match="requires a gradient"):
        iir.sosfilt(sos, xg, zi=zi.clone().requires_grad_(True))
    with pytest.raises(NotImplementedError, match="requires a gradient"):
        iir.sosfiltfilt(torch.from_numpy(sos).requires_grad_(True), xg)
    with pytest.raises(NotImplementedError, match="requires a gradient"):
        AudioSignal(xg.clone().requires_grad_(True), sr).sos_filter(torch.from_numpy(sos).requires_grad_(True),
                                                                     zero_phase=True)


def check_api(eng, sr=16000):
    from audiotools_b200.core import iir

    rng = np.random.default_rng(41)
    x = torch.from_numpy(G.make_batch(rng, sr, 2, sr // 2)).to(DEV)
    B, C, T = x.shape
    lib = eng.lib
    sos = G.random_sos(rng, sr, 2, B)
    zi = torch.zeros(2, B, C, 2, dtype=torch.float64, device=DEV)
    for fn, n in ((lambda: eng.sos_filter_zi(x, sos, zi), LAUNCHES_ZI),
                  (lambda: eng.sos_filtfilt(x, sos), LAUNCHES_FILTFILT),
                  (lambda: eng.sos_filtfilt(x, sos, padtype=None), LAUNCHES_FILTFILT),
                  (lambda: eng.sos_filtfilt_backward(x, sos), LAUNCHES_BACKWARD)):
        n0, k0 = eng.launches, lib.kernel_launches.value
        fn()
        assert eng.launches - n0 == n and lib.kernel_launches.value - k0 == n
    # float32 zi is taken as well
    y32, _ = eng.sos_filter_zi(x, sos, zi.float())
    assert torch.equal(y32, eng.sos_filter_zi(x, sos, zi)[0])
    k0 = lib.kernel_launches.value
    with pytest.raises(ValueError, match="padtype"):
        iir.sosfiltfilt(sos, x, padtype="reflect")
    with pytest.raises(ValueError, match="padlen"):
        iir.sosfiltfilt(sos, x, padlen=-1)
    with pytest.raises(ValueError, match="zi must be"):
        iir.sosfilt(sos, x, zi=torch.zeros(2, B, 2, device=DEV))
    with pytest.raises(ValueError, match="greater than the padding"):
        iir.sosfiltfilt(sos, x, padlen=T)
    with pytest.raises(ValueError, match="greater than the padding"):
        iir.sosfiltfilt(sos, x[..., :15].contiguous())  # 3 (2S + 1) = 15
    iir.sosfiltfilt(sos, x[..., :15].contiguous(), padlen=14)
    iir.sosfiltfilt(sos, x[..., :15].contiguous(), padtype=None)
    k0 = lib.kernel_launches.value
    p = x.data_ptr()
    bad_zi = [((None, None, B, C, T, p, 1, 2, p, p, None, p, None), b"null pointer"),
              ((p, None, B, C, T, p, 1, 2, None, p, None, p, None), b"null pointer"),
              ((p, None, B, C, T, p, 1, 9, p, p, None, p, None), b"sections"),
              ((p, None, B, C, T, p, 2, 2, p, p, None, p, None), b"sos_items"),
              ((p, None, B, 0, T, p, 1, 2, p, p, None, p, None), b"bad shape")]
    for args, msg in bad_zi:
        assert lib.b2a_sos_filter_zi_f32(*args) == -1 and msg in lib.b2a_last_error(), msg
    bad_ff = [((None, None, B, C, T, p, 1, 2, 1, -1, p, p, None), b"null pointer"),
              ((p, None, B, C, T, p, 1, 2, 5, -1, p, p, None), b"padtype"),
              ((p, None, B, C, T, p, 1, 2, -1, -1, p, p, None), b"padtype"),
              ((p, None, B, C, T, p, 1, 2, 1, T, p, p, None), b"must exceed the padding"),
              ((p, None, B, C, 15, p, 1, 2, 1, -1, p, p, None), b"must exceed the padding"),
              ((p, None, B, C, 1 << 61, p, 1, 2, 1, -1, p, p, None), b"overflows"),
              ((p, None, B, C, T, p, 1, 0, 1, -1, p, p, None), b"sections"),
              ((p, None, B, C, T, p, 3, 2, 1, -1, p, p, None), b"sos_items")]
    for args, msg in bad_ff:
        assert lib.b2a_sos_filtfilt_f32(*args) == -1 and msg in lib.b2a_last_error(), msg
        assert lib.b2a_sos_filtfilt_backward_f32(*args) == -1 and msg in lib.b2a_last_error(), msg
    assert lib.b2a_sos_filtfilt_workspace_bytes(B, C, 15, 2, 1, -1) == 0
    assert lib.b2a_sos_filtfilt_workspace_bytes(B, C, T, 2, 4, -1) == 0
    assert lib.b2a_sos_filtfilt_workspace_bytes(B, C, 16, 2, 1, -1) > 0
    assert lib.b2a_sos_filtfilt_workspace_bytes(B, C, 2, 2, 0, -1) > 0
    assert lib.kernel_launches.value == k0


# --------------------------------------------------------------------------- tests
def lengths(S):
    edge = 3 * (2 * S + 1)
    return (edge + 1, edge + 2, CHUNK - 1, CHUNK + 1, 32 * CHUNK - 1, 32 * CHUNK + 1, 70 * CHUNK + 5)


@pytest.mark.parametrize("S", list(range(1, 9)))
def test_zero_phase_against_float64(eng, S):
    for i, T in enumerate(lengths(S)):
        check_filtfilt(eng, 48000, 2, T, S, per_item=i % 2 == 1, seed=10 * S + i, gain=i % 3 == 0,
                       padtype=PADTYPES[i % 4])


@pytest.mark.parametrize("padtype", PADTYPES)
@pytest.mark.parametrize("padlen", [None, 0, 100])
def test_padding(eng, padtype, padlen):
    for sr, C, T, S in ((16000, 1, 2 * CHUNK + 7, 3), (44100, 2, 5 * CHUNK, 5), (192000, 5, 120, 2)):
        check_filtfilt(eng, sr, C, T, S, per_item=True, seed=T, padtype=padtype, padlen=padlen)


@pytest.mark.parametrize("kind", G.KINDS)
def test_every_kind_zero_phase(eng, kind):
    sr = 48000
    rows = [iir64.cookbook(kind, f, g, q, sr) for f in (10.0, 100.0, 0.45 * sr) for q in (0.1, 20.0)
            for g in (-24.0, 24.0)]
    sos = np.stack(rows)[:, None]
    rng = np.random.default_rng(3)
    x = np.stack([G.make_signal(SIGNALS[i % len(SIGNALS)], rng, sr, 1, 9 * CHUNK + 11) for i in range(len(rows))])
    check_filtfilt(eng, sr, 1, x.shape[-1], 1, x=x, sos=sos)


def test_a_long_row_zero_phase(eng):
    sr = 48000
    sos = np.concatenate([sps.butter(5, 30.0, "highpass", fs=sr, output="sos"),
                          iir64.cookbook("peaking", 20.0, 12.0, 8.0, sr)[None]])[None]
    rng = np.random.default_rng(9)
    x = np.stack([G.make_signal(s, rng, sr, 1, 1000 * CHUNK + 9) for s in ("noise", "low_tone", "drop")])
    check_filtfilt(eng, sr, 1, x.shape[-1], 4, x=x, sos=sos)


@pytest.mark.parametrize("S", [1, 2, 4, 8])
def test_streaming(eng, S):
    check_streaming(eng, 48000, 2, 70 * CHUNK + 3, S, seed=S)
    check_streaming(eng, 44100, 1, 3 * CHUNK, S, seed=S + 10, cuts=list(range(1, 40)) + [CHUNK - 1, CHUNK, CHUNK + 1])


def test_zero_state_equals_sos_filter(eng):
    check_zero_state_equals_sos_filter(eng)


def test_properties(eng):
    check_properties(eng)


def test_gradient(eng):
    check_gradient(eng)


def test_api(eng):
    check_api(eng)


def test_no_host_sync(eng):
    from audiotools_b200 import AudioSignal
    from audiotools_b200.core import iir

    x = 0.5 * torch.randn(4, 2, 48000, device=DEV)
    sos = torch.from_numpy(G.random_sos(np.random.default_rng(0), 48000, 3, 4)).to(DEV)
    zi = torch.zeros(3, 4, 2, 2, dtype=torch.float64, device=DEV)
    sig = AudioSignal(x.clone(), 48000)
    xg = x.clone().requires_grad_(True)
    db = torch.tensor(-16.0, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        sig.normalize(db).sos_filter(sos, zero_phase=True)
        iir.sosfilt(sos, x, zi=zi)
        iir.sosfiltfilt(sos, x, padtype="even", padlen=30)
        iir.sosfiltfilt(sos, xg).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_launches_match_the_profiler(eng):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    x = 0.5 * torch.randn(16, 2, 441000, device=DEV)
    sos = G.random_sos(np.random.default_rng(1), 44100, 4, 1)
    eng.sos_filtfilt(x, sos)
    eng.sos_filtfilt_backward(x, sos)
    torch.cuda.synchronize()
    n0, k0 = eng.launches, eng.lib.kernel_launches.value
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        eng.sos_filtfilt(x, sos)
        eng.sos_filtfilt_backward(x, sos)
        torch.cuda.synchronize()
    added = eng.launches - n0
    assert eng.lib.kernel_launches.value - k0 == added
    gpu = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    if not gpu:
        pytest.skip("the profiler recorded no GPU activity")
    names = [e.name for e in gpu]
    want = LAUNCHES_FILTFILT + LAUNCHES_BACKWARD
    assert (sum("b2a::iir" in n for n in names), added) == (want, want), names
