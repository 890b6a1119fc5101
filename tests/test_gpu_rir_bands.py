"""Octave-band walls and air absorption of ``core.room.image_source_ir(..., bands=K, air_absorption=)`` and
``transforms.SyntheticRoomImpulseResponse(bands=)`` on the H100 (``-m gpu``): csrc/rir.cu's band path (DESIGN.md K20
"Bands") against the float64 oracle of tests/rir_bands64.py.

* the flat path is untouched: equal beta in every band and no air give the ``bands=None`` output bit for bit, images
  only and hybrid, K = 1, 3 and 8, 8 to 96 kHz; K = 1 with its own beta is the flat call with that beta;
* per sample against float64: |y - y64| <= sum_k |LP_k| * (w_k + w_{k+1}) + w_{K'-1} + the crossovers' fftconv budget
  (tests/timedomain64.py) + the rounding of the differences and of the final sum, with w_k = 8 u G_k (G_k rir64.bound
  of band k's images) plus, with a tail, the tail's terms of tests/test_gpu_rir_diffuse.py; at 8 to 96 kHz, around the tile, the window and the lowest crossover's
  length, with beta 0 and 1, per wall and per band, air on and off, C = 1, 2 and 8, max_order -1 to 10, the hybrid;
* physics: each octave's level of an anechoic direct path falls by a_k d dB; the per-octave Schroeder T20 of a hybrid
  response follows the bands' Sabine RT60s and the images-only response of the same room; exact zeros before the
  direct path - Tw/2 - half_0;
* bands at or above Nyquist are checked but not computed: K = 8 at 8 kHz equals K = 6, bit for bit;
* the API: refusals that launch nothing, reruns and a batch against its items bit for bit, no host sync, launch
  counts against the profiler, more than 2^31 band-row elements, and the transform's seeded draws.
tests/test_sim_rir_bands.py runs the same checks at small sizes on the CPU simulator."""
import math

import numpy as np
import pytest
import torch

from tests import rir64
from tests import rir_bands64 as R64
from tests import rir_diffuse64 as D
from tests import timedomain64 as T64
from tests.test_gpu_rir import ROOMS, scene, walls

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
K_BUDGET = 8.0   # u, the images' per-sample bound (tests/test_gpu_rir.py)
ENV_REL = 1e-4   # the tail's amplitude against the converged envelope (tests/test_gpu_rir_diffuse.py)
TILE = 512       # csrc/rir.cu: samples per CTA
WORST = {}       # worst |y - y64| / bound per rate


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


def rir(room, src, mics, fs, L, beta=None, rt60=None, bands=None, air=None, td=None, seed=None, high_pass=False,
        max_order=-1):
    from audiotools_b200.core.room import image_source_ir

    return image_source_ir(room, src, mics, fs, L, beta=beta, rt60=rt60, bands=bands, air_absorption=air,
                           high_pass=high_pass, diffuse_after=td, seed=seed, max_order=max_order,
                           device=DEV).audio_data


def band_walls(rng, kind, K):
    """beta [6, K]: 'per' a different value per wall and band, 'zero' / 'one' everywhere, 'mixed' some bands 0 or 1."""
    if kind == "per":
        return rng.uniform(0.3, 0.97, (6, K))
    if kind in ("zero", "one"):
        return np.full((6, K), 0.0 if kind == "zero" else 1.0)
    b = rng.uniform(0.3, 0.97, (6, K))
    b[:, ::3] = 1.0
    if K > 1:
        b[2, 1] = 0.0
    return b


def crossover_taps(eng, fs, kept):
    """The library's crossover taps as correlation taps, float64 [K' - 1, 2 half0 + 1]."""
    g, half = eng.octave_crossovers(fs, kept, torch.device(DEV))
    assert half == R64.half0(fs)
    return torch.flip(g, dims=[1]).cpu().double().numpy()


# --------------------------------------------------------------------------- checks
def check_unchanged(eng, rates=(8000, 16000, 44100, 48000, 96000), L=1500, C=2):
    rng = np.random.default_rng(5)
    rooms = np.array([ROOMS[1], ROOMS[4], ROOMS[0]])
    for fs in rates:
        geo = [scene(rng, r, "random", C) for r in rooms]
        src, mics = np.stack([g[0] for g in geo]), np.stack([g[1] for g in geo])
        beta = np.stack([walls(rng, "per") for _ in rooms])
        td, seed = np.array([0.01, 0.03, 0.002]), [3, 4, 5]
        for tail in (False, True):
            kw = dict(td=td, seed=seed) if tail else {}
            flat = rir(rooms, src, mics, fs, L, beta, **kw)
            flat_hp = rir(rooms, src, mics, fs, L, beta, high_pass=True, **kw)
            for K in (1, 3, 8):
                bb = np.repeat(beta[:, :, None], K, axis=2)
                assert torch.equal(rir(rooms, src, mics, fs, L, bb, bands=K, **kw), flat), (fs, tail, K)
                assert torch.equal(rir(rooms, src, mics, fs, L, bb, bands=K, air=np.zeros(K), high_pass=True, **kw),
                                   flat_hp), (fs, tail, K)
            # K = 1 with its own beta is the flat call with that beta, air 0 included
            other = np.stack([walls(rng, "per") for _ in rooms])
            assert torch.equal(rir(rooms, src, mics, fs, L, other[:, :, None], bands=1, air=[0.0], **kw),
                               rir(rooms, src, mics, fs, L, other, **kw)), (fs, tail)


def check_bands(eng, fs, L, K=8, C=2, kinds=("per", "mixed", "zero", "one", "per"), air_on=True, td=None,
                max_order=-1, seed=0):
    """One batch of rooms with per-item bands against the oracle, per sample.  Returns the worst error / bound."""
    rng = np.random.default_rng(seed)
    rooms = np.array([ROOMS[i % len(ROOMS)] for i in range(len(kinds))])
    geo = [scene(rng, r, ("corner", "near", "random")[i % 3], C) for i, r in enumerate(rooms)]
    src, mics = np.stack([g[0] for g in geo]), np.stack([g[1] for g in geo])
    beta = np.stack([band_walls(rng, k, K) for k in kinds])
    air = rng.uniform(0.0, 0.3, (len(kinds), K)) if air_on else None
    if air is not None:
        air[0] = 0.0
    tds = None if td is None else np.full(len(kinds), td)
    seeds = None if td is None else rng.integers(0, 2 ** 62, len(kinds))
    y = rir(rooms, src, mics, fs, L, beta, bands=K, air=air, td=tds, seed=seeds,
            max_order=max_order).cpu().double().numpy()
    kept = R64.kept(K, fs)
    taps = crossover_taps(eng, fs, kept) if kept > 1 else np.zeros((0, 1))
    worst = 0.0
    for b in range(len(kinds)):
        for c in range(C):
            r, w = [], []
            for k in range(kept):
                a = 0.0 if air is None else air[b, k]
                rk, G, t, sc = R64.band(rooms[b], src[b], mics[b, c], beta[b, :, k], a, fs, L, max_order,
                                        None if td is None else td, None if td is None else int(seeds[b]), c)
                r.append(rk)
                w.append(K_BUDGET * rir64.U * G + ENV_REL * np.abs(t) + rir64.U * (4 * sc + 2 * np.abs(rk)))
            r, w = np.array(r), np.array(w)
            y64 = R64.combine(r, taps)
            terms = np.abs(r[-1]) + sum(np.abs(R64.conv_centred(r[k] - r[k + 1], taps[k])) for k in range(kept - 1))
            tol = R64.spread(w, taps) + kept * rir64.U * terms  # the sum's rounding
            if kept > 1:  # the crossovers' FFT error, per 1024-sample block, from the float32 differences they filter
                diff = (r[:-1] - r[1:]).astype(np.float32)
                for k in range(kept - 1):
                    _, scale = T64.fftconv64(diff[k][None], np.ascontiguousarray(taps[k][None, ::-1]), 1,
                                             offset0=R64.half0(fs), pad_mode="constant")
                    fb = T64.fft_budget("fftconv", taps.shape[1]) * scale[0]
                    tol += np.repeat(fb, T64.FFT_BLOCK)[:L] + rir64.U * R64.conv_centred(np.abs(diff[k]),
                                                                                        np.abs(taps[k]))
            err = np.abs(y[b, c] - y64)
            assert (err <= tol).all(), (fs, L, b, c, int(np.argmax(err - tol)), float((err / tol).max()))
            z = R64.first_zero_end(src[b], mics[b, c], fs, None if td is None else td)
            assert (y[b, c, :max(0, math.ceil(z))] == 0).all(), (fs, b, c)
            worst = max(worst, float((err / np.maximum(tol, 1e-300)).max()))
    WORST[fs] = max(WORST.get(fs, 0.0), worst)
    return worst


def check_nyquist(eng, fs=8000, L=1200):
    """At 8 kHz bands 6 and 7 (lower crossovers 5.7 and 11.3 kHz) are dropped: K = 8 equals K = 6."""
    assert R64.kept(8, fs) == 6 and eng.rir_bands_kept(8, fs) == 6
    rng = np.random.default_rng(8)
    room, src, mics = ROOMS[1], *scene(rng, ROOMS[1], "random", 2)
    beta = rng.uniform(0.3, 0.95, (6, 8))
    air = rng.uniform(0, 0.2, 8)
    for kw in ({}, dict(td=0.02, seed=7)):
        y8 = rir(room, src, mics, fs, L, beta, bands=8, air=air, high_pass=True, **kw)
        y6 = rir(room, src, mics, fs, L, beta[:, :6], bands=6, air=air[:6], high_pass=True, **kw)
        assert torch.equal(y8, y6)


def band_levels(y, fs, centres):
    """|Y(f)| in dB at the given frequencies (zero-padded DFT)."""
    n = 1 << (len(y) * 4 - 1).bit_length()
    Y = np.abs(np.fft.rfft(y, n))
    f = np.fft.rfftfreq(n, 1 / fs)
    return 20 * np.log10(np.interp(centres, f, Y))


def check_air(eng, fs=48000, L=4096):
    """Anechoic (beta = 0): y_air(f_k) / y(f_k) = 10^(-a_k d / 20) at every band's centre, within the leakage of the
    neighbouring bands through the crossovers' transition (the computed bands only)."""
    room, src, mic = [30.0, 20.0, 10.0], [5.0, 5.0, 5.0], [12.0, 6.0, 5.5]
    d = float(np.linalg.norm(np.subtract(src, mic)))
    air = 0.4 * np.arange(8)
    y0 = rir(room, src, [mic], fs, L, np.zeros((6, 8)), bands=8)[0, 0].cpu().double().numpy()
    y1 = rir(room, src, [mic], fs, L, np.zeros((6, 8)), bands=8, air=air)[0, 0].cpu().double().numpy()
    kept = R64.kept(8, fs)
    centres = 125.0 * 2.0 ** np.arange(kept)
    got = band_levels(y1, fs, centres) - band_levels(y0, fs, centres)
    want = -air[:kept] * d
    assert np.abs(got - want).max() <= 0.5, (got, want)
    return float(np.abs(got - want).max())


def schroeder_t20(y, fs):
    edc = np.cumsum((y ** 2)[::-1])[::-1]
    db = 10 * np.log10(np.maximum(edc / edc[0], 1e-300))
    sel = (db <= -5) & (db >= -25)
    slope = np.polyfit(np.flatnonzero(sel) / fs, db[sel], 1)[0]
    return -60.0 / slope


def octave(y, fs, k):
    """Band k of y [..., T] through a 4th-order Butterworth band-pass between the crossovers e_{k-1} and e_k (a
    brick-wall FFT mask would spread the direct sound's ringing over the whole response)."""
    import scipy.signal as ss

    sos = ss.butter(4, [R64.crossover(k - 1), R64.crossover(k)], btype="bandpass", fs=fs, output="sos")
    return ss.sosfilt(sos, y, axis=-1)


def check_decay(eng, fs=16000, L=14400, M=4, report=None):
    """Per-band Sabine RT60s falling with frequency: the hybrid response's per-octave T20 falls with them and agrees
    with the images-only response's within T20_REL (a target set from data: H100 and simulator runs)."""
    room, src, mic = [6.0, 5.0, 3.0], [1.0, 1.0, 1.5], [4.0, 3.0, 1.2]
    rt = np.array([0.8, 0.6, 0.4, 0.25])
    rng = np.random.default_rng(2)
    mics = np.clip(np.asarray(mic) + rng.uniform(-0.3, 0.3, (M, 3)), 0.2, np.asarray(room) - 0.2)[:, None]
    K = len(rt)
    hyb = rir(room, src, mics, fs, L, rt60=rt, bands=K, td=0.05, seed=np.arange(M), high_pass=True)
    ism = rir(room, src, mics, fs, L, rt60=rt, bands=K, high_pass=True)
    hyb, ism = hyb[:, 0].cpu().double().numpy(), ism[:, 0].cpu().double().numpy()
    t_h = np.array([np.mean([schroeder_t20(octave(v, fs, k), fs) for v in hyb]) for k in range(1, K)])
    t_i = np.array([np.mean([schroeder_t20(octave(v, fs, k), fs) for v in ism]) for k in range(1, K)])
    if report is not None:
        report.append((rt[1:], t_h, t_i))
    assert np.all(np.diff(t_h) < 0) and np.all(np.diff(t_i) < 0), (t_h, t_i)
    assert np.all(np.abs(t_h / t_i - 1) <= T20_REL), (t_h, t_i)


# the hybrid's per-octave T20 against the images-only one: measured 21 % (250 Hz octave, H100, 16 kHz) and 13 %
# (simulator, 8 kHz); the tail's envelope decays somewhat faster than the images' low octaves
T20_REL = 0.3


def check_api(eng, fs=8000):
    from audiotools_b200 import AudioSignal
    from audiotools_b200.core import room as R
    from audiotools_b200.data import transforms as tfm

    lib = eng.lib
    rng = np.random.default_rng(4)
    room, src, mics = [4.0, 3.0, 2.5], [1.0, 1.0, 1.0], [[2.0, 2.0, 1.5], [2.5, 2.0, 1.5]]
    b3 = rng.uniform(0.3, 0.9, (6, 3))
    # reruns, and a batch against its items, bit for bit
    kw = dict(beta=b3, bands=3, air_absorption=[0.0, 0.05, 0.2], diffuse_after=0.02, seed=5, device=DEV)
    a = R.image_source_ir(room, src, mics, fs, 900, **kw).audio_data
    assert torch.equal(a, R.image_source_ir(room, src, mics, fs, 900, **kw).audio_data)
    Bn, C, K = 4, 3, 5
    rooms = np.stack([ROOMS[i % len(ROOMS)] for i in range(Bn)])
    srcs = np.stack([rng.uniform(0.05, r - 0.05) for r in rooms])
    mm = np.stack([rng.uniform(0.05, r - 0.05, (C, 3)) for r in rooms])
    betas = rng.uniform(0.2, 1.0, (Bn, 6, K))
    air = rng.uniform(0.0, 0.3, (Bn, K))
    td = rng.uniform(0.002, 0.1, Bn)
    seeds = rng.integers(0, 2 ** 63 - 1, Bn)
    for tail in (False, True):
        t = dict(diffuse_after=td, seed=seeds) if tail else {}
        y = R.image_source_ir(rooms, srcs, mm, fs, 1500, beta=betas, bands=K, air_absorption=air, device=DEV,
                              **t).audio_data
        for b in range(Bn):
            tb = dict(diffuse_after=td[b], seed=int(seeds[b])) if tail else {}
            one = R.image_source_ir(rooms[b], srcs[b], mm[b], fs, 1500, beta=betas[b], bands=K, air_absorption=air[b],
                                    device=DEV, **tb).audio_data
            assert torch.equal(y[b:b + 1], one), (tail, b)
    # rt60 per band is Sabine's beta per band
    rt = np.array([0.5, 0.4, 0.3])
    want = np.swapaxes(R.sabine_beta(np.asarray(room)[None], rt[None]), 1, 2)[0]
    assert torch.equal(R.image_source_ir(room, src, mics, fs, 700, rt60=rt, bands=3, device=DEV).audio_data,
                       R.image_source_ir(room, src, mics, fs, 700, beta=want, bands=3, device=DEV).audio_data)
    # refusals launch nothing
    k0 = lib.kernel_launches.value
    ok = dict(beta=np.full((6, 3), 0.5), bands=3, device=DEV)
    bad = [(dict(ok, bands=0), "bands"), (dict(ok, bands=9), "bands"), (dict(ok, bands=2.0), "bands"),
           (dict(ok, bands=True), "bands"),
           (dict(ok, beta=np.full((6, 2), 0.5)), "beta"), (dict(ok, beta=np.full(6, 0.5)), "beta"),
           (dict(ok, beta=np.full((6, 3), 1.5)), "beta"),
           (dict(beta=None, rt60=[0.3, 0.3], bands=3, device=DEV), "rt60"),
           (dict(ok, air_absorption=[0.1, 0.1]), "air_absorption"),
           (dict(ok, air_absorption=[0.1, -0.1, 0.0]), "air_absorption"),
           (dict(ok, air_absorption=[0.1, float("nan"), 0.0]), "air_absorption"),
           (dict(ok, air_absorption=[0.1, float("inf"), 0.0]), "air_absorption"),
           (dict(beta=np.full(6, 0.5), air_absorption=[0.1], device=DEV), "bands"),
           (dict(ok, beta=np.full((3, 6, 3), 0.5)), "batch")]
    for kw, msg in bad:
        with pytest.raises(ValueError, match=msg):
            R.image_source_ir([room, room], src, mics, fs, 800, **kw)
    many = np.tile(np.asarray(mics[:1]), (8192, 1))  # 1 x 8192 x 8 rows
    with pytest.raises(ValueError, match="rows"):
        R.image_source_ir(room, src, many, fs, 100, beta=np.full((6, 8), 0.5), bands=8, device=DEV)
    for name, kw in (("beta", dict(beta=torch.full((6, 3), 0.5, dtype=torch.float64, requires_grad=True))),
                     ("rt60", dict(rt60=torch.full((3,), 0.3, dtype=torch.float64, requires_grad=True))),
                     ("air_absorption", dict(beta=np.full((6, 3), 0.5),
                                             air_absorption=torch.zeros(3, dtype=torch.float64, requires_grad=True)))):
        with pytest.raises(NotImplementedError, match=name):
            R.image_source_ir(room, src, mics, fs, 800, bands=3, device=DEV, **kw)
    z = torch.zeros(1, 3, dtype=torch.float64, device=DEV)
    p = z.data_ptr()
    for args, msg in (((None, p, p, p, None, None, None, 1, 1, 3, 10, fs, 343.0, -1, p, None), b"null pointer"),
                      ((p, p, p, p, None, None, None, 1, 1, 0, 10, fs, 343.0, -1, p, None), b"bands"),
                      ((p, p, p, p, None, None, None, 1, 1, 9, 10, fs, 343.0, -1, p, None), b"bands"),
                      ((p, p, p, p, None, None, None, 300, 100, 3, 10, fs, 343.0, -1, p, None), b"65535"),
                      ((p, p, p, p, None, p, None, 1, 1, 3, 10, fs, 343.0, -1, p, None), b"t_d and seed"),
                      ((p, p, p, p, None, p, p, 1, 1, 3, 10, fs, 343.0, 2, p, None), b"max_order"),
                      ((p, p, p, p, None, None, None, 1, 1, 3, 10, 100.0, 343.0, -1, p, None), b"fs=")):
        assert lib.b2a_rir_f32(*args) == -1 and msg in lib.b2a_last_error(), msg
        assert lib.b2a_last_error().startswith(b"rir:")
    assert lib.b2a_rir_band_sum_f32(p, p, None, 1, 1, 10, fs, 343.0, 5, p, p, 0, p, None) == -1
    assert lib.b2a_rir_band_sum_f32(None, p, None, 1, 1, 10, fs, 343.0, 5, p, p, 1, p, None) == -1
    assert lib.kernel_launches.value == k0
    # the transform: bands=None keeps the draws and keys; bands adds one draw per band after all the others
    T, C = 4000, 2
    x = torch.from_numpy(np.random.default_rng(3).standard_normal((4, C, T)).astype(np.float32)).to(DEV)
    sig = AudioSignal(x.clone(), fs)
    ratios = (("uniform", 0.8, 1.2), ("const", 1.0), ("uniform", 0.3, 0.6))
    for td in (None, ("uniform", 0.02, 0.08)):
        plain = tfm.SyntheticRoomImpulseResponse(rt60=("uniform", 0.05, 0.4), duration=None, diffuse_after=td)
        t = tfm.SyntheticRoomImpulseResponse(rt60=("uniform", 0.05, 0.4), duration=None, diffuse_after=td, bands=3,
                                             band_rt60=ratios, air_absorption=[0.0, 0.01, 0.05])
        assert "band_rt60" not in plain.keys and "band_rt60" in t.keys
        kp = plain.batch_instantiate(list(range(4)), sig)[plain.name]
        kw = t.batch_instantiate(list(range(4)), sig)[t.name]
        assert "band_rt60" not in kp
        for k in kp:
            if k != "mask":
                assert torch.equal(kw[k], kp[k]), k
        for i in range(4):
            st = np.random.RandomState(i)
            dims = np.array([st.uniform(3.0, 10.0), st.uniform(3.0, 8.0), st.uniform(2.4, 4.0)])
            rt60 = st.uniform(0.05, 0.4)
            st.uniform(np.full(3, 0.5), dims - 0.5), st.uniform(0.05, 0.2), st.uniform(0.0, 2 * np.pi)
            st.uniform(np.full(3, 0.5), np.full(3, 2.0))
            if td is not None:
                st.uniform(0.02, 0.08), st.randint(0, 2 ** 31 - 1)
            rt60 = max(rt60, 1.01 * float(R.min_rt60(dims)))
            assert float(kw["rt60"][i]) == rt60
            lo = 1.01 * float(R.min_rt60(dims))
            want = [max(st.uniform(0.8, 1.2) * rt60, lo), max(1.0 * rt60, lo), max(st.uniform(0.3, 0.6) * rt60, lo)]
            assert np.array_equal(kw["band_rt60"][i].cpu().numpy(), np.array(want)), i
        y = t(AudioSignal(x.clone(), fs), **t.batch_instantiate(list(range(4)), sig)).audio_data
        L = min(T, int(np.ceil(float(kw["band_rt60"].max()) * fs)))
        extra = {} if td is None else dict(diffuse_after=kw["diffuse_after"], seed=kw["seed"])
        ir = R.image_source_ir(kw["room"], kw["source"], kw["mics"], fs, L, rt60=kw["band_rt60"], bands=3,
                               air_absorption=[0.0, 0.01, 0.05], device=DEV, **extra)
        assert torch.equal(y, AudioSignal(x.clone(), fs).apply_ir(ir).audio_data)
    for bad_kw in (dict(bands=9), dict(bands=2, band_rt60=(("const", 1.0),)), dict(bands=2, air_absorption=[0.1]),
                   dict(air_absorption=[0.1, 0.1]), dict(band_rt60=(("const", 1.0),))):
        with pytest.raises(ValueError):
            tfm.SyntheticRoomImpulseResponse(**bad_kw)


def fftconv_launches(eng, rows, L, taps):
    """Launches of one Engine.fftconv of [rows, L] with these taps (counted on a zero input)."""
    k0 = eng.lib.kernel_launches.value
    eng.fftconv(torch.zeros(rows, L, device=DEV), taps, rows_per_filt=max(1, rows // taps.shape[0]),
                offset0=(taps.shape[1] - 1) // 2, pad_mode="constant")
    return eng.lib.kernel_launches.value - k0


def check_launches(eng, fs=8000):
    """b2a_rir_f32: 1 launch (2 with a tail); K' > 1 adds fftconv's and the sum's 1; the high-pass 3."""
    from audiotools_b200.core.room import image_source_ir

    room, src, mics = [4.0, 3.0, 2.5], [1.0, 1.0, 1.0], [[2.0, 2.0, 1.5], [2.5, 2.0, 1.5]]
    L = 800
    for K, tail, hp in ((1, False, False), (1, True, True), (3, False, False), (3, True, True), (8, True, False)):
        kept = eng.rir_bands_kept(K, fs)
        image_source_ir(room, src, mics, fs, L, beta=np.full((6, K), 0.6), bands=K, device=DEV)  # design the taps
        conv = 0 if kept == 1 else fftconv_launches(eng, (kept - 1) * 2, L, eng.octave_crossovers(fs, kept, DEV)[0])
        want = (2 if tail else 1) + (conv + 1 if kept > 1 else 0) + (3 if hp else 0)
        n0, k0 = eng.launches, eng.lib.kernel_launches.value
        t = dict(diffuse_after=0.01, seed=1) if tail else {}
        image_source_ir(room, src, mics, fs, L, beta=np.full((6, K), 0.6), bands=K, high_pass=hp, device=DEV, **t)
        assert eng.launches - n0 == want and eng.lib.kernel_launches.value - k0 == want, (K, tail, hp, want)


# --------------------------------------------------------------------------- tests
def test_unchanged_path(eng):
    check_unchanged(eng)


def test_crossover_taps_against_float64(eng):
    for fs in (8000, 16000, 44100, 48000, 96000):
        kept = R64.kept(8, fs)
        got = crossover_taps(eng, fs, kept)
        want = R64.lowpass64(fs, kept - 1)
        err = float(np.abs(got - want).max() / np.abs(want).max())
        print(f"rir bands crossover taps at {fs} Hz: max error {err:.3g} of the largest tap")
        assert err <= 64 * rir64.U, (fs, err)


@pytest.mark.parametrize("fs", [8000, 16000, 44100, 48000, 96000])
def test_against_float64(eng, fs):
    h = R64.half0(fs)
    for L in (TILE - 1, TILE + 1, rir64.window(fs) + 3, 2 * h + 5):
        check_bands(eng, fs, L, seed=L)
    check_bands(eng, fs, 3 * TILE + 7, K=3, C=1, kinds=("per", "one"), air_on=False, seed=1)
    check_bands(eng, fs, 2 * TILE, K=8, C=2, kinds=("per", "mixed"), td=0.01, seed=2)


@pytest.mark.parametrize("max_order", [-1, 0, 1, 3, 10])
def test_orders_and_microphones(eng, max_order):
    fs = 16000
    for C in (1, 2, 8):
        check_bands(eng, fs, 1500, K=4, C=C, kinds=("per", "mixed"), max_order=max_order, seed=C)


def test_report_worst_k(eng):
    for fs, w in sorted(WORST.items()):
        print(f"rir bands worst error / bound at {fs} Hz: {w:.3g}")


def test_bands_above_nyquist(eng):
    check_nyquist(eng)


def test_air_absorption(eng):
    print(f"rir bands air absorption: worst band-centre level error {check_air(eng):.3f} dB")


def test_decay_follows_the_bands(eng):
    rows = []
    check_decay(eng, report=rows)
    for rt, t_h, t_i in rows:
        print(f"rir bands Sabine RT60 {rt} s: T20 hybrid {np.round(t_h, 3)} s, images only {np.round(t_i, 3)} s")


def test_api(eng):
    check_api(eng)


def test_no_host_sync(eng):
    from audiotools_b200 import AudioSignal
    from audiotools_b200.core import util
    from audiotools_b200.core.room import image_source_ir
    from audiotools_b200.data import transforms as tfm

    x = 0.5 * torch.randn(4, 2, 16000, device=DEV)
    t = tfm.SyntheticRoomImpulseResponse(diffuse_after=("uniform", 0.03, 0.08), bands=6,
                                         band_rt60=(("uniform", 0.9, 1.1),) * 6, air_absorption=[0.01] * 6)
    sig = AudioSignal(x.clone(), 16000)
    kw = util.prepare_batch(t.batch_instantiate(list(range(4)), sig), DEV)
    sub = kw[t.name]
    t(AudioSignal(x.clone(), 16000), **kw)  # designs the crossovers
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        image_source_ir(sub["room"], sub["source"], sub["mics"], 16000, 4000, rt60=sub["band_rt60"], bands=6,
                        diffuse_after=sub["diffuse_after"], seed=sub["seed"], device=DEV)
        t(sig, **kw)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_launch_counts(eng):
    check_launches(eng)


def test_launches_match_the_profiler(eng):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    from audiotools_b200.core.room import image_source_ir

    args = ([5.0, 4.0, 3.0], [1.0, 1.0, 1.5], [[3.0, 2.5, 1.2]] * 2, 16000, 8000)
    kw = dict(rt60=[0.6, 0.5, 0.4, 0.3, 0.3, 0.2], bands=6, air_absorption=[0.0] * 3 + [0.01] * 3,
              diffuse_after=0.05, seed=3, device=DEV)
    image_source_ir(*args, **kw)
    torch.cuda.synchronize()
    n0, k0 = eng.launches, eng.lib.kernel_launches.value
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        image_source_ir(*args, **kw)
        torch.cuda.synchronize()
    added = eng.launches - n0
    assert eng.lib.kernel_launches.value - k0 == added
    gpu = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    if not gpu:
        pytest.skip("the profiler recorded no GPU activity")
    names = [e.name for e in gpu if "b2a::" in e.name]
    assert len(names) == added, names
    assert sum("b2a::rir" in n for n in names) == 3 and sum("b2a::iir" in n for n in names) == 3, names


def test_more_than_2_31_band_elements(eng):
    """32767 items x 1 microphone x 2 bands x 32800 samples at max_order = 0: 2.15e9 band-row elements; the last item
    equals the item alone, and an item with equal bands equals the flat call."""
    from audiotools_b200.core.room import image_source_ir

    B, L, fs, K = 32767, 32800, 8000, 2
    room = torch.tensor([6.0, 5.0, 4.0], dtype=torch.float64).expand(B, 3).clone()
    src = torch.tensor([1.0, 1.0, 1.0], dtype=torch.float64).expand(B, 3).clone()
    mics = torch.tensor([[5.0, 4.0, 3.0]], dtype=torch.float64).expand(B, 1, 3).clone()
    mics[-1, 0, 0] = 3.0
    beta = np.tile(np.array([0.7, 0.4]), (B, 6, 1))
    beta[0] = 0.7
    y = image_source_ir(room, src, mics, fs, L, beta=beta, bands=K, max_order=0, high_pass=False,
                        device=DEV).audio_data
    assert B * K * L > 2 ** 31
    one = image_source_ir(room[-1], src[-1], mics[-1], fs, L, beta=beta[-1], bands=K, max_order=0, high_pass=False,
                          device=DEV).audio_data
    flat = image_source_ir(room[0], src[0], mics[0], fs, L, beta=np.full(6, 0.7), max_order=0, high_pass=False,
                           device=DEV).audio_data
    assert torch.equal(y[-1], one[0]) and torch.equal(y[1], y[-2]) and torch.equal(y[0], flat[0])
    assert float(y[-1].abs().max()) > 0
    del y
    torch.cuda.empty_cache()
