"""Microphone and source directivity of ``core.room.image_source_ir(..., mic_pattern=, mic_orientation=,
source_pattern=, source_orientation=)`` and ``transforms.SyntheticRoomImpulseResponse(mic_pattern=, source_pattern=)``
on the H100 (``-m gpu``): csrc/rir.cu's directional kernels (DESIGN.md K20 "Directivity") against the float64 oracle of
tests/rir_dir64.py.

* per sample against float64: |y - y64| <= 8 u G, G rir64's bound with |g D_m D_s|, at 8 to 96 kHz, every named
  pattern and an arbitrary p, random orientations per item and per microphone, max_order -1, 0 and 2, and octave bands
  with and without air (the bound of tests/test_gpu_rir_bands.py);
* the hybrid: the bound of tests/test_gpu_rir_diffuse.py with the oracle's weighted envelope;
* bit identity: no directivity, omni at both ends and p = 1 with any orientation are the plain call; so is the
  directional kernel given p = 1 tables; equal bands without air are ``bands=None``;
* reciprocity: the source and a single microphone swapped with their patterns and orientations, with and without a
  tail; a free field: a cardioid is the omni response times (1 + cos theta) / 2, a figure-eight turned perpendicular
  to the source is silent to 1e-12;
* physics: the hybrid against the images-only response after the high-pass with a cardioid microphone and a
  hypercardioid source, median 10 ms-window difference within 1 dB;
* the API: launches (directivity adds none; the profiler agrees), refusals, the transform's draws and its moving source,
  a batch against its items.
tests/test_sim_rir_directivity.py runs the same checks at 8 kHz and small sizes on the CPU simulator."""
import math

import numpy as np
import pytest
import torch

from tests import rir64
from tests import rir_bands64 as R64
from tests import rir_diffuse64 as D
from tests import rir_dir64 as R
from tests import timedomain64 as T64
from tests.test_gpu_rir import ROOMS, scene, walls

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
K_BUDGET = 8.0   # u, the images' per-sample bound (tests/test_gpu_rir.py)
ENV_REL = 1e-4   # the tail's amplitude against the converged envelope (tests/test_gpu_rir_diffuse.py)
NAMES = ["omni", "subcardioid", "cardioid", "supercardioid", "hypercardioid", "figure8"]


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


def rir(room, src, mics, fs, L, high_pass=False, **kw):
    from audiotools_b200.core.room import image_source_ir

    return image_source_ir(room, src, mics, fs, L, high_pass=high_pass, device=DEV, **kw).audio_data


def unit(rng, *shape):
    v = rng.standard_normal(shape + (3,))
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def p_of(x) -> float:
    from audiotools_b200.core.room import PATTERNS

    return PATTERNS[x] if isinstance(x, str) else float(x)


def patterns(rng, B, C):
    """Per-microphone p [B, C] and per-item source p [B]: every name and 0.37 appear."""
    pool = [p_of(n) for n in NAMES] + [0.37]
    mp = np.array([[pool[(b * C + c) % len(pool)] for c in range(C)] for b in range(B)])
    sp = np.array([pool[(3 * b + 2) % len(pool)] for b in range(B)])
    return mp, sp


def batch(rng, C, kinds=("corner", "near", "random", "random", "near"), rooms=ROOMS):
    rooms = np.asarray(rooms, np.float64)
    geo = [scene(rng, r, k, C) for r, k in zip(rooms, kinds)]
    return rooms, np.stack([g[0] for g in geo]), np.stack([g[1] for g in geo])


# --------------------------------------------------------------------------- checks
def check_accuracy(eng, fs, L, C=2, max_order=-1, seed=0):
    """One batch with per-item geometry, per-microphone patterns and orientations against the oracle, per sample."""
    rng = np.random.default_rng(seed)
    rooms, src, mics = batch(rng, C)
    beta = np.stack([walls(rng, b) for b in ["per", "one", "zero", "per", "per"]])
    B = len(rooms)
    mp, sp = patterns(rng, B, C)
    mo, so = unit(rng, B, C), unit(rng, B)
    y = rir(rooms, src, mics, fs, L, beta=beta, max_order=max_order, mic_pattern=mp, mic_orientation=mo,
            source_pattern=sp, source_orientation=so).cpu().double().numpy()
    worst = 0.0
    for b in range(B):
        for c in range(C):
            y64, G = R.ir(rooms[b], src[b], mics[b, c], beta[b], fs, L, (mp[b, c], mo[b, c]), (sp[b], so[b]),
                          max_order)
            got = y[b, c]
            assert (got[G == 0] == 0).all(), (fs, L, b, c)
            live = G > 0
            k = float((np.abs(got - y64)[live] / G[live]).max() / rir64.U) if live.any() else 0.0
            assert k <= K_BUDGET, (fs, L, b, c, max_order, k)
            worst = max(worst, k)
    return worst


def check_bands(eng, fs, L, K=4, C=2, air_on=True, seed=0):
    """Octave bands with per-band walls (and air) and directivity against the oracle, the bound of
    tests/test_gpu_rir_bands.py."""
    from tests.test_gpu_rir_bands import band_walls, crossover_taps

    rng = np.random.default_rng(seed)
    rooms, src, mics = batch(rng, C, kinds=("near", "random", "corner"), rooms=ROOMS[1:4])
    B = len(rooms)
    beta = np.stack([band_walls(rng, k, K) for k in ("per", "mixed", "per")])
    air = rng.uniform(0.0, 0.3, (B, K)) if air_on else None
    mp, sp = patterns(rng, B, C)
    mo, so = unit(rng, B, C), unit(rng, B)
    y = rir(rooms, src, mics, fs, L, beta=beta, bands=K, air_absorption=air, mic_pattern=mp, mic_orientation=mo,
            source_pattern=sp, source_orientation=so).cpu().double().numpy()
    kept = R64.kept(K, fs)
    taps = crossover_taps(eng, fs, kept) if kept > 1 else np.zeros((0, 1))
    for b in range(B):
        for c in range(C):
            r, w = [], []
            for k in range(kept):
                rk, G, _, _ = R.band(rooms[b], src[b], mics[b, c], beta[b, :, k], 0.0 if air is None else air[b, k],
                                     fs, L, (mp[b, c], mo[b, c]), (sp[b], so[b]))
                r.append(rk)
                w.append(K_BUDGET * rir64.U * G + rir64.U * 2 * np.abs(rk))
            r, w = np.array(r), np.array(w)
            y64 = R64.combine(r, taps)
            terms = np.abs(r[-1]) + sum(np.abs(R64.conv_centred(r[k] - r[k + 1], taps[k])) for k in range(kept - 1))
            tol = R64.spread(w, taps) + kept * rir64.U * terms
            if kept > 1:
                diff = (r[:-1] - r[1:]).astype(np.float32)
                for k in range(kept - 1):
                    _, scale = T64.fftconv64(diff[k][None], np.ascontiguousarray(taps[k][None, ::-1]), 1,
                                             offset0=R64.half0(fs), pad_mode="constant")
                    fb = T64.fft_budget("fftconv", taps.shape[1]) * scale[0]
                    tol += np.repeat(fb, T64.FFT_BLOCK)[:L] + rir64.U * R64.conv_centred(np.abs(diff[k]),
                                                                                        np.abs(taps[k]))
            err = np.abs(y[b, c] - y64)
            assert (err <= tol).all(), (fs, L, K, b, c, int(np.argmax(err - tol)))


def hybrid_tol(G, t, sc, got):
    return K_BUDGET * rir64.U * G + ENV_REL * np.abs(t) + rir64.U * (4 * sc + 2 * np.abs(got))


def check_hybrid(eng, fs, L, C=2, seed=0):
    """Per-item diffuse_after, seeds, patterns and orientations against the images and the weighted envelope."""
    from tests.test_gpu_rir_diffuse import tds_at_tile_edges

    rng = np.random.default_rng(seed)
    rooms, src, mics = batch(rng, C)
    B = len(rooms)
    beta = np.stack([walls(rng, b) for b in ["per", "one", "zero", "per", "per"]])
    td = tds_at_tile_edges(fs, B)
    seeds = rng.integers(0, 2 ** 62, B)
    mp, sp = patterns(rng, B, C)
    mo, so = unit(rng, B, C), unit(rng, B)
    y = rir(rooms, src, mics, fs, L, beta=beta, diffuse_after=td, seed=seeds, mic_pattern=mp, mic_orientation=mo,
            source_pattern=sp, source_orientation=so).cpu().double().numpy()
    for b in range(B):
        for c in range(C):
            r, G, t, sc = R.band(rooms[b], src[b], mics[b, c], beta[b], 0.0, fs, L, (mp[b, c], mo[b, c]),
                                 (sp[b], so[b]), td=td[b], seed=int(seeds[b]), ch=c)
            got = y[b, c]
            err = np.abs(got - r)
            tol = hybrid_tol(G, t, sc, got)
            assert (err <= tol).all(), (fs, b, c, int(np.argmax(err - tol)))


def check_bit_identity(eng, fs, L, C=2):
    from audiotools_b200.core.room import image_source_ir

    rng = np.random.default_rng(7)
    rooms, src, mics = batch(rng, C, kinds=("random", "near", "corner"), rooms=ROOMS[:3])
    B = len(rooms)
    beta = np.stack([walls(rng, "per") for _ in range(B)])
    mo, so = unit(rng, B, C), unit(rng, B)
    for tail in ({}, dict(diffuse_after=np.array([0.01, 0.03, 0.002]), seed=[3, 4, 5])):
        plain = rir(rooms, src, mics, fs, L, beta=beta, **tail)
        none = dict(mic_pattern=None, mic_orientation=None, source_pattern=None, source_orientation=None)
        assert torch.equal(rir(rooms, src, mics, fs, L, beta=beta, **none, **tail), plain)
        assert torch.equal(rir(rooms, src, mics, fs, L, beta=beta, mic_pattern="omni", mic_orientation=mo,
                               source_pattern="omni", source_orientation=so, **tail), plain)
        assert torch.equal(rir(rooms, src, mics, fs, L, beta=beta, mic_pattern=np.ones((B, C)), mic_orientation=mo,
                               source_pattern=np.ones(B), source_orientation=so, **tail), plain)
        assert torch.equal(rir(rooms, src, mics, fs, L, beta=beta, mic_pattern=1.0, source_pattern="omni", **tail),
                           plain)
        # the directional kernels themselves, given p = 1 tables: the factor is exactly 1
        dev = torch.device(DEV)
        t64 = lambda a: torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device=dev)  # noqa: E731
        md = t64(np.concatenate([np.ones((B, C, 1)), mo], axis=-1))
        sd = t64(np.concatenate([np.ones((B, 1)), so], axis=-1))
        kw = {}
        if tail:
            kw = dict(diffuse_after=t64(tail["diffuse_after"]),
                      seed=torch.as_tensor(tail["seed"], dtype=torch.int64, device=dev))
        geo = (t64(rooms), t64(src), t64(mics), t64(beta[:, :, None]))
        for m_, s_ in ((md, sd), (md, None), (None, sd)):
            assert torch.equal(eng.image_source_ir(*geo, L, fs, high_pass=False, mic_dir=m_, src_dir=s_, **kw),
                               plain), (bool(tail), m_ is None, s_ is None)
        # equal bands without air are bands=None, with directivity too
        dkw = dict(mic_pattern="cardioid", mic_orientation=mo, source_pattern=0.3, source_orientation=so, **tail)
        flat = rir(rooms, src, mics, fs, L, beta=beta, **dkw)
        assert not torch.equal(flat, plain)
        for K in (1, 3):
            bb = np.repeat(beta[:, :, None], K, axis=2)
            assert torch.equal(image_source_ir(rooms, src, mics, fs, L, beta=bb, bands=K, high_pass=False,
                                               device=DEV, **dkw).audio_data, flat), K


def check_reciprocity(eng, fs, L):
    """Source and a single microphone swapped with their patterns and orientations: within the per-sample bound of
    the original's oracle, images only and with a tail."""
    rng = np.random.default_rng(12)
    for i, (room, kind) in enumerate(zip(ROOMS, ("corner", "near", "random", "random", "near"))):
        src, mics = scene(rng, room, kind, 1)
        mic = mics[0]
        beta = walls(rng, "per")
        pm, ps = [(0.5, 0.25), (0.0, (math.sqrt(3) - 1) / 2), (0.37, 1.0), (1.0, 0.0), (0.75, 0.5)][i]
        vm, vs = unit(rng), unit(rng)
        for tail in (None, 0.4 * L / fs):
            kw = {} if tail is None else dict(diffuse_after=tail, seed=5 + i)
            fwd = rir(room, src, [mic], fs, L, beta=beta, mic_pattern=pm, mic_orientation=vm, source_pattern=ps,
                      source_orientation=vs, **kw)[0, 0].cpu().double().numpy()
            rev = rir(room, mic, [src], fs, L, beta=beta, mic_pattern=ps, mic_orientation=vs, source_pattern=pm,
                      source_orientation=vm, **kw)[0, 0].cpu().double().numpy()
            r, G, t, sc = R.band(room, src, mic, beta, 0.0, fs, L, (pm, vm), (ps, vs), td=tail,
                                 seed=None if tail is None else 5 + i)
            for got in (fwd, rev):
                tol = hybrid_tol(G, t, sc, got)
                assert (np.abs(got - r) <= tol).all(), (i, tail)


def check_free_field(eng, fs=16000, L=1024):
    """beta = 0: only the direct path.  A cardioid at either end scales it by (1 + cos theta) / 2; a figure-eight
    microphone perpendicular to the source leaves less than 1e-12 of the omni peak."""
    room, src, mic = [5.0, 4.0, 3.0], np.array([1.3, 1.1, 1.7]), np.array([3.1, 2.4, 1.2])
    kw = dict(beta=np.zeros(6))
    omni = rir(room, src, [mic], fs, L, **kw)[0, 0].cpu().double().numpy()
    u = (src - mic) / np.linalg.norm(src - mic)  # the direction the sound arrives from at the microphone
    rng = np.random.default_rng(1)
    for v in (u, -u, unit(rng), unit(rng)):
        cm = rir(room, src, [mic], fs, L, mic_pattern="cardioid", mic_orientation=v, **kw)[0, 0].cpu().double()
        cs = rir(room, src, [mic], fs, L, source_pattern="cardioid", source_orientation=v, **kw)[0, 0].cpu().double()
        for got, f in ((cm.numpy(), 0.5 + 0.5 * float(u @ v)), (cs.numpy(), 0.5 - 0.5 * float(u @ v))):
            want = f * omni  # the factor's own rounding in double: 1e-15 of the peak
            assert (np.abs(got - want) <= 4 * rir64.U * np.abs(want) + 1e-15 * np.abs(omni).max()).all(), (v, f)
    perp = np.cross(u, [0.3, -0.5, 0.8])
    f8 = rir(room, src, [mic], fs, L, mic_pattern="figure8", mic_orientation=perp, **kw)[0, 0].cpu().double()
    assert float(f8.abs().max()) < 1e-12 * float(np.abs(omni).max())


def check_physics(eng, fs=16000, L=8000, B=8, rooms=None, report=None):
    """Hybrid against images-only after the high-pass, cardioid microphones and a hypercardioid source with random
    orientations: median 10 ms-window energy difference after n_d within 1 dB per room."""
    from tests.test_gpu_rir_diffuse import PHYSICS_ROOMS, energy_windows

    td = 0.05
    n_d = D.n_diffuse(td, fs)
    rng = np.random.default_rng(3)
    for i, (room, src, mic, wall) in enumerate(PHYSICS_ROOMS if rooms is None else rooms):
        mics = np.clip(np.asarray(mic) + rng.uniform(-0.3, 0.3, (B, 3)), 0.2, np.asarray(room) - 0.2)[:, None]
        kw = dict(rt60=wall) if np.isscalar(wall) else dict(beta=wall)
        dkw = dict(mic_pattern="cardioid", mic_orientation=unit(rng, B, 1), source_pattern="hypercardioid",
                   source_orientation=unit(rng))
        tail = dict(diffuse_after=td, seed=np.arange(B) + 100 * i)
        f, h = (rir(room, src, mics, fs, L, high_pass=True, **kw, **dkw, **t)[:, 0].cpu().double().numpy()
                for t in ({}, tail))
        ef, eh = energy_windows(f, n_d, fs // 100).sum(0), energy_windows(h, n_d, fs // 100).sum(0)
        med = float(np.median(10 * np.log10(eh / ef)))
        assert abs(med) <= 1.0, (room, wall, med)
        if report is not None:
            report.append((room, wall, med))


def check_launches(eng, fs=8000):
    """Directivity adds no launch: images 1, with a tail 2 (the high-pass adds 3); bands add the crossovers' and the
    sum's launches either way."""
    room, src, mics = [4.0, 3.0, 2.5], [1.0, 1.0, 1.0], [[2.0, 2.0, 1.5], [2.5, 2.0, 1.5]]
    dkw = dict(mic_pattern="cardioid", mic_orientation=[1.0, 0.0, 0.0], source_pattern=0.25,
               source_orientation=[0.0, 1.0, 0.0])
    lib = eng.lib
    counts = {}
    for name, kw, want in (("flat", dict(rt60=0.3), 1), ("hp", dict(rt60=0.3, high_pass=True), 4),
                           ("tail", dict(rt60=0.3, diffuse_after=0.01, seed=1), 2),
                           ("bands", dict(rt60=[0.3, 0.4, 0.5], bands=3), None)):
        for d in ({}, dkw):
            n0, k0 = eng.launches, lib.kernel_launches.value
            rir(room, src, mics, fs, 800, **kw, **d)
            n = eng.launches - n0
            assert lib.kernel_launches.value - k0 == n
            counts.setdefault(name, set()).add(n)
        assert len(counts[name]) == 1, (name, counts[name])
        if want is not None:
            assert counts[name] == {want}, (name, counts[name])
    return counts


def check_errors(eng, fs=8000):
    from audiotools_b200.core.room import image_source_ir

    lib = eng.lib
    room, src, mics = [4.0, 3.0, 2.5], [1.0, 1.0, 1.0], [[2.0, 2.0, 1.5], [2.5, 2.0, 1.5]]
    v = [1.0, 0.0, 0.0]
    k0 = lib.kernel_launches.value
    bad = [(dict(mic_pattern="cardioid", mic_orientation=[0.0, 0.0, 0.0]), "non-zero"),
           (dict(mic_pattern="cardioid", mic_orientation=[float("nan"), 1.0, 0.0]), "finite"),
           (dict(source_pattern="cardioid", source_orientation=[float("inf"), 1.0, 0.0]), "finite"),
           (dict(mic_pattern=1.5, mic_orientation=v), r"\[0, 1\]"),
           (dict(mic_pattern=-0.1, mic_orientation=v), r"\[0, 1\]"),
           (dict(source_pattern=float("nan"), source_orientation=v), r"\[0, 1\]"),
           (dict(mic_pattern="shotgun", mic_orientation=v), "shotgun"),
           (dict(source_pattern="Cardioid", source_orientation=v), "Cardioid"),
           (dict(mic_pattern="cardioid"), "needs a mic_orientation"),
           (dict(source_pattern=[1.0, 0.5], source_orientation=None), "needs a source_orientation"),
           (dict(mic_orientation=v), "without a mic_pattern"),
           (dict(source_orientation=v), "without a source_pattern"),
           (dict(mic_pattern="cardioid", mic_orientation=[1.0, 0.0]), "3 coordinates"),
           (dict(mic_pattern=[0.5, 0.5, 0.5], mic_orientation=v), "microphones"),
           (dict(mic_pattern="cardioid", mic_orientation=[v, v, v]), "microphones"),
           (dict(mic_pattern=np.full((3, 2), 0.5), mic_orientation=v), "batch"),
           (dict(mic_pattern="cardioid", mic_orientation=np.ones((3, 2, 3))), "batch"),
           (dict(source_pattern=[0.5, 0.5, 0.5], source_orientation=v), "batch"),
           (dict(source_pattern="cardioid", source_orientation=[v, v, v]), "batch")]
    for kw, msg in bad:
        with pytest.raises(ValueError, match=msg):
            image_source_ir([room, room], src, mics, fs, 400, rt60=0.3, device=DEV, **kw)
    for kw in (dict(mic_pattern=torch.tensor(0.5, dtype=torch.float64, requires_grad=True), mic_orientation=v),
               dict(mic_pattern=0.5, mic_orientation=torch.tensor(v, dtype=torch.float64, requires_grad=True)),
               dict(source_pattern=torch.tensor(0.5, dtype=torch.float64, requires_grad=True), source_orientation=v),
               dict(source_pattern=0.5, source_orientation=torch.tensor(v, dtype=torch.float64, requires_grad=True))):
        with pytest.raises(NotImplementedError, match="pattern|orientation"):
            image_source_ir(room, src, mics, fs, 400, rt60=0.3, device=DEV, **kw)
    z = torch.zeros(1, 3, dtype=torch.float64, device=DEV)
    beta = torch.full((1, 6, 1), 0.5, dtype=torch.float64, device=DEV)
    with pytest.raises(ValueError, match="mic_dir"):
        eng.image_source_ir(z + 1, z + 1, z[None] + 2, beta, 10, fs, mic_dir=torch.zeros(1, 1, 3, dtype=torch.float64,
                                                                                         device=DEV))
    with pytest.raises(ValueError, match="src_dir"):
        eng.image_source_ir(z + 1, z + 1, z[None] + 2, beta, 10, fs, src_dir=torch.zeros(2, 4, dtype=torch.float64,
                                                                                         device=DEV))
    assert lib.kernel_launches.value == k0
    # the transform refuses a bad pattern when it is made
    from audiotools_b200.data import transforms as tfm

    for kw in (dict(mic_pattern="shotgun"), dict(source_pattern=1.2), dict(mic_pattern=[0.5, 0.5])):
        with pytest.raises(ValueError, match="pattern"):
            tfm.SyntheticRoomImpulseResponse(**kw)


def _replay(i):
    """The state after the draws of the default transform without options for item i."""
    st = np.random.RandomState(i)
    st.uniform(3.0, 10.0), st.uniform(3.0, 8.0), st.uniform(2.4, 4.0), st.uniform(0.2, 0.8)
    st.uniform(np.full(3, 0.5), np.full(3, 2.0)), st.uniform(0.05, 0.2), st.uniform(0.0, 2 * np.pi)
    st.uniform(np.full(3, 0.5), np.full(3, 2.0))
    return st


def check_transform(eng, fs=8000, T=4000, C=2, B=4):
    from audiotools_b200 import AudioSignal
    from audiotools_b200.core import room as Rm
    from audiotools_b200.data import transforms as tfm

    x = torch.from_numpy(np.random.default_rng(3).standard_normal((B, C, T)).astype(np.float32)).to(DEV)
    sig = AudioSignal(x.clone(), fs)
    idx = list(range(B))
    plain = tfm.SyntheticRoomImpulseResponse(duration=0.1)
    kp = plain.batch_instantiate(idx, sig)[plain.name]
    assert list(kp) == ["room", "rt60", "source", "mics", "mask"], list(kp)
    # without the options nothing new is drawn: the same values as a transform that has never heard of directivity
    for opt in (dict(mic_pattern=None), dict(source_pattern=None), {}):
        t = tfm.SyntheticRoomImpulseResponse(duration=0.1, **opt)
        k2 = t.batch_instantiate(idx, sig)[t.name]
        assert list(k2) == list(kp) and all(torch.equal(k2[k], kp[k]) for k in kp)
    for opts in (dict(mic_pattern="cardioid", source_pattern="hypercardioid"), dict(mic_pattern=0.3),
                 dict(source_pattern="figure8", source_yaw=("const", 0.0))):
        t = tfm.SyntheticRoomImpulseResponse(duration=0.1, **opts)
        kw = t.batch_instantiate(idx, sig)[t.name]
        new = [k for k in ("mic_orientation", "source_orientation") if opts.get(k.split("_")[0] + "_pattern")]
        assert list(kw) == ["room", "rt60", "source", "mics"] + new + ["mask"], list(kw)
        for k in ("room", "rt60", "source", "mics"):
            assert torch.equal(kw[k], kp[k]), k
        for i in idx:  # the draws after all the old ones: the azimuth, then the yaw
            st = _replay(i)
            if "mic_orientation" in new:
                az = st.uniform(0.0, 2 * np.pi)
                assert np.array_equal(kw["mic_orientation"][i].numpy(), [np.cos(az), np.sin(az), 0.0])
            if "source_orientation" in new:
                yaw = st.uniform(-0.5 * np.pi, 0.5 * np.pi) if "source_yaw" not in opts else 0.0
                to = kw["mics"][i].numpy().mean(0) - kw["source"][i].numpy()
                a = np.arctan2(to[1], to[0]) + yaw
                assert np.array_equal(kw["source_orientation"][i].numpy(), [np.cos(a), np.sin(a), 0.0])
        y = t(AudioSignal(x.clone(), fs), **t.batch_instantiate(idx, sig)).audio_data
        L = int(np.ceil(0.1 * fs))
        mo = kw.get("mic_orientation")
        ir = Rm.image_source_ir(kw["room"], kw["source"], kw["mics"], fs, L, rt60=kw["rt60"],
                                mic_pattern=opts.get("mic_pattern"),
                                mic_orientation=None if mo is None else mo[:, None].expand(B, C, 3),
                                source_pattern=opts.get("source_pattern"),
                                source_orientation=kw.get("source_orientation"), device=DEV)
        assert torch.equal(y, AudioSignal(x.clone(), fs).apply_ir(ir).audio_data)
        # a batch equals its items one at a time
        for i in idx:
            one = {t.name: {k: v[i:i + 1] for k, v in kw.items()}}
            yi = t(AudioSignal(x[i:i + 1].clone(), fs), **one).audio_data
            assert torch.equal(yi, y[i:i + 1]), i
    # a moving source keeps its orientation at every waypoint
    t = tfm.SyntheticRoomImpulseResponse(duration=0.1, mic_pattern="cardioid", source_pattern=0.4,
                                         source_speed=("uniform", 0.5, 2.0), diffuse_after=0.02)
    kw = t.batch_instantiate(idx, sig)[t.name]
    assert list(kw)[-3:] == ["mic_orientation", "source_orientation", "mask"]
    y = t(AudioSignal(x.clone(), fs), **t.batch_instantiate(idx, sig)).audio_data
    from audiotools_b200.engine import Engine

    hop = max(Engine.MOVING_IR_MIN_HOP, int(round(0.05 * fs)))
    K = (T - 1) // hop + 1
    path = t.path(kw["source"], kw["end"], kw["speed"], K, hop / fs)
    L = int(np.ceil(0.1 * fs))
    irs = torch.stack([torch.cat([Rm.image_source_ir(kw["room"][b], path[b, k], kw["mics"][b], fs, L, rt60=kw["rt60"][b],
                                                     diffuse_after=kw["diffuse_after"][b], seed=int(kw["seed"][b]),
                                                     mic_pattern="cardioid",
                                                     mic_orientation=kw["mic_orientation"][b],
                                                     source_pattern=0.4,
                                                     source_orientation=kw["source_orientation"][b],
                                                     device=DEV).audio_data for k in range(K)]) for b in idx])
    want = AudioSignal(x.clone(), fs).apply_moving_ir(irs, hop).audio_data
    assert torch.equal(y, want)


# --------------------------------------------------------------------------- tests
@pytest.mark.parametrize("fs", [8000, 16000, 44100, 48000, 96000])
def test_against_float64(eng, fs):
    L = 3 * 512 + rir64.window(fs)
    worst = max(check_accuracy(eng, fs, L, max_order=mo, seed=fs + mo) for mo in (-1, 0, 2))
    print(f"rir directivity worst K at {fs} Hz: {worst:.3g} u")


@pytest.mark.parametrize("air_on", [False, True])
def test_bands_against_float64(eng, air_on):
    check_bands(eng, 16000, 2500, K=5, air_on=air_on)
    check_bands(eng, 48000, 3000, K=8, air_on=air_on, seed=1)


@pytest.mark.parametrize("fs", [8000, 16000, 48000])
def test_hybrid_against_float64(eng, fs):
    check_hybrid(eng, fs, min(6 * 512 + int(0.02 * fs), 6000), seed=fs)


@pytest.mark.parametrize("fs", [8000, 44100, 96000])
def test_bit_identity(eng, fs):
    check_bit_identity(eng, fs, 1500)


def test_reciprocity(eng):
    check_reciprocity(eng, 16000, 2000)


def test_free_field(eng):
    check_free_field(eng)


def test_physics(eng):
    rows = []
    check_physics(eng, report=rows)
    for room, wall, med in rows:
        print(f"rir directivity hybrid {room} {wall}: median window dB {med:+.2f}")


def test_launches(eng):
    check_launches(eng)


def test_launches_match_the_profiler(eng):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    args = ([5.0, 4.0, 3.0], [1.0, 1.0, 1.5], [[3.0, 2.5, 1.2]] * 2, 16000, 8000)
    kw = dict(rt60=0.5, diffuse_after=0.05, seed=3, high_pass=True, mic_pattern="cardioid",
              mic_orientation=[1.0, 1.0, 0.0], source_pattern="hypercardioid", source_orientation=[0.0, 1.0, 1.0])
    rir(*args, **kw)
    torch.cuda.synchronize()
    n0 = eng.launches
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        rir(*args, **kw)
        torch.cuda.synchronize()
    assert eng.launches - n0 == 5
    gpu = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    if not gpu:
        pytest.skip("the profiler recorded no GPU activity")
    names = [e.name for e in gpu]
    assert sum("b2a::rir::ism_dir_kernel" in n for n in names) == 1, names
    assert sum("b2a::rir::tail_dir_kernel" in n for n in names) == 1, names
    assert sum("b2a::iir" in n for n in names) == 3, names


def test_no_host_sync(eng):
    from audiotools_b200 import AudioSignal
    from audiotools_b200.core import util
    from audiotools_b200.data import transforms as tfm

    x = 0.5 * torch.randn(4, 2, 16000, device=DEV)
    t = tfm.SyntheticRoomImpulseResponse(diffuse_after=0.05, mic_pattern="cardioid", source_pattern=0.25)
    sig = AudioSignal(x.clone(), 16000)
    kw = util.prepare_batch(t.batch_instantiate(list(range(4)), sig), DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        t(sig, **kw)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_errors(eng):
    check_errors(eng)


def test_transform(eng):
    check_transform(eng)
