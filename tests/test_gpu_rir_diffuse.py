"""The diffuse late tail of ``core.room.image_source_ir(..., diffuse_after=, seed=)`` and
``transforms.SyntheticRoomImpulseResponse(diffuse_after=)`` on the H100 (``-m gpu``): csrc/rir.cu's hybrid path
(DESIGN.md K20 "Hybrid") against the float64 oracle of tests/rir_diffuse64.py.

* the images-only path is untouched: ``diffuse_after=None`` is the images-only call, a tail that starts at or after L
  changes nothing, and every 512-sample tile that ends before the tail's first sample n_d - Tw/2 is bit-identical to
  the images-only IR (the tile that straddles it meets K20's per-sample bound);
* per sample against float64: |y - (y64_early + tail64)| <= 8 u G_early + 1e-4 w sqrt(E) |xi| + 4 u sqrt(E) r
  + 2 u |y| (r the Box-Muller radius), at 8 to 96 kHz, with per-item diffuse_after, beta and seeds, with the tail
  starting around tile edges, beta = 1 (a flat envelope) and beta = 0 (no tail);
* physics: for five rooms at 16 kHz the hybrid IR (50 ms) against the full images-only IR, after the 100 Hz
  high-pass, in 10 ms windows after n_d (median energy difference within 1 dB per room) and in 5 ms windows around
  n_d (no dip or bump above 3 dB); the gap before the high-pass and the Schroeder T20 of both are printed;
* the generator over 1e7 samples: mean, variance, kurtosis, and correlations between neighbouring samples, microphones
  and seeds;
* the API: reruns and a batch against its items bit for bit, refusals, launch counts against the profiler, no host
  sync, more than 2^31 outputs, and the transform's seeded draws.
tests/test_sim_rir_diffuse.py runs the same checks at 8 kHz and small sizes on the CPU simulator."""
import math

import numpy as np
import pytest
import torch

from tests import rir64
from tests import rir_diffuse64 as D
from tests.test_gpu_rir import ROOMS, scene, walls

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
K_BUDGET = 8.0   # u, the images' per-sample bound (tests/test_gpu_rir.py)
ENV_REL = 1e-4   # relative error of the tail's amplitude against the converged envelope
TILE = 512       # csrc/rir.cu: samples per CTA
LAUNCHES = 2     # b2a_rir_f32 with a tail: the images, then the tail; the high-pass adds K19's three


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


def rir(room, src, mics, fs, L, beta, td=None, seed=None, high_pass=False):
    from audiotools_b200.core.room import image_source_ir

    return image_source_ir(room, src, mics, fs, L, beta=beta, high_pass=high_pass, diffuse_after=td, seed=seed,
                           device=DEV).audio_data


def tds_at_tile_edges(fs, B):
    """Per-item diffuse_after: tails starting 1 sample before, at and after a tile edge, a short one and a late one."""
    half = rir64.window(fs) // 2
    starts = [TILE - 1, 2 * TILE, 3 * TILE + 1, half // 2, 5 * TILE + 3]
    return np.array([(s + half) / fs for s in starts[:B]])


def check_unchanged(eng, fs=16000, L=3000, C=2):
    from audiotools_b200.core.room import image_source_ir

    rng = np.random.default_rng(11)
    rooms = np.array([ROOMS[1], ROOMS[4], ROOMS[0]])
    geo = [scene(rng, r, "random", C) for r in rooms]
    src, mics = np.stack([g[0] for g in geo]), np.stack([g[1] for g in geo])
    beta = np.stack([walls(rng, "per") for _ in rooms])
    ism = rir(rooms, src, mics, fs, L, beta)
    assert torch.equal(ism, image_source_ir(rooms, src, mics, fs, L, beta=beta, high_pass=False, diffuse_after=None,
                                            device=DEV).audio_data)
    half = rir64.window(fs) // 2
    # a tail that starts at or after L: the images-only IR, bit for bit
    late = (L + half + np.array([0.0, 1.0, 1e4])) / fs
    assert torch.equal(rir(rooms, src, mics, fs, L, beta, late, [1, 2, 3]), ism)
    # tiles that end before the tail's first sample are bit-identical; the straddling tile meets K20's bound
    td = tds_at_tile_edges(fs, 3)
    hyb = rir(rooms, src, mics, fs, L, beta, td, [4, 5, 6])
    for b in range(len(rooms)):
        start = max(0, D.n_diffuse(td[b], fs) - half)
        t_end = (start // TILE) * TILE
        assert torch.equal(hyb[b, :, :t_end], ism[b, :, :t_end]), b
        for c in range(C):
            y64, G = D.early(rooms[b], src[b], mics[b, c], beta[b], fs, L, td[b])
            got = hyb[b, c, t_end:start].cpu().double().numpy()
            assert (np.abs(got - y64[t_end:start]) <= K_BUDGET * rir64.U * G[t_end:start]).all(), (b, c)


def check_tail(eng, fs, L, C=2, seed=0):
    """One batch with per-item geometry, beta, diffuse_after and seeds against the oracle, per sample."""
    rng = np.random.default_rng(seed)
    kinds, betas = ["corner", "near", "random", "random", "near"], ["per", "one", "zero", "per", "per"]
    rooms = np.array(ROOMS)
    geo = [scene(rng, r, k, C) for r, k in zip(rooms, kinds)]
    src, mics = np.stack([g[0] for g in geo]), np.stack([g[1] for g in geo])
    beta = np.stack([walls(rng, b) for b in betas])
    td = tds_at_tile_edges(fs, len(rooms))
    seeds = rng.integers(0, 2 ** 62, len(rooms))
    y = rir(rooms, src, mics, fs, L, beta, td, seeds).cpu().double().numpy()
    worst = 0.0
    for b in range(len(rooms)):
        for c in range(C):
            e64, G = D.early(rooms[b], src[b], mics[b, c], beta[b], fs, L, td[b])
            t64, scale = D.tail(rooms[b], beta[b], fs, L, td[b], int(seeds[b]), c)
            got = y[b, c]
            err = np.abs(got - (e64 + t64))
            tol = K_BUDGET * rir64.U * G + ENV_REL * np.abs(t64) + rir64.U * (4 * scale + 2 * np.abs(got))
            assert (err <= tol).all(), (fs, b, c, int(np.argmax(err - tol)))
            if betas[b] == "zero":
                assert (t64 == 0).all()
            elif D.n_diffuse(td[b], fs) - rir64.window(fs) // 2 < L:
                assert np.abs(t64).max() > 0
            live = np.abs(t64) > 0
            if live.any():
                worst = max(worst, float((np.abs(got - e64 - t64)[live] / np.abs(t64)[live]).max()))
    return worst


def energy_windows(y, start, win):
    n = (y.shape[-1] - start) // win
    return (y[..., start:start + n * win] ** 2).reshape(*y.shape[:-1], n, win).sum(-1)


def schroeder_t20(y, fs):
    """T20 (s) of the Schroeder integral of y [T] (-5 to -25 dB, a least-squares line)."""
    edc = np.cumsum((y ** 2)[::-1])[::-1]
    db = 10 * np.log10(np.maximum(edc / edc[0], 1e-300))
    sel = (db <= -5) & (db >= -25)
    t = np.flatnonzero(sel) / fs
    slope = np.polyfit(t, db[sel], 1)[0]
    return -60.0 / slope


PHYSICS_ROOMS = [  # (room, source, microphone, beta or rt60)
    ([5.0, 4.0, 3.0], [1.0, 1.0, 1.5], [3.0, 2.5, 1.2], 0.5),
    ([6.0, 5.0, 3.0], [1.0, 1.0, 1.5], [4.0, 3.0, 1.2], 0.5),
    ([9.0, 3.0, 2.5], [2.0, 1.0, 1.2], [6.5, 2.0, 1.5], 0.5),
    ([4.0, 3.0, 2.5], [1.0, 1.0, 1.2], [3.0, 2.0, 1.5], 0.5),
    ([6.0, 5.0, 3.0], [1.0, 1.0, 1.5], [4.0, 3.0, 1.2], [0.95, 0.95, 0.9, 0.9, 0.6, 0.8]),
]


def check_physics(eng, fs=16000, L=8000, B=8, report=None):
    """Per room: B microphones around the given one, each with its own seed; energies summed over them.  The
    comparison runs after the 100 Hz high-pass: every image of a room with beta > 0 is positive, so before it the
    images-only IR carries a low-frequency (near-DC) part whose energy grows with the image density (about lambda
    times the diffuse part, lambda the images per sample) and which a zero-mean tail does not model; the median of
    that pre-high-pass gap is reported, not bounded."""
    from audiotools_b200.core.room import image_source_ir

    td = 0.05
    n_d = D.n_diffuse(td, fs)
    rng = np.random.default_rng(2)
    for i, (room, src, mic, wall) in enumerate(PHYSICS_ROOMS):
        mics = np.clip(np.asarray(mic) + rng.uniform(-0.3, 0.3, (B, 3)), 0.2, np.asarray(room) - 0.2)[:, None]
        kw = dict(rt60=wall) if np.isscalar(wall) else dict(beta=wall)
        tail = dict(diffuse_after=td, seed=np.arange(B) + 100 * i)
        y = {}
        for hp in (False, True):
            y[hp] = [image_source_ir(room, src, mics, fs, L, high_pass=hp, device=DEV, **kw, **t).audio_data[:, 0]
                     .cpu().double().numpy() for t in ({}, tail)]
        f, h = y[True]
        ef, eh = energy_windows(f, n_d, fs // 100).sum(0), energy_windows(h, n_d, fs // 100).sum(0)
        diff = 10 * np.log10(eh / ef)
        med = float(np.median(diff))
        assert abs(med) <= 1.0, (room, wall, med, diff)
        w5 = fs // 200
        around = slice(n_d - 2 * w5, n_d + 2 * w5)
        bump = 10 * np.log10(energy_windows(h[:, around], 0, w5).sum(0) / energy_windows(f[:, around], 0, w5).sum(0))
        assert np.abs(bump).max() <= 3.0, (room, wall, bump)
        pre = float(np.median(10 * np.log10(energy_windows(y[False][1], n_d, fs // 100).sum(0) /
                                            energy_windows(y[False][0], n_d, fs // 100).sum(0))))
        t20 = [float(np.mean([schroeder_t20(r, fs) for r in v])) for v in (f, h, *y[False])]
        if report is not None:
            report.append((room, wall, med, float(np.abs(bump).max()), pre, t20))


def check_generator(eng, fs=8000, B=10, C=10, L=100_000, skip=64):
    """beta = 1: a flat envelope, so y / sqrt(E) is xi once the ramp is over; B items of one geometry, one seed each."""
    room, src = [4.0, 3.0, 2.5], [1.0, 1.0, 1.0]
    mics = [[3.0, 2.0, 1.5 + 0.05 * c] for c in range(C)]
    y = rir(room, src, mics, fs, L, np.ones(6), 1e-3, np.arange(B) * 7919 + 1).double()
    n0 = D.n_diffuse(1e-3, fs) + rir64.window(fs) // 2
    xi = (y[..., n0 + skip:] / math.sqrt(float(D.envelope(room, np.ones(6), fs, [0])[0]))).cpu().numpy()
    x = xi.reshape(-1)
    N = x.size
    m, v = x.mean(), x.var()
    assert abs(m) < 5 / math.sqrt(N) and abs(v - 1) < 5 * math.sqrt(2 / N), (m, v)
    k = ((x - m) ** 4).mean() / v ** 2
    assert abs(k - 3) < 5 * math.sqrt(24 / N), k
    lim = 5 / math.sqrt(N)
    rho = lambda a, b: float(np.corrcoef(a.reshape(-1), b.reshape(-1))[0, 1])  # noqa: E731
    assert abs(rho(xi[..., 1:], xi[..., :-1])) < lim
    assert abs(rho(xi[:, 1:], xi[:, :-1])) < 5 / math.sqrt(xi[:, 1:].size)
    assert abs(rho(xi[1:], xi[:-1])) < 5 / math.sqrt(xi[1:].size)


def check_api(eng, fs=8000):
    from audiotools_b200 import AudioSignal
    from audiotools_b200.core import room as R
    from audiotools_b200.data import transforms as tfm

    lib = eng.lib
    rng = np.random.default_rng(4)
    room, src, mics = [4.0, 3.0, 2.5], [1.0, 1.0, 1.0], [[2.0, 2.0, 1.5], [2.5, 2.0, 1.5]]
    for hp, n in ((False, LAUNCHES), (True, LAUNCHES + 3)):
        n0, k0 = eng.launches, lib.kernel_launches.value
        R.image_source_ir(room, src, mics, fs, 800, rt60=0.3, high_pass=hp, diffuse_after=0.01, seed=1, device=DEV)
        assert eng.launches - n0 == n and lib.kernel_launches.value - k0 == n
    # the same seed, the same bits; another seed, another tail; a batch equals its items
    a = R.image_source_ir(room, src, mics, fs, 900, rt60=0.3, diffuse_after=0.01, seed=5, device=DEV).audio_data
    assert torch.equal(a, R.image_source_ir(room, src, mics, fs, 900, rt60=0.3, diffuse_after=0.01, seed=5,
                                            device=DEV).audio_data)
    assert not torch.equal(a, R.image_source_ir(room, src, mics, fs, 900, rt60=0.3, diffuse_after=0.01, seed=6,
                                                device=DEV).audio_data)
    Bn, C = 5, 3
    rooms = np.stack([ROOMS[i % len(ROOMS)] for i in range(Bn)])
    srcs = np.stack([rng.uniform(0.05, r - 0.05) for r in rooms])
    mm = np.stack([rng.uniform(0.05, r - 0.05, (C, 3)) for r in rooms])
    betas = rng.uniform(0.2, 1.0, (Bn, 6))
    td = rng.uniform(0.002, 0.1, Bn)
    seeds = rng.integers(0, 2 ** 63 - 1, Bn)
    y = R.image_source_ir(rooms, srcs, mm, fs, 1500, beta=betas, diffuse_after=td, seed=seeds, device=DEV).audio_data
    for b in range(Bn):
        one = R.image_source_ir(rooms[b], srcs[b], mm[b], fs, 1500, beta=betas[b], diffuse_after=td[b],
                                seed=int(seeds[b]), device=DEV).audio_data
        assert torch.equal(y[b:b + 1], one), b
    # a scalar tail time and seed broadcast over the batch
    y1 = R.image_source_ir(rooms, srcs, mm, fs, 600, beta=betas, diffuse_after=0.03, seed=9, device=DEV).audio_data
    y2 = R.image_source_ir(rooms, srcs, mm, fs, 600, beta=betas, diffuse_after=np.full(Bn, 0.03),
                           seed=np.full(Bn, 9), device=DEV).audio_data
    assert torch.equal(y1, y2)
    # refusals launch nothing
    k0 = lib.kernel_launches.value
    ok = dict(beta=np.full(6, 0.5), device=DEV)
    bad = [(dict(ok, diffuse_after=0.0, seed=1), "diffuse_after"),
           (dict(ok, diffuse_after=-0.1, seed=1), "diffuse_after"),
           (dict(ok, diffuse_after=float("nan"), seed=1), "diffuse_after"),
           (dict(ok, diffuse_after=float("inf"), seed=1), "diffuse_after"),
           (dict(ok, diffuse_after=0.05), "seed"),
           (dict(ok, seed=3), "seed"),
           (dict(ok, diffuse_after=0.05, seed=-1), "seed"),
           (dict(ok, diffuse_after=0.05, seed=1.5), "seed"),
           (dict(ok, diffuse_after=0.05, seed=1, max_order=3), "max_order"),
           (dict(ok, diffuse_after=0.05, seed=1, max_order=0), "max_order"),
           (dict(ok, diffuse_after=[0.05, 0.05, 0.05], seed=1), "batch"),
           (dict(ok, diffuse_after=0.05, seed=[1, 2, 3]), "batch")]
    for kw, msg in bad:
        with pytest.raises(ValueError, match=msg):
            R.image_source_ir([room, room], src, mics, fs, 800, **kw)
    with pytest.raises(NotImplementedError, match="diffuse_after"):
        R.image_source_ir(room, src, mics, fs, 800, beta=np.full(6, 0.5), seed=1, device=DEV,
                          diffuse_after=torch.tensor(0.05, dtype=torch.float64, requires_grad=True))
    z = torch.zeros(1, 3, dtype=torch.float64, device=DEV)
    with pytest.raises(ValueError, match="max_order"):
        eng.image_source_ir(z, z, z[None], torch.zeros(1, 6, 1, dtype=torch.float64, device=DEV), 10, fs, max_order=2,
                            diffuse_after=z[0, :1], seed=torch.zeros(1, dtype=torch.int64, device=DEV))
    p = z.data_ptr()
    for args, msg in (((None, p, p, p, None, p, p, 1, 1, 1, 10, fs, 343.0, -1, p, None), b"null pointer"),
                      ((p, p, p, p, None, None, p, 1, 1, 1, 10, fs, 343.0, -1, p, None), b"t_d and seed"),
                      ((p, p, p, p, None, p, None, 1, 1, 1, 10, fs, 343.0, -1, p, None), b"t_d and seed"),
                      ((p, p, p, p, None, p, p, 0, 1, 1, 10, fs, 343.0, -1, p, None), b"bad shape"),
                      ((p, p, p, p, None, p, p, 300, 300, 1, 10, fs, 343.0, -1, p, None), b"65535"),
                      ((p, p, p, p, None, p, p, 1, 1, 1, (1 << 30) + 1, fs, 343.0, -1, p, None), b"2^30"),
                      ((p, p, p, p, None, p, p, 1, 1, 1, 10, 100.0, 343.0, -1, p, None), b"fs="),
                      ((p, p, p, p, None, p, p, 1, 1, 1, 10, fs, 0.0, -1, p, None), b"sound speed")):
        assert lib.b2a_rir_f32(*args) == -1 and msg in lib.b2a_last_error(), msg
        assert lib.b2a_last_error().startswith(b"rir:")
    assert lib.kernel_launches.value == k0
    # the transform: with diffuse_after, two draws after the images-only ones
    T, C = 4000, 2
    x = torch.from_numpy(np.random.default_rng(3).standard_normal((4, C, T)).astype(np.float32)).to(DEV)
    sig = AudioSignal(x.clone(), fs)
    for spec in (("uniform", 0.02, 0.08), 0.04):
        t = tfm.SyntheticRoomImpulseResponse(rt60=("uniform", 0.05, 0.4), duration=None, diffuse_after=spec)
        plain = tfm.SyntheticRoomImpulseResponse(rt60=("uniform", 0.05, 0.4), duration=None)
        kw = t.batch_instantiate(list(range(4)), sig)[t.name]
        kp = plain.batch_instantiate(list(range(4)), sig)[plain.name]
        assert "seed" not in kp and "diffuse_after" not in kp
        for k in ("room", "rt60", "source", "mics"):
            assert torch.equal(kw[k], kp[k]), k
        for i in range(4):
            st = np.random.RandomState(i)
            st.uniform(3.0, 10.0), st.uniform(3.0, 8.0), st.uniform(2.4, 4.0), st.uniform(0.05, 0.4)
            st.uniform(np.full(3, 0.5), np.full(3, 2.0)), st.uniform(0.05, 0.2), st.uniform(0.0, 2 * np.pi)
            st.uniform(np.full(3, 0.5), np.full(3, 2.0))
            want_td = st.uniform(0.02, 0.08) if isinstance(spec, tuple) else spec
            assert float(kw["diffuse_after"][i]) == want_td
            assert int(kw["seed"][i]) == st.randint(0, 2 ** 31 - 1)
        y = t(AudioSignal(x.clone(), fs), **t.batch_instantiate(list(range(4)), sig)).audio_data
        L = min(T, int(np.ceil(float(kw["rt60"].max()) * fs)))
        ir = R.image_source_ir(kw["room"], kw["source"], kw["mics"], fs, L, rt60=kw["rt60"],
                               diffuse_after=kw["diffuse_after"], seed=kw["seed"], device=DEV)
        assert torch.equal(y, AudioSignal(x.clone(), fs).apply_ir(ir).audio_data)


# --------------------------------------------------------------------------- tests
def test_unchanged_path(eng):
    check_unchanged(eng)


@pytest.mark.parametrize("fs", [8000, 16000, 44100, 48000, 96000])
def test_against_float64(eng, fs):
    worst = check_tail(eng, fs, L=min(6 * TILE + int(0.02 * fs), 8000), seed=fs)
    print(f"rir tail worst relative error at {fs} Hz: {worst:.3g}")


def test_physics(eng):
    rows = []
    check_physics(eng, report=rows)
    for room, wall, med, bump, pre, t20 in rows:
        print(f"rir hybrid {room} {wall}: median window dB {med:+.2f}, worst 5 ms window around n_d {bump:.2f} dB, "
              f"before the high-pass {pre:+.2f} dB; T20 images {t20[0]:.3f} s, hybrid {t20[1]:.3f} s (before the "
              f"high-pass {t20[2]:.3f} / {t20[3]:.3f} s)")


def test_generator(eng):
    check_generator(eng)


def test_api(eng):
    check_api(eng)


def test_more_than_2_31_elements(eng):
    """65535 rows x 32800 samples with a tail from 10 ms: 2.15e9 outputs; the last row equals the item alone."""
    from audiotools_b200.core.room import image_source_ir

    B, L, fs = 65535, 32800, 8000
    room = torch.tensor([6.0, 5.0, 4.0], dtype=torch.float64).expand(B, 3).clone()
    src = torch.tensor([1.0, 1.0, 1.0], dtype=torch.float64).expand(B, 3).clone()
    mics = torch.tensor([[5.0, 4.0, 3.0]], dtype=torch.float64).expand(B, 1, 3).clone()
    mics[-1, 0, 0] = 3.0
    seed = np.zeros(B, dtype=np.int64)
    seed[-1] = 77
    y = image_source_ir(room, src, mics, fs, L, beta=np.full(6, 0.7), diffuse_after=0.01, seed=seed, high_pass=False,
                        device=DEV).audio_data
    assert B * L > 2 ** 31
    one = image_source_ir(room[-1], src[-1], mics[-1], fs, L, beta=np.full(6, 0.7), diffuse_after=0.01, seed=77,
                          high_pass=False, device=DEV).audio_data
    assert torch.equal(y[-1], one[0]) and torch.equal(y[0], y[-2])
    assert float(y[-1, 0, -100:].abs().max()) > 0
    del y
    torch.cuda.empty_cache()


def test_no_host_sync(eng):
    from audiotools_b200 import AudioSignal
    from audiotools_b200.core import util
    from audiotools_b200.core.room import image_source_ir
    from audiotools_b200.data import transforms as tfm

    x = 0.5 * torch.randn(4, 2, 16000, device=DEV)
    t = tfm.SyntheticRoomImpulseResponse(diffuse_after=("uniform", 0.03, 0.08))
    sig = AudioSignal(x.clone(), 16000)
    kw = util.prepare_batch(t.batch_instantiate(list(range(4)), sig), DEV)
    sub = kw[t.name]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        image_source_ir(sub["room"], sub["source"], sub["mics"], 16000, 4000, rt60=sub["rt60"],
                        diffuse_after=sub["diffuse_after"], seed=sub["seed"], device=DEV)
        t(sig, **kw)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_launches_match_the_profiler(eng):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    from audiotools_b200.core.room import image_source_ir

    args = ([5.0, 4.0, 3.0], [1.0, 1.0, 1.5], [[3.0, 2.5, 1.2]] * 2, 16000, 8000)
    kw = dict(rt60=0.5, diffuse_after=0.05, seed=3, device=DEV)
    image_source_ir(*args, **kw)
    torch.cuda.synchronize()
    n0, k0 = eng.launches, eng.lib.kernel_launches.value
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        image_source_ir(*args, **kw)
        torch.cuda.synchronize()
    added = eng.launches - n0
    assert eng.lib.kernel_launches.value - k0 == added == LAUNCHES + 3
    gpu = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    if not gpu:
        pytest.skip("the profiler recorded no GPU activity")
    names = [e.name for e in gpu]
    assert sum("b2a::rir" in n for n in names) == LAUNCHES and sum("b2a::iir" in n for n in names) == 3, names
