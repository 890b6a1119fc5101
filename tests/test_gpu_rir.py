"""``core.room.image_source_ir`` / ``Engine.image_source_ir`` / ``transforms.SyntheticRoomImpulseResponse`` on the H100
(``-m gpu``): the image-source kernel of csrc/rir.cu (DESIGN.md K20) against the float64 oracle of tests/rir64.py.

* per sample, before the high-pass: |y - y64| <= K u G[n] (G: the sum of |g| min(1, 1 / (pi |n - d|)) over the
  images reaching sample n), and exactly 0 where no image reaches; 8, 16, 44.1, 48 and 96 kHz; L = 1, below Tw,
  the tile +- 1, Tw/2 +- 1 and 1 s; rooms from 2 x 2 x 2 to 20 x 15 x 5 m and a 30 x 1.5 x 3 m corridor; sources and
  microphones 1 cm from walls and corners, microphones 5 cm from the source; beta = 0, 1 and per wall; max_order
  -1, 0, 1, 2, 10; C = 1, 2, 8; per-item geometry in one batch;
* the high-pass: against float64 sosfilt of the kernel's own output with the float32-rounded section, within twice the
  sequential float32 filter's error or 64 u (tests/iir64.py's budget);
* properties: the direct path in closed form, beta = 0 at every order, reciprocity, the mirrored room, order K minus
  order K - 1, batch == single items and reruns bit for bit;
* the API: refused arguments and gradients, launch counts, no host sync, the profiler, a batch past 2^31 elements,
  the transform's seeded draws, a partial mask, ``Compose`` and ``apply_ir``.
tests/test_sim_rir.py runs the same checks at 8 kHz and small sizes on the CPU simulator."""
import math

import numpy as np
import pytest
import torch

from tests import iir64, rir64

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
K_BUDGET = 8.0   # u, per sample, relative to G[n]; worst measured 4.96 (48 kHz) on an H100 80GB HBM3 at 700 W
TILE = 512       # csrc/rir.cu: samples per CTA
LAUNCHES = 1     # b2a_rir_f32; the high-pass adds K19's three
WORST = {}       # the largest K seen per rate (printed by test_report_worst_k)


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


def ism(room, src, mics, fs, L, beta, max_order=-1, high_pass=False):
    from audiotools_b200.core.room import image_source_ir

    return image_source_ir(room, src, mics, fs, L, beta=beta, max_order=max_order, high_pass=high_pass,
                           device=DEV).audio_data


# --------------------------------------------------------------------------- scenes
ROOMS = ([2.0, 2.0, 2.0], [5.0, 4.0, 3.0], [20.0, 15.0, 5.0], [30.0, 1.5, 3.0], [3.3, 2.7, 2.2])


def scene(rng, room, kind: str, C: int):
    """(src [3], mics [C, 3]) in ``room``: "corner" (1 cm from a corner and a wall), "near" (5 cm from the source)
    or "random"."""
    room = np.asarray(room)
    if kind == "corner":
        src = np.array([0.01, 0.01, 0.01])
        mics = np.stack([np.array([room[0] - 0.01, 0.5 * room[1], room[2] - 0.01 - 0.01 * c]) for c in range(C)])
        return src, mics
    src = rng.uniform(0.1, room - 0.1)
    if kind == "near":
        u = rng.standard_normal((C, 3))
        mics = src + 0.05 * u / np.linalg.norm(u, axis=1, keepdims=True)
        return src, np.clip(mics, 0.005, room - 0.005)
    return src, rng.uniform(0.01, room - 0.01, (C, 3))


def walls(rng, kind: str):
    if kind == "zero":
        return np.zeros(6)
    if kind == "one":
        return np.ones(6)
    return rng.uniform(0.3, 1.0, 6)


def check_accuracy(eng, fs, L, C, rooms, kinds, betas, max_order=-1, seed=0):
    """One batch with per-item geometry against the oracle, per sample; returns the worst K in u."""
    rng = np.random.default_rng(seed)
    geo = [scene(rng, r, k, C) for r, k in zip(rooms, kinds)]
    beta = np.stack([walls(rng, b) for b in betas])
    room = np.asarray(rooms, np.float64)
    src = np.stack([g[0] for g in geo])
    mics = np.stack([g[1] for g in geo])
    y = ism(room, src, mics, fs, L, beta, max_order).cpu().double().numpy()
    worst = 0.0
    for b in range(len(rooms)):
        for c in range(C):
            y64, G, hit, _ = rir64.ir(room[b], src[b], mics[b, c], beta[b], fs, L, max_order)
            got = y[b, c]
            # exactly 0 where no image, or only images of gain 0, reach the sample
            assert (got[(~hit) | (G == 0)] == 0).all(), (fs, L, b, c)
            live = G > 0
            ratio = np.abs(got - y64)[live] / G[live]
            k = float(ratio.max() / rir64.U) if live.any() else 0.0
            assert k <= K_BUDGET, (fs, L, C, b, c, max_order, k, int(np.flatnonzero(live)[np.argmax(ratio)]))
            worst = max(worst, k)
    WORST[fs] = max(WORST.get(fs, 0.0), worst)
    return worst


def lengths(fs):
    """L = 1, below Tw, the tile +- 1, Tw/2 +- 1."""
    Tw = rir64.window(fs)
    return sorted({1, Tw - 3, TILE - 1, TILE, TILE + 1, Tw // 2 - 1, Tw // 2 + 1, 3 * TILE + 7})


def check_rate(eng, fs, C=2, long_s=1.0):
    mixes = [(["corner", "near", "random", "random", "near"], ["per", "one", "zero", "per", "per"])]
    for i, L in enumerate(lengths(fs)):
        kinds, betas = mixes[0]
        check_accuracy(eng, fs, L, C, list(ROOMS), kinds, betas, max_order=(-1, 10, 2)[i % 3], seed=i)
    # a long IR in the large rooms (the image count grows with L^3 / V)
    # (the corridor's 1.3e6 images per second of IR at 8 and 16 kHz only: the oracle's cost grows with the window)
    L = int(long_s * fs)
    check_accuracy(eng, fs, L, C, [ROOMS[2], ROOMS[3] if fs <= 16000 else ROOMS[2]], ["random", "corner"],
                   ["per", "per"], seed=99)


def check_orders_and_channels(eng, fs=16000, L=2000):
    for mo in (-1, 0, 1, 2, 10):
        for C in (1, 2, 8):
            check_accuracy(eng, fs, L, C, [ROOMS[1], ROOMS[4]], ["random", "near"], ["per", "one"], mo, seed=mo + C)


def check_highpass(eng, fs=16000, L=4000):
    from audiotools_b200.core.room import image_source_ir

    rng = np.random.default_rng(5)
    room = np.array([ROOMS[1], ROOMS[4]])
    src = np.stack([rng.uniform(0.5, r - 0.5) for r in room])
    mics = np.stack([rng.uniform(0.5, r - 0.5, (2, 3)) for r in room])
    pre = image_source_ir(room, src, mics, fs, L, rt60=[0.4, 0.7], high_pass=False, device=DEV).audio_data
    hp = image_source_ir(room, src, mics, fs, L, rt60=[0.4, 0.7], device=DEV).audio_data
    x = pre.cpu().numpy()
    s32 = iir64.coefficients(rir64.highpass_sos(fs), 2)
    e_k = iir64.block_error(hp.cpu().numpy(), iir64.reference(x, s32))
    e_b = iir64.block_error(iir64.baseline(x, s32), iir64.reference(x, s32))
    assert (e_k <= np.maximum(2.0 * e_b, 64.0)).all(), (e_k, e_b)


def check_properties(eng, fs=8000, L=1200):
    rng = np.random.default_rng(7)
    room = np.array(ROOMS[1])
    src = np.array([1.2, 0.9, 1.4])
    mic = np.array([[3.1, 2.6, 1.1]])
    beta = rng.uniform(0.4, 0.95, 6)
    # max_order = 0: the direct path in closed form
    dist = float(np.linalg.norm(src - mic[0]))
    d = np.array([dist * fs / 343.0])
    g = np.array([1.0 / (4 * math.pi * dist)])
    Tw = rir64.window(fs)
    direct = ism(room, src, mic, fs, L, beta, 0)[0, 0].cpu().double().numpy()
    G = rir64.bound(d, g, Tw, L)
    assert (np.abs(direct - rir64.render(d, g, Tw, L)) <= K_BUDGET * rir64.U * G).all()
    # beta = 0: the direct path at every order, bit for bit
    for mo in (-1, 1, 2, 10):
        assert np.array_equal(ism(room, src, mic, fs, L, np.zeros(6), mo)[0, 0].cpu().double().numpy(),
                              ism(room, src, mic, fs, L, np.zeros(6), 0)[0, 0].cpu().double().numpy())
    full = ism(room, src, mic, fs, L, beta)[0, 0].cpu().double().numpy()
    _, Gf, _, _ = rir64.ir(room, src, mic[0], beta, fs, L)
    tol = 2 * K_BUDGET * rir64.U * Gf
    # reciprocity: source and microphone swapped
    swapped = ism(room, mic[0], src[None], fs, L, beta)[0, 0].cpu().double().numpy()
    assert (np.abs(swapped - full) <= tol).all()
    # the room mirrored along x, with its x walls swapped
    flip = lambda p: np.array([room[0] - p[0], p[1], p[2]])  # noqa: E731
    bm = beta[[1, 0, 2, 3, 4, 5]]
    mirrored = ism(room, flip(src), flip(mic[0])[None], fs, L, bm)[0, 0].cpu().double().numpy()
    assert (np.abs(mirrored - full) <= tol).all()
    # order K minus order K - 1 equals the order-K images
    d_all, g_all, o_all = rir64.images(room, src, mic[0], beta, fs, L)
    prev = ism(room, src, mic, fs, L, beta, 0)[0, 0].cpu().double().numpy()
    for K in (1, 2, 3):
        cur = ism(room, src, mic, fs, L, beta, K)[0, 0].cpu().double().numpy()
        sel = o_all == K
        want = rir64.render(d_all[sel], g_all[sel], Tw, L)
        Gk = rir64.bound(d_all[o_all <= K], g_all[o_all <= K], Tw, L)
        assert (np.abs((cur - prev) - want) <= 2 * K_BUDGET * rir64.U * Gk).all(), K
        prev = cur
    # a batch == its items one at a time, and reruns, bit for bit
    B, C = 5, 3
    rooms = np.stack([ROOMS[i % len(ROOMS)] for i in range(B)])
    srcs = np.stack([rng.uniform(0.05, r - 0.05) for r in rooms])
    mics = np.stack([rng.uniform(0.05, r - 0.05, (C, 3)) for r in rooms])
    betas = rng.uniform(0.2, 1.0, (B, 6))
    y = ism(rooms, srcs, mics, fs, 1500, betas)
    assert torch.equal(y, ism(rooms, srcs, mics, fs, 1500, betas))
    for b in range(B):
        assert torch.equal(y[b:b + 1], ism(rooms[b], srcs[b], mics[b], fs, 1500, betas[b]))


def check_api(eng, fs=8000):
    from audiotools_b200 import AudioSignal
    from audiotools_b200.core import room as R
    from audiotools_b200.data import transforms as tfm

    lib = eng.lib
    room, src, mics = [4.0, 3.0, 2.5], [1.0, 1.0, 1.0], [[2.0, 2.0, 1.5], [2.5, 2.0, 1.5]]
    # launch counts: one, and K19's three for the high-pass
    for hp, n in ((False, LAUNCHES), (True, LAUNCHES + 3)):
        n0, k0 = eng.launches, lib.kernel_launches.value
        R.image_source_ir(room, src, mics, fs, 800, rt60=0.3, high_pass=hp, device=DEV)
        assert eng.launches - n0 == n and lib.kernel_launches.value - k0 == n
    # Sabine
    b = R.sabine_beta(room, 0.5)
    assert b.shape == (6,) and np.allclose(b, rir64.sabine_beta(room, 0.5), rtol=1e-15)
    assert (R.sabine_beta(room, 0.0) == 0).all()
    lo = float(R.min_rt60(room))
    with pytest.raises(ValueError, match="smallest feasible RT60"):
        R.sabine_beta(room, 0.9 * lo)
    a = R.image_source_ir(room, src, mics, fs, 800, rt60=0.5, device=DEV).audio_data
    b = R.image_source_ir(room, src, mics, fs, 800, beta=b, device=DEV).audio_data
    assert torch.equal(a, b)
    # refusals launch nothing
    k0 = lib.kernel_launches.value
    ok = dict(beta=np.full(6, 0.5), device=DEV)
    bad = [((room, src, mics, fs, 800), dict(beta=np.full(6, 0.5), rt60=0.3), "exactly one"),
           ((room, src, mics, fs, 800), dict(), "exactly one"),
           (([4.0, 0.0, 2.5], src, mics, fs, 800), ok, "positive"),
           (([4.0, -3.0, 2.5], [1.0, -1.0, 1.0], mics, fs, 800), ok, "positive"),
           ((room, [0.0, 1.0, 1.0], mics, fs, 800), ok, "inside"),
           ((room, [4.0, 1.0, 1.0], mics, fs, 800), ok, "inside"),
           ((room, src, [[2.0, 3.0, 1.5]], fs, 800), ok, "inside"),
           ((room, src, [[1.0005, 1.0, 1.0]], fs, 800), ok, "from the source"),
           ((room, src, mics, fs, 0), ok, "length"),
           ((room, src, mics, 124.9, 100), ok, "sample_rate"),
           ((room, src, mics, fs, 800), dict(ok, max_order=-2), "max_order"),
           ((room, src, mics, fs, 800), dict(beta=[0.5, 0.5, 1.01, 0.5, 0.5, 0.5], device=DEV), r"\[0, 1\]"),
           ((room, src, mics, fs, 800), dict(beta=[0.5, 0.5, -0.1, 0.5, 0.5, 0.5], device=DEV), r"\[0, 1\]"),
           ((room, src, mics, fs, 800), dict(rt60=0.5 * lo, device=DEV), "smallest feasible"),
           (([room, room], [src, src, src], mics, fs, 800), ok, "batch")]
    for args, kw, msg in bad:
        with pytest.raises(ValueError, match=msg):
            R.image_source_ir(*args, **kw)
    for name in ("room", "source", "mics", "beta"):
        kw = dict(room=torch.tensor(room), source=torch.tensor(src), mics=torch.tensor(mics),
                  beta=torch.full((6,), 0.5))
        kw[name] = kw[name].double().requires_grad_()
        with pytest.raises(NotImplementedError, match=name):
            R.image_source_ir(kw["room"], kw["source"], kw["mics"], fs, 800, beta=kw["beta"], device=DEV)
    with pytest.raises(NotImplementedError, match="rt60"):
        R.image_source_ir(room, src, mics, fs, 800, rt60=torch.tensor(0.4, requires_grad=True), device=DEV)
    z = torch.zeros(1, 3, dtype=torch.float64, device=DEV)
    with pytest.raises(ValueError, match="rows"):
        eng.image_source_ir(z.expand(70000, 3), z.expand(70000, 3), torch.zeros(70000, 1, 3, dtype=torch.float64,
                            device=DEV), torch.zeros(70000, 6, 1, dtype=torch.float64, device=DEV), 10, fs)
    p = z.data_ptr()
    for args, msg in (((None, p, p, p, None, None, None, 1, 1, 1, 10, fs, 343.0, -1, p, None), b"null pointer"),
                      ((p, p, p, p, None, None, None, 0, 1, 1, 10, fs, 343.0, -1, p, None), b"bad shape"),
                      ((p, p, p, p, None, None, None, 1, 1, 1, 0, fs, 343.0, -1, p, None), b"bad shape"),
                      ((p, p, p, p, None, None, None, 300, 300, 1, 10, fs, 343.0, -1, p, None), b"65535"),
                      ((p, p, p, p, None, None, None, 1, 1, 1, (1 << 30) + 1, fs, 343.0, -1, p, None), b"2^30"),
                      ((p, p, p, p, None, None, None, 1, 1, 1, 10, 100.0, 343.0, -1, p, None), b"fs="),
                      ((p, p, p, p, None, None, None, 1, 1, 1, 10, 400000.0, 343.0, -1, p, None), b"fs="),
                      ((p, p, p, p, None, None, None, 1, 1, 1, 10, fs, 0.0, -1, p, None), b"sound speed"),
                      ((p, p, p, p, None, None, None, 1, 1, 1, 10, fs, 343.0, -2, p, None), b"max_order")):
        assert lib.b2a_rir_f32(*args) == -1 and msg in lib.b2a_last_error(), msg
    assert lib.kernel_launches.value == k0
    # the transform: seeded draws against a numpy restatement of the documented order
    T, C = 4000, 2
    x = torch.from_numpy(np.random.default_rng(3).standard_normal((4, C, T)).astype(np.float32)).to(DEV)
    t = tfm.SyntheticRoomImpulseResponse(rt60=("uniform", 0.05, 0.4), duration=None, prob=0.5)
    comp = tfm.Compose([t])
    sig = AudioSignal(x.clone(), fs)
    kw = comp.batch_instantiate(list(range(4)), sig)
    sub = kw[comp.name][t.name]
    for i in range(4):
        st = np.random.RandomState(i)
        dims = np.array([st.uniform(3.0, 10.0), st.uniform(3.0, 8.0), st.uniform(2.4, 4.0)])
        rt = st.uniform(0.05, 0.4)
        s = st.uniform(np.full(3, 0.5), dims - 0.5)
        sp = st.uniform(0.05, 0.2)
        az = st.uniform(0.0, 2 * np.pi)
        ax = np.array([np.cos(az), np.sin(az), 0.0])
        ext = 0.5 * (C - 1) * sp * np.abs(ax)
        ctr = st.uniform(0.5 + ext, dims - 0.5 - ext)
        rt = max(rt, 1.01 * float(R.min_rt60(dims)))
        assert np.array_equal(sub["room"][i].numpy(), dims) and np.array_equal(sub["source"][i].numpy(), s)
        assert float(sub["rt60"][i]) == rt
        assert np.allclose(sub["mics"][i].numpy(), ctr + (np.arange(C) - 0.5)[:, None] * sp * ax, rtol=0, atol=1e-15)
        assert bool(sub["mask"][i]) == (st.rand() <= 0.5)
    mask = sub["mask"]
    assert 0 < int(mask.sum()) < 4
    y = comp(sig.clone(), **kw).audio_data
    m = mask.to(y.device)
    L = min(T, int(np.ceil(float(sub["rt60"][mask].max()) * fs)))
    ir = R.image_source_ir(sub["room"][mask], sub["source"][mask], sub["mics"][mask], fs, L, rt60=sub["rt60"][mask],
                           device=DEV)
    want = AudioSignal(x[m].clone(), fs).apply_ir(ir).audio_data
    assert torch.equal(y[~m], x[~m])
    assert torch.equal(y[m], want)
    # apply_ir with the result, and the single-item instantiate
    assert torch.isfinite(want).all() and not torch.equal(want, x[m])
    one = t.instantiate(0, sig)[t.name]
    assert one["mics"].shape == (C, 3) and one["room"].shape == (3,)
    with pytest.raises(ValueError, match="too small"):
        tfm.SyntheticRoomImpulseResponse(room=(("const", 0.9), ("const", 3.0), ("const", 3.0))).instantiate(0, sig)
    with pytest.raises(ValueError, match="too small"):
        tfm.SyntheticRoomImpulseResponse(room=(("const", 1.2), ("const", 1.2), ("const", 3.0)),
                                         mic_spacing=("const", 0.5)).instantiate(0, AudioSignal(x[:, :1].repeat(
                                             1, 8, 1), fs))
    t2 = tfm.SyntheticRoomImpulseResponse(duration=0.05)
    y2 = t2(AudioSignal(x.clone(), fs), **t2.batch_instantiate(list(range(4)), sig)).audio_data
    assert y2.shape == x.shape and torch.isfinite(y2).all()


# --------------------------------------------------------------------------- tests
@pytest.mark.parametrize("fs", [8000, 16000, 44100, 48000, 96000])
def test_against_float64(eng, fs):
    check_rate(eng, fs)


def test_orders_and_channels(eng):
    check_orders_and_channels(eng)


def test_high_pass(eng):
    check_highpass(eng)


def test_properties(eng):
    check_properties(eng)


def test_api(eng):
    check_api(eng)


def test_report_worst_k(eng):
    print("rir worst K (u) per rate:", {k: round(v, 3) for k, v in sorted(WORST.items())}, "budget", K_BUDGET)


def test_more_than_2_31_elements(eng):
    """65535 rows x 32800 samples at max_order = 0: 2.15e9 outputs; the last row equals the item alone."""
    from audiotools_b200.core.room import image_source_ir

    B, L, fs = 65535, 32800, 8000
    room = torch.tensor([6.0, 5.0, 4.0], dtype=torch.float64).expand(B, 3).clone()
    src = torch.tensor([1.0, 1.0, 1.0], dtype=torch.float64).expand(B, 3).clone()
    mics = torch.tensor([[5.0, 4.0, 3.0]], dtype=torch.float64).expand(B, 1, 3).clone()
    mics[-1, 0, 0] = 3.0
    y = image_source_ir(room, src, mics, fs, L, beta=np.full(6, 0.7), max_order=0, high_pass=False,
                        device=DEV).audio_data
    assert B * L > 2 ** 31
    one = image_source_ir(room[-1], src[-1], mics[-1], fs, L, beta=np.full(6, 0.7), max_order=0, high_pass=False,
                          device=DEV).audio_data
    assert torch.equal(y[-1], one[0]) and torch.equal(y[0], y[-2])
    del y
    torch.cuda.empty_cache()


def test_no_host_sync(eng):
    from audiotools_b200 import AudioSignal
    from audiotools_b200.core import util
    from audiotools_b200.core.room import image_source_ir
    from audiotools_b200.data import transforms as tfm

    x = 0.5 * torch.randn(4, 2, 16000, device=DEV)
    t = tfm.SyntheticRoomImpulseResponse()
    sig = AudioSignal(x.clone(), 16000)
    kw = util.prepare_batch(t.batch_instantiate(list(range(4)), sig), DEV)
    sub = kw[t.name]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        image_source_ir(sub["room"], sub["source"], sub["mics"], 16000, 4000, rt60=sub["rt60"], device=DEV)
        t(sig, **kw)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_launches_match_the_profiler(eng):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    from audiotools_b200.core.room import image_source_ir

    args = ([5.0, 4.0, 3.0], [1.0, 1.0, 1.5], [[3.0, 2.5, 1.2]] * 2, 16000, 8000)
    image_source_ir(*args, rt60=0.5, device=DEV)
    torch.cuda.synchronize()
    n0, k0 = eng.launches, eng.lib.kernel_launches.value
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        image_source_ir(*args, rt60=0.5, device=DEV)
        torch.cuda.synchronize()
    added = eng.launches - n0
    assert eng.lib.kernel_launches.value - k0 == added == LAUNCHES + 3
    gpu = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    if not gpu:
        pytest.skip("the profiler recorded no GPU activity")
    names = [e.name for e in gpu]
    assert sum("b2a::rir" in n for n in names) == LAUNCHES and sum("b2a::iir" in n for n in names) == 3, names
