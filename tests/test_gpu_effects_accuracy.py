"""The effect kernels of csrc/effects.cu, the MFCC basis product of csrc/dft.cu and the gather of csrc/collate.cu on the
H100 (``-m gpu``), per element against float64 (tests/effects64.py) at the edges of their tiling: order statistics and
quantiles across the 1024-thread stride with ties, signed zeros, denormals, infinities and NaN of either sign;
``alter_drr`` with early regions clipped by the row's ends, tied and NaN maxima, and the reference's NaN rows; mu-law
and linear quantisation at every level boundary on both walks; the peak-scale backward in both modes at ties, the
1e-8 clamp and NaN; the DCT past its 32-coefficient register chunk and at the largest basis; ``pack_rows``' float4 tail,
offsets and strides; refusals through the C ABI, reruns, batch against single items, power-of-two scaling.
tests/probes/effects_accuracy_probe.py prints the table of DESIGN.md "Effect kernel accuracy"."""
import ctypes
import math

import numpy as np
import pytest
import torch

from tests import effects64 as o

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
U = o.U
NAN, INF = float("nan"), float("inf")
INT_MAX = 2 ** 31 - 1
OS_T = [1, 2, 1023, 1024, 1025, 10 ** 6]
DRR_T = [511, 512, 513, 1023, 1024, 1025, 4000]
PS_T = [1, 255, 256, 257, 4097]
MFCC = [1, 13, 31, 32, 33, 64, 65, 128]
MELS = [1, 40, 80, 128, 256]
FRAMES = [1, 127, 128, 129, 300]
Q_LEVELS = [2, 3, 8, 256, 65536]


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


def dev(t):
    return torch.as_tensor(t).to(DEV)


def stream_of(t):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream) if t.is_cuda else None


def rng(seed):
    return np.random.default_rng(seed)


def worst(acc, key, v):
    v = float(v)
    if acc is not None and not math.isnan(v):
        acc[key] = max(acc.get(key, 0.0), v)


def neg_nan():
    return np.frombuffer(np.uint32(0xFFC00000).tobytes(), dtype=np.float32)[0]


# --------------------------------------------------------------------------- order statistics and quantile
def os_rows(T, seed):
    """Rows of T floats that stress the radix passes: all equal, half one value, keys differing in the low byte only,
    and a mix of signed zeros, denormals and infinities; plus a plain random row."""
    r = rng(seed)
    f32 = np.float32
    rows = {"random": r.standard_normal(T).astype(f32), "equal": np.full(T, f32(0.375))}
    half = r.standard_normal(T).astype(f32)
    half[r.permutation(T)[: T // 2]] = f32(-1.25)
    rows["half"] = half
    base = np.frombuffer(np.uint32(0x3F800000).tobytes(), dtype=f32)[0]
    low = (np.uint32(0x3F800000) + r.integers(0, 256, T).astype(np.uint32)).view(f32)  # 1.0 .. 1.0 + 255 ulp
    rows["low_byte"] = np.where(r.random(T) < 0.5, low, -low).astype(f32) if T > 1 else np.array([base], f32)
    special = np.array([0.0, -0.0, 1e-45, -1e-45, 1.17e-38, -3e-39, INF, -INF, 1.0, -1.0], dtype=f32)
    rows["special"] = special[r.integers(0, special.size, T)]
    return rows


def os_ks(T):
    ks = sorted({0, 1, T // 3, T // 2, T - 2, T - 1})
    return [k for k in ks if 0 <= k < T] + [-5, T, T + 7]  # both clamps


def check_order_stats(eng, row, ks=None):
    ks = os_ks(row.size) if ks is None else ks
    got = eng.order_stats(dev(torch.from_numpy(row)), torch.tensor(ks)).cpu().numpy()
    want = o.order_stats(row, ks)
    assert o.same_values(got, want), (row.size, ks, got, want)
    if np.isnan(want).any():  # a NaN statistic is the positive quiet NaN, whatever the sign of the input's NaN
        assert (got[np.isnan(want)].view(np.uint32) == 0x7FFFFFFF).all()
    return got


@pytest.mark.parametrize("T", OS_T)
def test_order_stats_exact(eng, T):
    for name, row in os_rows(T, T).items():
        check_order_stats(eng, row)


def test_order_stats_at_thirty_million(eng):
    r = rng(3)
    row = r.standard_normal(30_000_000).astype(np.float32)
    row[r.integers(0, row.size, 1000)] = np.float32(0.5)  # ties
    ks = [0, 1, 12_345_678, 15_000_000, row.size - 2, row.size - 1]
    got = eng.order_stats(dev(torch.from_numpy(row)), torch.tensor(ks)).cpu().numpy()
    assert o.same_values(got, np.partition(row, ks)[ks].astype(np.float64))


def check_nan_rows(eng, T, where, sign):
    row = rng(T).standard_normal(T).astype(np.float32)
    row[0 if where == "first" else T - 1] = np.float32(NAN) if sign > 0 else neg_nan()
    check_order_stats(eng, row)
    got = eng.quantile(dev(torch.from_numpy(row)), torch.tensor([0.0, 0.25, 0.5, 1.0])).cpu()
    assert got.isnan().all(), got  # torch.quantile: NaN for every q
    assert torch.quantile(torch.from_numpy(row), torch.tensor([0.0, 0.5])).isnan().all()


@pytest.mark.parametrize("T", [1, 2, 1025, 4096])
@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("sign", [1, -1])
def test_order_stats_and_quantile_nan(eng, T, where, sign):
    check_nan_rows(eng, T, where, sign)


def test_order_stats_k_count_limit(eng):
    row = dev(torch.randn(3000))
    ks = torch.arange(65535) % 3000
    got = eng.order_stats(row, ks).cpu().numpy()
    assert o.same_values(got, np.sort(row.cpu().numpy())[ks.numpy()])
    with pytest.raises(RuntimeError):
        eng.order_stats(row, torch.arange(65536) % 3000)


def check_quantile(eng, row, qs, acc=None):
    """Integer ranks bit for bit against torch.quantile on the same device; other ranks within C_Q u (|a| + |b|)."""
    x = dev(torch.from_numpy(row))
    q = torch.tensor(qs, dtype=torch.float32)
    got = eng.quantile(x, q).cpu()
    want, a, b, integer = o.quantile(row, qs)
    if row.size <= 2 ** 24:
        tq = torch.quantile(x, dev(q)).cpu()
        ii = torch.from_numpy(integer)
        assert torch.equal(got[ii].view(torch.int32), tq[ii].view(torch.int32)) or \
            o.same_values(got[ii].numpy(), tq[ii].numpy()), (got, tq)
    g = got.double().numpy()
    assert np.array_equal(np.isnan(g), np.isnan(want))
    fin = ~np.isnan(want)
    err = np.abs(g - want)[fin] / np.maximum(U * (np.abs(a) + np.abs(b))[fin], 1e-300)
    err[np.abs(g - want)[fin] == 0] = 0.0
    worst(acc, "quantile", err.max() if err.size else 0.0)
    assert (err <= o.C_Q).all(), (qs, err.max())


@pytest.mark.parametrize("T", [1, 2, 1023, 1024, 1025, 10 ** 6])
def test_quantile(eng, T):
    n1 = max(T - 1, 1)
    qs = [0.0, 1.0, 0.5, 1.0 / n1, 3.0 / n1 if T > 4 else 0.0, 0.05, 0.95, 0.333]
    for name, row in os_rows(T, T + 1).items():
        if name == "special" and T > 1:
            row = row.copy()
            row[row == INF] = 2.0  # lerp between +-inf is NaN in both; keep the budget finite
            row[row == -INF] = -2.0
        check_quantile(eng, row, qs)


def test_quantile_past_two_to_the_24(eng):
    """torch.quantile refuses rows over 2^24 elements: numpy (same float32 ranks) is the reference."""
    row = rng(5).standard_normal(30_000_000).astype(np.float32)
    check_quantile(eng, row, [0.0, 0.5, 1.0, 0.01, 0.99])


@pytest.mark.parametrize("nan_row", [0, 2])
def test_clip_distortion_nan(eng, nan_row):
    """The reference clamps every item at quantiles of ROW 0: a NaN there makes every threshold, so every sample, NaN;
    a NaN in another row changes nothing but that sample."""
    from audiotools_b200 import AudioSignal

    x = torch.from_numpy(rng(9).standard_normal((3, 1, 4000)).astype(np.float32)) * 0.3
    x[nan_row, 0, 17] = NAN
    q = torch.tensor([0.1, 0.2, 0.05])
    got = AudioSignal(dev(x), 16000).clip_distortion(q).audio_data.cpu()
    lo = torch.quantile(x, q / 2, dim=-1)[:, :1, :]
    hi = torch.quantile(x, 1 - q / 2, dim=-1)[:, :1, :]
    want = x.clamp(lo, hi)
    assert torch.equal(got.isnan(), want.isnan())
    assert torch.equal(got.nan_to_num(), want.nan_to_num())


# --------------------------------------------------------------------------- alter_drr
def check_drr(eng, ir, sr, drr, acc=None, key="alter_drr"):
    ir = torch.as_tensor(ir, dtype=torch.float32)
    drr = torch.as_tensor(drr, dtype=torch.float32).reshape(-1)
    got = eng.alter_drr(dev(ir), sr, dev(drr)).cpu()
    r, mism = o.alter_drr_err(got, ir, sr, drr)
    worst(acc, key, r)
    assert mism == 0, (ir.shape, mism)
    assert r <= o.C_DRR, (ir.shape, r)
    return got


def ir_like(B, C, T, seed, peaks=None):
    """Decaying noise with a direct path per row at ``peaks`` (a sample index per row, default T // 5)."""
    r = rng(seed)
    x = r.standard_normal((B, C, T)) * np.exp(-np.arange(T) / (0.2 * T + 1)) * 0.2
    for bc in range(B * C):
        p = (T // 5) if peaks is None else peaks[bc % len(peaks)]
        x[bc // C, bc % C, p] = 1.0 + 0.1 * bc
    return torch.from_numpy(x.astype(np.float32))


@pytest.mark.parametrize("T", DRR_T)
def test_alter_drr_strides(eng, T):
    check_drr(eng, ir_like(3, 2, T, T, peaks=[T // 3, T // 3 + 7]), 44100, [-5.0, 3.0, 12.0])


@pytest.mark.parametrize("where", ["0", "t0", "T-1-t0", "T-1"])
def test_alter_drr_direct_path_at_row_ends(eng, where):
    sr, T = 44100, 2000
    t0 = int(sr * 0.0025)
    p = {"0": 0, "t0": t0, "T-1-t0": T - 1 - t0, "T-1": T - 1}[where]
    check_drr(eng, ir_like(2, 2, T, 11, peaks=[p, p]), sr, [0.0, 8.0])


def test_alter_drr_t0_zero_and_short_rows(eng):
    check_drr(eng, ir_like(2, 1, 700, 12), 300, [2.0, -2.0])  # t0 = 0 below 400 Hz
    check_drr(eng, ir_like(2, 2, 150, 13, peaks=[70, 75]), 44100, [2.0, 6.0])  # T < 2 t0 + 1


def test_alter_drr_tied_maxima_and_negative_response(eng):
    x = ir_like(2, 1, 3000, 14, peaks=[500])
    x[0, 0, 2500] = x[0, 0, 500]  # tie: the first index is the direct path
    x[1] = -x[1].abs() - 0.01  # all negative
    check_drr(eng, x, 44100, [4.0, 4.0])


def test_alter_drr_second_channel_beyond_t0(eng):
    """Channel 1's direct path lies beyond t0 from channel 0's: its early region misses the window, a = 0, and the
    reference's row is NaN."""
    got = check_drr(eng, ir_like(1, 2, 3000, 15, peaks=[300, 900]), 44100, [3.0])
    assert got[0, 1].isnan().all() and not got[0, 0].isnan().any()


def test_alter_drr_target_edges(eng):
    """c cancelled exactly (channel 1: E_out == L at 0 dB), c > 0 (no real root: NaN row), alpha on the min_alpha
    floor (channel 0 at -20 dB, channel 1 at 0.5 dB).  t0 = 110: channel 0's window is [0, 210], channel 1's early
    region [190, 410]."""
    T, sr = 1000, 44100
    x = torch.zeros(3, 2, T)
    x[:, 0, 100], x[:, 0, 800] = 1.0, 0.75
    x[:, 1, 300] = 1.0           # channel 1's direct path, outside the window
    x[:, 1, 200] = 0.5           # in the window and in channel 1's early region: a = 0.25
    x[:, 1, 350] = 0.5           # early, outside the window: E_out = 1 + 0.25
    x[:, 1, 600], x[:, 1, 700] = 1.0, 0.5  # late: L = 1.25
    drr = torch.tensor([0.0, -20.0, 0.5])
    got = check_drr(eng, x, sr, drr)
    _, info = o.alter_drr(x, sr, drr)
    assert float(info["c"][0, 1]) == 0.0 and not got[0].isnan().any()
    assert float(info["c"][1, 1]) > 0 and got[1, 1].isnan().all() and not got[1, 0].isnan().any()
    assert float(info["raw"][1, 0]) < float(info["min_alpha"][1, 0])
    assert float(info["raw"][2, 1]) < float(info["min_alpha"][2, 1])


@pytest.mark.parametrize("C", [1, 2, 5])
def test_alter_drr_channels(eng, C):
    B = 7
    peaks = [200 + 13 * c for c in range(C)]
    check_drr(eng, ir_like(B, C, 2049, 20 + C, peaks=peaks), 48000, torch.linspace(-10, 15, B))


def test_alter_drr_seventy_thousand_rows(eng):
    check_drr(eng, ir_like(35000, 2, 300, 16, peaks=[40, 45]), 16000, torch.linspace(-6, 12, 35000))


@pytest.mark.parametrize("where", ["window", "early", "late", "channel0"])
def test_alter_drr_nan(eng, where):
    """A NaN is the arg-max of its row (torch.argmax), so its row's alpha, and the whole row, is NaN; a NaN in
    channel 0 also moves the window of the item's other channels."""
    x = ir_like(2, 2, 2000, 17, peaks=[300, 305])
    i = {"window": (0, 0, 302), "early": (0, 1, 305 + 60), "late": (0, 1, 1500), "channel0": (1, 0, 1200)}[where]
    x[i] = NAN
    got = check_drr(eng, x, 44100, [3.0, 3.0])
    assert got[i[0], i[1]].isnan().all()


# --------------------------------------------------------------------------- quantisation
def quant_inputs(q):
    xs = [o.mulaw_boundaries(q), o.linear_boundaries(q),
          np.array([0.0, -0.0, 1e-45, -1e-45, 1e-39, 1.5, -3.0, INF, -INF, NAN, 1.0, -1.0], np.float32)]
    return np.concatenate(xs)


def check_quant(eng, x, q, mulaw, acc=None):
    """GPU: bit for bit against the reference's float32 expressions on the same device.  CPU simulator: host libm
    replaces libdevice, so a mu-law sample may differ by one level where the float64 level lies within 16 u of an
    integer (a few u of the encoded value, which the level scales by mu / 2), or by a few u in the decoded value;
    the level flips are counted."""
    x = torch.as_tensor(x, dtype=torch.float32)
    xd = dev(x)
    got = eng.quantize(xd, torch.as_tensor(q, dtype=torch.float32), mulaw=mulaw).cpu()
    ref = (o.mulaw_ref if mulaw else o.linear_ref)(xd, q).cpu()
    nan_ok = torch.equal(got.isnan(), ref.isnan())
    assert nan_ok
    same = (got == ref) | got.isnan()
    if DEV != "cpu" or not mulaw:
        assert bool(same.all()), (q, mulaw, int((~same).sum()))
        return 0
    z = o.mulaw_level64(x.numpy(), np.asarray(q, dtype=np.float64).reshape(-1))
    mu = np.asarray(q, dtype=np.float64).reshape(-1, 1, 1) - 1
    with np.errstate(invalid="ignore"):
        near = torch.from_numpy(np.abs(z - np.round(z)) <= 16 * U * np.maximum(mu, 1.0))
    close = (got.double() - ref.double()).abs() <= 8 * U * ref.double().abs()
    bad = ~same & ~(close | near)
    assert not bool(bad.any()), (q, x[bad][:5], got[bad][:5], ref[bad][:5])
    flips = int((~same & ~close).sum())
    worst(acc, "mulaw level flips (sim)", flips)
    return flips


@pytest.mark.parametrize("mulaw", [True, False])
@pytest.mark.parametrize("q", Q_LEVELS)
def test_quantize_level_boundaries(eng, q, mulaw):
    x = quant_inputs(q)
    n = x.size - x.size % 4
    check_quant(eng, x[:n].reshape(1, 1, -1), q, mulaw)  # float4 walk
    check_quant(eng, x[: n - 1].reshape(1, 1, -1), q, mulaw)  # scalar walk


@pytest.mark.parametrize("mulaw", [True, False])
def test_quantize_per_item_and_q1(eng, mulaw):
    x = torch.from_numpy(rng(21).uniform(-1.2, 1.2, (4, 2, 1001)).astype(np.float32))
    check_quant(eng, x, [2.0, 17.0, 256.0, 65536.0], mulaw)
    if not mulaw:
        check_quant(eng, x, 1.0, mulaw)
    else:  # q = 1: mu = 0, log1p(0) = 0: 0 / 0 in both
        got = eng.quantize(dev(x), torch.tensor(1.0), mulaw=True).cpu()
        assert torch.equal(got.isnan(), o.mulaw_ref(x, 1.0).isnan())


@pytest.mark.parametrize("mulaw", [True, False])
@pytest.mark.parametrize("n", [4096, 4097, 4098, 4099])
def test_quantize_walks(eng, n, mulaw):
    """Aligned float4 rows (n % 4 == 0) and the scalar walk: lengths 1, 2, 3 mod 4 and views offset by one float."""
    buf = torch.from_numpy(rng(n).uniform(-1.1, 1.1, 3 * n + 1).astype(np.float32))
    check_quant(eng, buf[: 3 * n].reshape(3, 1, n), [256.0, 8.0, 3.0], mulaw)
    check_quant(eng, buf[1: 3 * n + 1].reshape(3, 1, n), [256.0, 8.0, 3.0], mulaw)
    if DEV != "cpu":
        b = dev(buf)
        view = b[1: 3 * n + 1].reshape(3, 1, n)  # misaligned by one float on the device
        got = eng.quantize(view, torch.tensor([256.0, 8.0, 3.0]), mulaw=mulaw).cpu()
        ref = (o.mulaw_ref if mulaw else o.linear_ref)(view, [256.0, 8.0, 3.0]).cpu()
        assert torch.equal(got, ref)


# --------------------------------------------------------------------------- peak-scale backward
def check_ps(eng, g, y, x_ref=None, max_abs=1.0, bypass=None, acc=None, key="peak_scale"):
    g, y = torch.as_tensor(g, dtype=torch.float32), torch.as_tensor(y, dtype=torch.float32)
    xd = None if x_ref is None else dev(torch.as_tensor(x_ref, dtype=torch.float32))
    gy, gx = eng.peak_scale_backward(dev(g), dev(y), xd, max_abs=max_abs, bypass=bypass)
    r, mism = o.peak_scale_err(gy.cpu(), None if gx is None else gx.cpu(), g, y,
                               None if x_ref is None else torch.as_tensor(x_ref, dtype=torch.float32), max_abs,
                               None if bypass is None else torch.as_tensor(bypass))
    worst(acc, key, r)
    assert mism == 0, (y.shape, mism)
    assert r <= o.C_PS, (y.shape, r)
    return gy, gx


def ps_data(rows, T, seed, scale=1.5):
    r = rng(seed)
    return (torch.from_numpy(r.standard_normal((rows, T)).astype(np.float32)),
            torch.from_numpy((r.standard_normal((rows, T)) * scale).astype(np.float32)),
            torch.from_numpy((r.standard_normal((rows, T)) * 0.7).astype(np.float32)))


@pytest.mark.parametrize("T", PS_T)
def test_peak_scale_strides(eng, T):
    g, y, x = ps_data(5, T, T)
    check_ps(eng, g, y)
    check_ps(eng, g, y, max_abs=0.25)
    check_ps(eng, g, y, x)


def test_peak_scale_ties_and_row_ends(eng):
    T = 1000
    g, y, x = ps_data(6, T, 30, scale=0.3)
    y[0, 10], y[0, 700] = 1.5, -1.5   # tie of |y|, opposite signs: the first index
    y[1, 700], y[1, 10] = 1.5, -1.5
    y[2, 0] = -2.0                    # peak at the first sample
    y[3, T - 1] = 2.0                 # ... at the last
    x[4, 5], x[4, 600] = -1.0, 1.0    # tie in x_ref
    y[5, 300], y[5, 301] = 2.0, 2.0   # tie, same sign
    check_ps(eng, g, y)
    check_ps(eng, g, y, x)


def test_peak_scale_limit_edges(eng):
    """My equal to max_abs and one float to either side; My and Mx straddling 1e-8; zero rows."""
    g, y, x = ps_data(9, 300, 31, scale=0.01)
    f = np.float32
    for r, v in enumerate([0.5, np.nextafter(f(0.5), f(1)), np.nextafter(f(0.5), f(0))]):
        y[r] *= 0.1
        y[r, 50] = float(v)
    e8 = f(1e-8)
    for r, v in zip((3, 4, 5), [e8, np.nextafter(e8, f(1)), np.nextafter(e8, f(0))]):
        y[r] = y[r] / y[r].abs().max() * float(v)
        x[r] = x[r] / x[r].abs().max() * float(v)
    y[6] = 0.0
    x[7] = 0.0
    y[8], x[8] = 0.0, 0.0
    check_ps(eng, g, y, max_abs=0.5)
    check_ps(eng, g, y, x)


def test_peak_scale_bypass_and_many_rows(eng):
    g, y, x = ps_data(70000, 3, 32)
    bypass = torch.zeros(70000, dtype=torch.bool)
    bypass[::3] = True
    check_ps(eng, g, y)
    check_ps(eng, g, y, x, bypass=bypass)


@pytest.mark.parametrize("where", [0, 137, 299])
@pytest.mark.parametrize("restore", [False, True])
def test_peak_scale_nan(eng, where, restore):
    """A NaN sample is its row's peak, as in torch.max(dim): limit mode keeps the gain 1 (gradient g), restore mode's
    clamp keeps the NaN (gradient NaN on the whole row)."""
    g, y, x = ps_data(3, 300, 33)
    y[1, where] = NAN
    y[2, where] = -NAN
    gy, gx = check_ps(eng, g, y, x if restore else None)
    gy = gy.cpu()
    if restore:
        assert gy[1:].isnan().all() and not gy[0].isnan().any()
    else:
        assert torch.equal(gy[1:].nan_to_num(), g[1:]) and not gy.isnan().any()
    if restore:  # a NaN in x_ref only: the scale is NaN
        x[0, where] = NAN
        check_ps(eng, g, torch.nan_to_num(y), x)


def test_peak_scale_forward_with_nan(eng):
    """ensure_max_of_audio and apply_ir's restore with a NaN sample: the reference's peak is NaN, so its gain is 1
    (limit) and its scale NaN (restore)."""
    from audiotools_b200 import AudioSignal

    x = torch.from_numpy(rng(34).standard_normal((2, 1, 500)).astype(np.float32)) * 2
    x[1, 0, 77] = NAN
    got = AudioSignal(dev(x), 16000).ensure_max_of_audio().audio_data.cpu()
    peak = x.abs().max(dim=-1, keepdim=True)[0]
    gain = torch.ones_like(peak)
    gain[peak > 1] = 1 / peak[peak > 1]
    assert torch.equal(got.nan_to_num(), (x * gain).nan_to_num()) and torch.equal(got.isnan(), (x * gain).isnan())
    assert torch.equal(eng.row_absmax(dev(x)).cpu().isnan(), peak.isnan())


# --------------------------------------------------------------------------- MFCC DCT
def check_dct(eng, rows, n_mels, n_mfcc, N, seed, acc=None, transposed=False):
    r = rng(seed)
    v = torch.from_numpy((r.standard_normal((rows, 1, n_mels, N)) * 4 - 6).astype(np.float32))
    d = torch.from_numpy(r.standard_normal((n_mfcc, n_mels) if transposed else (n_mels, n_mfcc)).astype(np.float32))
    if transposed:
        d = d.t()  # the backward's basis: dct.t().contiguous() of a [n_mfcc, n_mels] tensor
    got = eng.mel_dct(dev(v), dev(d.contiguous())).cpu()
    e = o.mel_dct_err(got, v, d)
    worst(acc, "mel_dct", e)
    assert e <= o.C_DCT, (n_mels, n_mfcc, N, e)
    return v, d, got


@pytest.mark.parametrize("n_mfcc", MFCC)
def test_mel_dct_coefficient_chunks(eng, n_mfcc):
    for n_mels in MELS:
        for N in FRAMES:
            check_dct(eng, 2, n_mels, n_mfcc, N, n_mfcc * 1000 + n_mels + N)


@pytest.mark.parametrize("n_mfcc,n_mels", [(80, 40), (33, 128), (128, 256)])
def test_mel_dct_transposed_basis(eng, n_mfcc, n_mels):
    check_dct(eng, 3, n_mels, n_mfcc, 129, 7, transposed=True)


def test_mel_dct_largest_basis_and_refusals(eng):
    check_dct(eng, 1, 256, 200, 130, 8)  # 256 x 200 x 4 B = 200 KB
    v = dev(torch.zeros(1, 1, 256, 4))
    with pytest.raises(RuntimeError):
        eng.mel_dct(v, dev(torch.zeros(256, 201)))
    check_dct(eng, 65535, 4, 3, 2, 9)
    with pytest.raises(RuntimeError):
        eng.mel_dct(dev(torch.zeros(65536, 1, 4, 2)), dev(torch.zeros(4, 3)))


def test_mfcc_forward_and_backward_at_the_defaults(eng):
    """AudioSignal.mfcc() at the reference's defaults (n_mfcc 40, n_mels 80, log offset 1e-6) against a float64 product
    of the reference's DCT with log(mel + 1e-6) (torch's log: within 2 u of the fused one); the DCT's backward
    (the same kernel with the transposed basis) against a float64 product; the full backward reaches the samples."""
    from audiotools_b200 import AudioSignal
    from audiotools_b200.core import grad as G

    x = torch.from_numpy(rng(40).standard_normal((2, 1, 22050)).astype(np.float32)) * 0.1
    mf = AudioSignal(dev(x), 22050).mfcc().cpu()
    logmel = torch.log(AudioSignal(dev(x), 22050).mel_spectrogram(n_mels=80) + 1e-6).cpu()
    dct = AudioSignal.get_dct(40, 80, "ortho", "cpu")
    assert mf.shape[-2] == 40
    assert o.mel_dct_err(mf, logmel, dct) <= o.C_DCT + 2
    lm = dev(logmel).requires_grad_(True)
    g = torch.from_numpy(rng(41).standard_normal(tuple(mf.shape)).astype(np.float32))
    G.MelDCT.apply(lm, dev(dct)).backward(dev(g))
    assert o.mel_dct_err(lm.grad.cpu(), g, dct.t()) <= o.C_DCT
    xd = dev(x).requires_grad_(True)
    AudioSignal(xd, 22050).mfcc().backward(dev(g))
    assert bool(torch.isfinite(xd.grad).all()) and bool((xd.grad != 0).any())


# --------------------------------------------------------------------------- pack_rows
def pack_c(eng, views, offsets, C, T_out):
    """b2a_pack_rows_f32 through the C ABI: views are [C, len] tensors of any row stride (the engine copies those)."""
    table = torch.tensor([[v.data_ptr(), v.shape[-1], v.stride(0), off] for v, off in zip(views, offsets)],
                         dtype=torch.int64).t().contiguous().to(DEV)
    out = torch.full((len(views), C, T_out), 7.0, device=DEV)
    rc = eng.lib.b2a_pack_rows_f32(ctypes.c_void_p(table[0].data_ptr()), ctypes.c_void_p(table[1].data_ptr()),
                                   ctypes.c_void_p(table[2].data_ptr()), ctypes.c_void_p(table[3].data_ptr()),
                                   len(views), C, T_out, ctypes.c_void_p(out.data_ptr()), stream_of(out))
    assert rc == 0
    if DEV != "cpu":
        torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("T_out", [4, 1024, 1021, 1022, 1023, 4096])
def test_pack_rows_tails_offsets_strides(eng, T_out):
    """Items 1, 2 and 3 samples short of a multiple of 4 in front of non-zero memory (the float4 tail), negative
    offsets and offsets past the end, views offset by one float, and [C, T] slices whose row stride is not T."""
    big = dev(torch.from_numpy(rng(T_out).standard_normal((2, 6000)).astype(np.float32)) + 10.0)
    views, offs = [], []
    for length in (1021, 1022, 1023, 1024, 5):
        for off in (0, 4, -3, -4, 1024 - length + 4, 5000):
            views.append(big[:, :length])     # row stride 6000, aligned
            offs.append(off)
    views += [big[:, 1:1023], big[:, 3:3000], big[:, 4:1026]]  # one float off, and aligned again
    offs += [0, 1, 4]
    got = pack_c(eng, views, offs, 2, T_out)
    want = o.pack_rows([v.cpu().numpy() for v in views], offs, T_out)
    assert np.array_equal(got, want)
    via_engine = eng.pack_rows(views, T_out, offsets=offs).cpu().numpy()  # contiguous copies, same values
    assert np.array_equal(via_engine, want)


def test_pack_rows_row_limit(eng):
    x = dev(torch.arange(12, dtype=torch.float32).reshape(1, 12))
    got = pack_c(eng, [x] * 65535, [0] * 65535, 1, 8)
    assert np.array_equal(got, np.tile(np.arange(8, dtype=np.float32), (65535, 1, 1)))
    lib = eng.lib
    p = ctypes.c_void_p(x.data_ptr())
    n0 = lib.kernel_launches.value
    assert lib.b2a_pack_rows_f32(p, p, p, p, 65536, 1, 8, p, stream_of(x)) == -1
    assert lib.b2a_pack_rows_f32(p, p, p, p, 32768, 2, 8, p, stream_of(x)) == -1
    assert lib.kernel_launches.value == n0


# --------------------------------------------------------------------------- refusals and invariances
def test_refusals_through_the_c_abi(eng):
    """alter_drr refuses rows whose int sample index would overflow (T > INT_MAX - 512, or td + t0 past INT_MAX);
    mel_dct refuses frame counts whose last 128-frame tile passes INT_MAX.  Nothing is launched (the buffers are never
    read)."""
    lib = eng.lib
    buf = dev(torch.zeros(1024))
    p = ctypes.c_void_p(buf.data_ptr())
    o_ = dev(torch.zeros(1024))
    q = ctypes.c_void_p(o_.data_ptr())
    st = stream_of(buf)
    n0 = lib.kernel_launches.value
    assert lib.b2a_alter_drr_f32(p, q, 1, 1000, 1, INT_MAX - 999, p, 1.0, st) == -1
    assert lib.b2a_alter_drr_f32(p, q, 1, 1000, 1, -1, p, 1.0, st) == -1
    for T in (INT_MAX - 511, INT_MAX, 2 ** 31):
        assert lib.b2a_alter_drr_f32(p, q, 1, T, 1, 0, p, 1.0, st) == -1, T
    for N in (INT_MAX - 126, INT_MAX, 2 ** 31):
        assert lib.b2a_mel_dct_f32(p, 1, 1, N, p, 1, q, st) == -1, N
    assert lib.b2a_order_stats_f32(p, 64, p, 65536, q, st) == -1
    assert lib.b2a_order_stats_f32(p, 0, p, 1, q, st) == -1
    assert lib.kernel_launches.value == n0


def test_reruns_bit_identical(eng):
    x = dev(ir_like(3, 2, 1500, 50))
    drr = dev(torch.tensor([1.0, 5.0, 9.0]))
    g, y, xr = (dev(t) for t in ps_data(4, 1000, 51))
    v = dev(torch.randn(2, 1, 80, 300))
    d = dev(torch.randn(80, 40))
    row = dev(torch.randn(5000))
    ks = torch.tensor([0, 17, 2500, 4999])
    runs = [[eng.alter_drr(x, 44100, drr), *eng.peak_scale_backward(g, y, xr), eng.peak_scale_backward(g, y)[0],
             eng.mel_dct(v, d), eng.order_stats(row, ks), eng.quantize(y, torch.tensor(256.0), mulaw=True)]
            for _ in range(3)]
    for a in runs[1:]:
        for s, t in zip(runs[0], a):
            assert torch.equal(s.view(torch.int32), t.view(torch.int32))


def test_batch_equals_single_items(eng):
    x = ir_like(4, 2, 1200, 60, peaks=[100, 104])
    drr = torch.tensor([-3.0, 2.0, 7.0, 14.0])
    full = eng.alter_drr(dev(x), 44100, dev(drr)).cpu()
    g, y, xr = ps_data(4, 900, 61)
    gy, gx = eng.peak_scale_backward(dev(g), dev(y), dev(xr))
    v, d = torch.randn(4, 1, 40, 200), torch.randn(40, 33)
    mf = eng.mel_dct(dev(v), dev(d)).cpu()
    for b in range(4):
        assert torch.equal(eng.alter_drr(dev(x[b:b + 1]), 44100, dev(drr[b:b + 1])).cpu(), full[b:b + 1])
        sy, sx = eng.peak_scale_backward(dev(g[b:b + 1]), dev(y[b:b + 1]), dev(xr[b:b + 1]))
        assert torch.equal(sy.cpu(), gy[b:b + 1].cpu()) and torch.equal(sx.cpu(), gx[b:b + 1].cpu())
        assert torch.equal(eng.mel_dct(dev(v[b:b + 1]), dev(d)).cpu(), mf[b:b + 1])


def test_power_of_two_scaling_is_exact(eng):
    """Scaling the input by 2^k scales order statistics, the DCT and pack_rows by exactly 2^k."""
    row = torch.randn(5000)
    ks = torch.tensor([0, 100, 2500, 4999])
    v, d = torch.randn(2, 1, 80, 150), torch.randn(80, 40)
    a = torch.randn(2, 3000)
    for k in (-3, 5):
        s = 2.0 ** k
        assert torch.equal(eng.order_stats(dev(row * s), ks).cpu(), eng.order_stats(dev(row), ks).cpu() * s)
        assert torch.equal(eng.mel_dct(dev(v * s), dev(d)).cpu(), eng.mel_dct(dev(v), dev(d)).cpu() * s)
        assert torch.equal(eng.pack_rows([dev(a * s)], 1001, offsets=[-5]).cpu(),
                           eng.pack_rows([dev(a)], 1001, offsets=[-5]).cpu() * s)
