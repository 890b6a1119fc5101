"""The time-domain engines on the H100 (``-m gpu``) against float64, per sample and per block (tests/timedomain64.py):
``fir_direct_kernel`` (low / high-pass up to 320 taps, the decimating resampler), the overlap-save engine (``fftconv``:
long low-pass, equaliser, circular convolution), ``resample_kernel`` and the K-weighting (``kweight_energy_warp_kernel``
+ ``lufs_gate_kernel``), at the tap counts, lengths, strides and rates where their tiling changes, and exact
invariances (power-of-two scaling, row independence).  Each error is held to its route's budget (tests/timedomain64.py,
measured on an H100 80GB HBM3 at a 400 W power limit); the K-weighting is also held to a stated factor of the error of
the reference's sequential float32 cascade on the same input.  tests/probes/timedomain_accuracy_probe.py prints the table
of DESIGN.md "Time-domain accuracy"."""
import math

import numpy as np
import pytest
import torch

from tests import timedomain64 as td

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


def _noise(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(*shape, generator=g, dtype=torch.float64)).float()


def _taps(n_filt, K, seed):
    g = torch.Generator().manual_seed(1000 + seed)
    return (torch.randn(n_filt, K, generator=g, dtype=torch.float64) / math.sqrt(K)).float()


# --------------------------------------------------------------------------- fir_direct
def check_fir_direct(eng, T, K, stride, pad_mode="replicate", subtract=False, left0=None, rows=3, bypass=None,
                     levels=(1.0, 1e-3, 1e-6)):
    """Rows at three levels (one filter per row), per sample against the float64 direct sum."""
    x = torch.cat([_noise((1, T), 7 * K + T + r, lv) for r, lv in zip(range(rows), levels * rows)], 0)
    taps = _taps(rows, K, K + stride)
    left = torch.arange(rows, dtype=torch.int32) * 3
    left0 = K // 2 if left0 is None else left0
    out_len = (T + stride - 1) // stride
    got = eng.fir_direct(x.to(DEV), taps.to(DEV), 1, left=left.to(DEV), left0=left0, stride=stride, out_len=out_len,
                         pad_mode=pad_mode, subtract_from_input=subtract,
                         bypass=None if bypass is None else torch.tensor(bypass))
    y, a = td.fir_direct64(x, taps, 1, left=left, left0=left0, stride=stride, out_len=out_len, pad_mode=pad_mode,
                           subtract=subtract, bypass=bypass)
    e = td.direct_errors(got, y, a)
    if bypass is not None:
        for r, b in enumerate(bypass):
            if b:
                assert torch.equal(got[r].cpu(), x[r, :out_len]), "bypassed row not copied exactly"
    return e.max() / (td.U * math.sqrt(K))


FIR_K = [1, 7, 8, 9, 103, 319, 320]
FIR_STRIDE = [1, 2, 3, 6]


@pytest.mark.parametrize("K", FIR_K)
@pytest.mark.parametrize("stride", FIR_STRIDE)
def test_fir_direct_per_sample(eng, K, stride):
    for T in sorted({1, max(1, K - 1), 2047, 2048, 2049, 3 * 2048 * stride + 5}):
        if not eng.lib.b2a_fir_direct_supported(T, K, stride):
            continue
        c = check_fir_direct(eng, T, K, stride)
        assert c <= td.BUDGET_C["fir_direct"], (T, K, stride, c)


@pytest.mark.parametrize("pad_mode", ["replicate", "constant"])
@pytest.mark.parametrize("subtract", [False, True])
def test_fir_direct_pad_subtract_bypass(eng, pad_mode, subtract):
    """``left`` beyond K (the whole filter reads the padding at the edges), x - y, mixed bypass."""
    for K, T in ((103, 5000), (320, 4099)):
        c = check_fir_direct(eng, T, K, 1, pad_mode=pad_mode, subtract=subtract, left0=K + 37, rows=4,
                             bypass=[0, 1, 0, 1])
        assert c <= td.BUDGET_C["fir_direct"], (K, T, c)


def test_fir_direct_largest_stride(eng):
    """The largest stride the direct kernel accepts for a decimator of 2 width + stride taps, width = ceil(24 stride /
    0.945) (julius' geometry when the reduced new rate is 1)."""
    def taps(st):
        return 2 * math.ceil(24 * st / 0.945) + st

    s = max(st for st in range(1, 4096) if eng.lib.b2a_fir_direct_supported(20000, taps(st), st))
    K = taps(s)
    c = check_fir_direct(eng, 20000, K, s)
    assert c <= td.BUDGET_C["fir_direct"], (s, c)


# --------------------------------------------------------------------------- fftconv
def check_fftconv(eng, T, L, pad_mode="replicate", rows_per_filt=1, n_filt=2, offset=None, offset0=0,
                  post_scale=None, subtract=False, seed=0):
    rows = rows_per_filt * n_filt
    x = torch.cat([_noise((1, T), seed + 11 * r, 10.0 ** (-3 * (r % 3))) for r in range(rows)], 0)
    g = _taps(n_filt, L, L + seed)
    got = eng.fftconv(x.to(DEV), g.to(DEV), rows_per_filt, offset=None if offset is None else offset.to(DEV),
                      offset0=offset0, pad_mode=pad_mode, post_scale=None if post_scale is None else post_scale.to(DEV),
                      subtract_from_input=subtract)
    y, scale = td.fftconv64(x, g, rows_per_filt, offset=offset, offset0=offset0, pad_mode=pad_mode,
                            post_scale=post_scale, subtract=subtract)
    return td.block_errors(got, y, scale).max() / td.fft_budget("fftconv", L) * td.BUDGET_C["fftconv"]


FFT_L = [1, 1023, 1024, 1025, 2049, 4097, 44983]
FFT_T = [1, 1023, 1024, 1025, 9000]


@pytest.mark.parametrize("L", FFT_L)
def test_fftconv_per_block(eng, L):
    for T in FFT_T:
        c = check_fftconv(eng, T, L, offset0=L // 2)
        assert c <= td.BUDGET_C["fftconv"], (T, L, c)


@pytest.mark.parametrize("pad_mode", ["replicate", "constant", "circular"])
def test_fftconv_modes_offsets_scale(eng, pad_mode):
    """All three extensions, per-filter offsets up to L - 1, post_scale and x - y."""
    for L, T in ((641, 5000), (2049, 7000)):
        off = torch.tensor([0, L - 1], dtype=torch.int32)
        ps = torch.tensor([0.5, -3.0])
        for subtract in (False, True):
            c = check_fftconv(eng, T, L, pad_mode=pad_mode, offset=off, offset0=0, post_scale=ps, subtract=subtract)
            assert c <= td.BUDGET_C["fftconv"], (L, T, subtract, c)


def test_fftconv_many_block_ctas(eng):
    """T > 524 288 with L > 1024 taps: several freq_fir_kernel CTAs along the block index."""
    c = check_fftconv(eng, 600_001, 2049, offset0=1024, n_filt=1)
    assert c <= td.BUDGET_C["fftconv"], c


def _fftconv_chunk_rows(T, L):
    """fftconv.cu ``layout``: rows per chunk = 256 MB / (per-row X spectra, and Y with several partitions)."""
    NB = (T + td.FFT_BLOCK - 1) // td.FFT_BLOCK
    P = (L + td.FFT_BLOCK - 1) // td.FFT_BLOCK
    per_row = 1025 * (NB + P - 1 + (NB if P > 1 else 0)) * 8
    return max(1, (256 << 20) // per_row)


def test_fftconv_rows_straddle_chunks(eng):
    """Two rows per filter, T chosen so the row chunk is odd: filter 'chunk // 2' has one row in each chunk."""
    L = 641
    T = next(t for t in range(441_000, 600_000, 1024) if _fftconv_chunk_rows(t, L) % 2 == 1)
    chunk = _fftconv_chunk_rows(T, L)
    n_filt = chunk // 2 + 2
    x = _noise((2 * n_filt, T), 5)
    g = _taps(n_filt, L, 3)
    got = eng.fftconv(x.to(DEV), g.to(DEV), 2, offset0=L // 2).cpu()
    f = chunk // 2  # rows 2f (chunk 0) and 2f + 1 (chunk 1)
    keep = [0, 2 * f, 2 * f + 1, 2 * n_filt - 1]
    y, scale = td.fftconv64(x[keep], g[[0, f, f, n_filt - 1]], 1, offset0=L // 2)
    c = td.block_errors(got[keep], y, scale).max() / td.fft_budget("fftconv", L) * td.BUDGET_C["fftconv"]
    assert c <= td.BUDGET_C["fftconv"], (chunk, c)
    alone = eng.fftconv(x[2 * f + 1:2 * f + 2].to(DEV), g[f:f + 1].to(DEV), 1, offset0=L // 2).cpu()
    assert torch.equal(alone[0], got[2 * f + 1]), "a row in the second chunk differs from the row alone"


# --------------------------------------------------------------------------- circular convolution
def check_circconv(eng, T, L, n_ir_items, C=2, roll=True, seed=0, ir=None):
    B = 2
    x = _noise((B, C, T), seed)
    if ir is None:
        ir = _noise((n_ir_items, C if n_ir_items > 1 else 1, L), seed + 1) * 0.3
    got = eng.circular_convolve(x.to(DEV), ir.to(DEV), roll_to_peak=roll).cpu()
    irb = ir.expand(B, C, -1) if ir.shape[0] == 1 or ir.shape[1] == 1 else ir
    irb = irb.expand(B, C, -1).reshape(B * C, -1)
    y, scale = td.circconv64(x.reshape(B * C, T), irb, 1, roll)
    return td.block_errors(got.reshape(B * C, T), y, scale).max() / td.fft_budget("circconv", min(L, T)) \
        * td.BUDGET_C["circconv"]


@pytest.mark.parametrize("T,L", [(3000, 3000), (5000, 1200), (2000, 4500), (1, 1)])
@pytest.mark.parametrize("roll", [True, False])
def test_circconv_per_block(eng, T, L, roll):
    for n_items in (1, 2):
        c = check_circconv(eng, T, L, n_items, roll=roll)
        assert c <= td.BUDGET_C["circconv"], (T, L, n_items, c)


def test_circconv_tied_and_tiny_peaks(eng):
    """Tied peaks roll to the first; a peak below 1e-5 is scaled by 1e5, not by 1 / peak."""
    ir = torch.zeros(1, 1, 700)
    ir[0, 0, 100] = 0.5
    ir[0, 0, 400] = -0.5
    ir[0, 0, 200] = 0.25
    assert check_circconv(eng, 4000, 700, 1, ir=ir) <= td.BUDGET_C["circconv"]
    c = check_circconv(eng, 4000, 700, 1, ir=_noise((1, 1, 700), 3, 1e-7))
    assert c <= td.BUDGET_C["circconv"], c


# --------------------------------------------------------------------------- resample
RESAMPLE = [(48000, 16000), (44100, 22050), (96000, 16000), (44100, 16000), (16000, 44100), (44100, 48000),
            (48000, 44100), (8000, 44100), (44100, 8000)]


def check_resample(eng, old_sr, new_sr, T, rows=3):
    x = torch.cat([_noise((1, T), T + r, lv) for r, lv in zip(range(rows), (1.0, 1e-3, 1e-6))], 0)
    got = eng.resample(x.to(DEV), old_sr, new_sr)
    kt, width, old, new = eng._resample_kernel(old_sr, new_sr, DEV)  # the taps the device formed
    y, a = td.resample64(x, old_sr, new_sr, kt)
    return td.direct_errors(got, y, a).max() / (td.U * math.sqrt(kt.shape[0]))


@pytest.mark.parametrize("old_sr,new_sr", RESAMPLE)
def test_resample_per_sample(eng, old_sr, new_sr):
    g = math.gcd(old_sr, new_sr)
    old, new = old_sr // g, new_sr // g
    width = td.resample_width(old_sr, new_sr)
    K = 2 * width + old
    tile_in = 1024 * old // new  # input samples behind one 1024-output tile
    for T in sorted({1, 2, max(1, width - 1), max(1, K - 1), tile_in - 1, tile_in + old, 3 * tile_in + 1}):
        if new * T // old < 1:
            continue
        c = check_resample(eng, old_sr, new_sr, T)
        rt = td.resample_route(eng.lib, T, old_sr, new_sr)
        assert c <= td.BUDGET_C[rt], (old_sr, new_sr, T, rt, c)


# --------------------------------------------------------------------------- invariances
def test_power_of_two_scaling_is_exact(eng):
    x = _noise((2, 1, 9000), 1)
    taps = _taps(1, 103, 1)
    g = _taps(1, 2049, 2)
    ops = {
        "fir_direct": lambda v: eng.fir_direct(v, taps.to(DEV), 2, left0=51),
        "fftconv": lambda v: eng.fftconv(v, g.to(DEV), 2, offset0=1024),
        "resample": lambda v: eng.resample(v, 44100, 16000),
        "decimate": lambda v: eng.resample(v, 48000, 16000),
    }
    for name, op in ops.items():
        base = op(x.to(DEV)).cpu()
        for k in (-20, -7, 1, 13, 20):
            assert torch.equal(op((x * 2.0 ** k).to(DEV)).cpu(), base * 2.0 ** k), (name, k)
    blocks = eng.lufs(x.to(DEV), 44100, want_blocks=True)["blocks"].cpu()
    for k in (-20, -3, 5, 20):
        assert torch.equal(eng.lufs((x * 2.0 ** k).to(DEV), 44100, want_blocks=True)["blocks"].cpu(),
                           blocks * 4.0 ** k), k


@pytest.mark.parametrize("n_rows", [1, 7, 300])
def test_rows_are_independent(eng, n_rows):
    T = 5000
    x = _noise((n_rows, T), n_rows)
    r = n_rows // 2
    taps = _taps(1, 103, 4)
    g = _taps(1, 1025, 5)
    for name, op in {"fir_direct": lambda v: eng.fir_direct(v, taps.to(DEV), v.shape[0], left0=51),
                     "fftconv": lambda v: eng.fftconv(v, g.to(DEV), v.shape[0], offset0=512),
                     "resample": lambda v: eng.resample(v, 44100, 16000)}.items():
        assert torch.equal(op(x.to(DEV))[r].cpu(), op(x[r:r + 1].to(DEV))[0].cpu()), name


def test_tile_shift_is_exact(eng):
    """Interior outputs move exactly under a shift by a whole tile."""
    x = _noise((1, 30000), 9)
    taps = _taps(1, 103, 6)
    s = 2048
    a = eng.fir_direct(x.to(DEV), taps.to(DEV), 1, left0=51).cpu()
    b = eng.fir_direct(x[:, s:].to(DEV), taps.to(DEV), 1, left0=51).cpu()
    assert torch.equal(a[:, s + 200:-200], b[:, 200:-200])
    g = _taps(1, 1500, 7)
    a = eng.fftconv(x.to(DEV), g.to(DEV), 1, offset0=700).cpu()
    b = eng.fftconv(x[:, 1024:].to(DEV), g.to(DEV), 1, offset0=700).cpu()
    assert torch.equal(a[:, 1024 + 2048:-2048], b[:, 2048:-2048])
    # resample 44.1k -> 16k: old = 441, new = 160; a 1024-output tile spans 1024 / new frames = 6.4 -- shift by
    # 5 tiles (32 frames, 32 * 441 input samples)
    a = eng.resample(x.to(DEV), 44100, 16000).cpu()
    b = eng.resample(x[:, 32 * 441:].to(DEV), 44100, 16000).cpu()
    assert torch.equal(a[:, 5120 + 200:5120 + 200 + 4000], b[:, 200:4200])


# --------------------------------------------------------------------------- K-weighting
KW_RATES = [8000, 11025, 16000, 22050, 44100, 48000, 96000, 192000]


def kw_signals(sr, T, seed=0):
    """{name: [T] float64}: noise at three levels, a DC step, 20-60 Hz tones over noise 20 dB down, loud then -100 dB.
    The drop lands on a gating interval boundary inside a 64-sample lane chunk, where one lane's energy is split
    between a loud and a quiet interval."""
    g = np.random.default_rng(seed + sr)
    t = np.arange(T) / sr
    n = g.standard_normal(T)
    stride = td.kweight_geometry(T, sr)[1]
    # the first boundary past T / 2 that is not a multiple of 64 (at 48 kHz every one is: the drop is then at T / 2 + 4800
    # + 32, inside an interval and inside a lane chunk)
    drop = next((j * stride for j in range(T // (2 * stride), T // stride) if (j * stride) % 64), T // 2 + stride + 32)
    out = {"noise": 0.3 * n, "noise_1e-3": 1e-3 * n, "noise_1e-6": 1e-6 * n,
           "dc_step": np.where(t < t[-1] / 3, 0.5, -0.2) + 1e-3 * n,
           "loud_then_-100dB": np.where(np.arange(T) < drop, 0.5 * n, 0.5e-5 * n)}
    for f in (20, 30, 45, 60):
        out[f"sin{f}+noise"] = 0.5 * np.sin(2 * np.pi * f * t + 0.3) + 0.05 * n
    return out


def check_kweight(eng, sr, T, C=1, names=None, seed=0, vs_seq32=True):
    """(worst budget ratio, worst ratio to the sequential float32 cascade) over every row of every signal."""
    sig = kw_signals(sr, T, seed)
    names = names or list(sig)
    x = np.stack([np.stack([sig[n] * (1.0 - 0.1 * c) for c in range(C)]) for n in names]).astype(np.float32)
    z = eng.lufs(torch.from_numpy(x).to(DEV), sr, want_blocks=True)["blocks"].cpu().double().numpy()
    z64 = td.kweight_blocks64(x, sr)
    e = td.kweight_block_errors(z, z64).max(-1) / td.U  # [B, C] in u
    budget = np.array([td.kweight_budget(sr, n) for n in names])[:, None]
    worst_budget = (e / budget).max()
    worst_vs = 0.0
    if vs_seq32:
        zr = td.kweight_blocks64(x, sr, filtered=td.kweight_seq32(x, td.kweight_coef(sr)))
        er = td.kweight_block_errors(zr, z64).max(-1) / td.U
        # a floor of 16 u: both are at rounding level there and their ratio says nothing
        factor = np.array([td.kweight_vs_seq32(n) for n in names])[:, None]
        worst_vs = (e / np.maximum(er, 16.0) / factor).max() * td.KW_VS_SEQ32
    return worst_budget, worst_vs, e


@pytest.mark.parametrize("sr", KW_RATES)
def test_kweight_per_block_against_float64(eng, sr):
    b, v, e = check_kweight(eng, sr, int(2.5 * sr))
    assert b <= 1.0, (sr, e.max())
    assert v <= td.KW_VS_SEQ32, (sr, v)


@pytest.mark.parametrize("C", [2, 5])
def test_kweight_channels(eng, C):
    b, v, e = check_kweight(eng, 44100, 3 * 44100, C=C, names=["noise", "sin30+noise", "dc_step"])
    assert b <= 1.0 and v <= td.KW_VS_SEQ32, (C, e.max(), v)


@pytest.mark.parametrize("T", [100, 2047, 2048, 17640, 17641, 2048 * 5 + 3])
def test_kweight_short_rows(eng, T):
    """Rows shorter than a block, of one segment, a few segments (padded_length = T)."""
    b, v, e = check_kweight(eng, 44100, T, names=["noise", "sin20+noise"], vs_seq32=False)
    assert b <= 1.0, (T, e.max())


@pytest.mark.parametrize("sr", [44100, 22050])
def test_kweight_runs_agree(eng, sr):
    """The row count sets run_len (runs per row = resident warps / rows, at least 4 warm-ups long) and with it where
    warm-ups start.  The same row in a batch of 1 (run_len 12 segments at 44.1 kHz on 132 SMs), of 300 (5 runs per row)
    and of 2000 (more rows than resident warps: one run per row, no warm-up) is held to float64 per block within the
    budget, and to its factor of the sequential float32 cascade.  The row falls by 100 dB on a gating-interval boundary inside
    a lane chunk, where a too-short warm-up or a shared lane sum would carry the loud part into the quiet one."""
    T = 20 * sr
    row = kw_signals(sr, T)["loud_then_-100dB"].astype(np.float32)
    z64 = td.kweight_blocks64(row.astype(np.float64), sr)
    er = td.kweight_block_errors(td.kweight_blocks64(row, sr, filtered=td.kweight_seq32(row, td.kweight_coef(sr))),
                                 z64).max() / td.U
    for n in (1, 300, 2000):
        x = torch.from_numpy(row).to(DEV).expand(n, 1, T).contiguous()
        z = eng.lufs(x, sr, want_blocks=True)["blocks"][n // 2, 0].cpu().double().numpy()
        del x
        e = td.kweight_block_errors(z, z64).max() / td.U
        assert e <= td.kweight_budget(sr, "loud_then_-100dB"), (n, e)
        assert e <= td.kweight_vs_seq32("loud_then_-100dB") * max(er, 16.0), (n, e, er)


def loudness64(z, rate, C):
    """Integrated loudness (BS.1770 gating) of float64 block energies z [C, nblk]."""
    from audiotools_b200.core import kweighting

    G = kweighting.CHANNEL_GAINS[:C]
    l = -0.691 + 10 * np.log10((G[:, None] * z).sum(0))
    keep = l > -70
    zr = z[:, keep].mean(-1)
    gr = -0.691 + 10 * np.log10((G * zr).sum()) - 10
    keep &= l > gr
    return -0.691 + 10 * np.log10((G * z[:, keep].mean(-1)).sum())


@pytest.mark.parametrize("sr", [44100, 48000])
def test_integrated_loudness_against_float64(eng, sr):
    """Bass tones over noise: the gated loudness within the per-block budget of float64 (the blocks are far from
    either gate threshold)."""
    T = 3 * sr
    t = np.arange(T) / sr
    g = np.random.default_rng(sr)
    x = np.stack([0.5 * np.sin(2 * np.pi * f * t) + 0.05 * g.standard_normal(T) for f in (20, 30, 45)])
    x = x[:, None, :].astype(np.float32)
    got = eng.lufs(torch.from_numpy(x).to(DEV), sr)["lufs"].cpu().double().numpy()
    z64 = td.kweight_blocks64(x.astype(np.float64), sr)
    want = np.array([loudness64(z64[b], sr, 1) for b in range(x.shape[0])])
    # the result is float32 (ulp 1.9e-6 dB at -20 LUFS) and its blocks are within a few hundred u of float64
    # (1e-5 dB); measured 2.2e-5 dB, against -0.014 .. -0.0003 dB before the state basis change
    tol = 5e-5
    assert np.abs(got - want).max() <= tol, (got - want)


# --------------------------------------------------------------------------- adjoints on the same references
@pytest.mark.parametrize("old_sr,new_sr", [(48000, 16000), (44100, 16000), (16000, 44100), (11025, 96000)])
def test_resample_backward_per_sample(eng, old_sr, new_sr):
    """Both routes' adjoint (11 025 -> 96 000 is the phase-tiled one), per input sample against the float64 adjoint."""
    kt, width, old, new = eng._resample_kernel(old_sr, new_sr, DEV)
    for T in (5, 3001):
        n_out = new * T // old
        g = torch.cat([_noise((1, n_out), T + r, lv) for r, lv in enumerate((1.0, 1e-4))], 0)
        got = eng.resample_backward(g.to(DEV), T, old_sr, new_sr)
        gx, a = td.resample_backward64(g, T, old_sr, new_sr, kt)
        c = td.direct_errors(got, gx, a).max() / (td.U * math.sqrt(kt.shape[0]))
        assert c <= td.BUDGET_C["resample"], (old_sr, new_sr, T, c)


def test_equalizer_backward_per_sample(eng):
    """``fftconv`` in constant mode + ``fir_pad_fold`` against the float64 adjoint of the replicate-padded FIR."""
    B, C, T = 2, 2, 6000
    db = torch.tensor([[3.0, -6.0, 1.0, 0.0, -2.0, 4.0], [-1.0, 2.0, 0.5, -3.0, 1.0, 0.0]])
    g = _noise((B, C, T), 4)
    got = eng.equalizer_backward(g.to(DEV), 44100, db)
    h, half = eng._equalizer_taps(44100, db, B, DEV)
    gx, a = td.fir_backward64(g, h, C, half)
    # as the overlap-save forward: per 1024-sample block against ||h|| rms(g) (g is stationary noise)
    ref_scale = np.linalg.norm(td._np64(h), axis=1).repeat(C)[:, None] * np.sqrt((td._np64(g).reshape(B * C, T) ** 2)
                                                                                 .mean(-1, keepdims=True))
    c = td.block_errors(got, gx, np.broadcast_to(ref_scale, (B * C, (T + 1023) // 1024))).max()
    assert c <= td.fft_budget("fftconv", h.shape[1]), c / td.fft_budget("fftconv", h.shape[1])


@pytest.mark.parametrize("T,L", [(3000, 3000), (5000, 1200), (2000, 4500)])
def test_circconv_backward_per_block(eng, T, L):
    B, C = 2, 2
    g = _noise((B, C, T), 8)
    ir = _noise((B, C, L), 9) * 0.3
    got = eng.circular_convolve_backward(g.to(DEV), ir.to(DEV)).cpu()
    gx, scale = td.circconv_backward64(g.reshape(B * C, T), ir.reshape(B * C, L), 1)
    c = td.block_errors(got.reshape(B * C, T), gx, scale).max()
    assert c <= td.fft_budget("circconv", min(L, T)), c / td.fft_budget("circconv", min(L, T))
