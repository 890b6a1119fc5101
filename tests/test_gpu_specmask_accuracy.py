"""The spectral masks and the spectral gate of csrc/specmask.cu on the H100 (``-m gpu``), per cell against float64
(tests/specmask64.py) at the edges of their tiling: the band masks bit for bit at both block sizes, on both axes, with
bands on and one float beside grid values; ``rotate`` past the grid-stride cap; ``mask_low_magnitudes`` with its
batch-wide floor, silent batches, infinite cut-offs and cells built at 0.5 and 2 decision margins from the cut-off;
the gate stage by stage (thresholds, smoothed mask, output) around its 16 x 64 tiles and halos up to 8, with an
asymmetric smoothing that pins the orientation of the cross-correlation; NaN and inf against the reference's arithmetic;
refusals through the C ABI, reruns, and rows past flat index 2^31.
tests/probes/specmask_accuracy_probe.py prints the table of DESIGN.md "Spectral mask accuracy"."""
import ctypes
import math

import numpy as np
import pytest
import torch

from audiotools_b200.ml.layers.spectral_gate import _ramp
from tests import specmask64 as s

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
U = s.U
F_EDGES = [1, 15, 16, 17, 33, 1025]
N_EDGES = [1, 63, 64, 65, 255, 256, 257, 1000]
HALVES = [0, 1, 3, 5, 8]
NZ_FRAMES = [1, 2, 50, 2584]
ASYM_F = [1.0, 2.0, 4.0]              # odd, asymmetric: a convolution would flip them
ASYM_T = [0.5, 1.0, 3.0, 0.25, 2.0]


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


def cplx(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.complex(torch.randn(shape, generator=g), torch.randn(shape, generator=g)) * scale).to(torch.complex64)


def dev(t):
    return t.to(DEV)


def worst(acc, key, v):
    v = float(v)
    if not math.isnan(v):
        acc[key] = max(acc.get(key, 0.0), v)


# --------------------------------------------------------------------------- band masks
def band_edges(v):
    """Per-item (lo, hi) for 3 items: exactly on grid values, one float below, one float above."""
    L = v.numel()
    k, j = L // 3, min(L - 1, (2 * L) // 3 + 1)
    lo0 = float(v[k])
    hi0 = float(v[j]) if j > k else float(np.nextafter(np.float32(lo0), np.float32(np.inf)))
    f32 = np.float32
    lo = [lo0, np.nextafter(f32(lo0), f32(-np.inf)), np.nextafter(f32(lo0), f32(np.inf))]
    hi = [hi0, np.nextafter(f32(hi0), f32(np.inf)), np.nextafter(f32(hi0), f32(-np.inf))]
    return torch.tensor(lo, dtype=torch.float32), torch.tensor(hi, dtype=torch.float32)


def with_zeros(X):
    """X with cells set to each of the four signed zeros (the backward's X == 0 rule)."""
    X = X.clone()
    flat = torch.view_as_real(X).reshape(-1, 2)
    n = flat.shape[0]
    for i, (re, im) in enumerate(((0.0, 0.0), (-0.0, 0.0), (0.0, -0.0), (-0.0, -0.0))):
        idx = torch.arange(i, n, 7 + i)
        flat[idx, 0] = re
        flat[idx, 1] = im
    return X


def check_band(eng, F, N, axis, val=0.7, seed=0):
    B, C = 3, 2
    X = with_zeros(cplx((B, C, F, N), seed + F * 1009 + N))
    Gr = cplx((B, C, F, N), seed + 7)
    v = torch.linspace(0, 8000.0, F) if axis == 0 else torch.linspace(0, 1.5, N)
    lo, hi = band_edges(v)
    m = s.band(v, lo, hi, F, N, C, axis)
    want = s.band_forward(X, m, val)
    Xd = dev(X)
    got_in = eng.spec_band_mask(Xd.clone(), dev(v), dev(lo), dev(hi), axis, val)
    got_out = eng.spec_band_mask_out(Xd, dev(v), dev(lo), dev(hi), axis, val)
    gx = eng.spec_band_mask_backward(dev(Gr), Xd, dev(v), dev(lo), dev(hi), axis)
    where = (F, N, axis)
    assert torch.equal(s.bits(got_in), s.bits(want)), where
    assert torch.equal(s.bits(got_out), s.bits(want)), where
    assert torch.equal(s.bits(Xd), s.bits(X)), where  # out of place leaves its input alone
    assert torch.equal(s.bits(gx), s.bits(s.band_backward(Gr, X, m))), where
    return int(m.sum())


@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("F", F_EDGES)
def test_band_masks_bit_for_bit(eng, F, axis):
    for N in N_EDGES:
        check_band(eng, F, N, axis)


# --------------------------------------------------------------------------- rotate
def check_rotate(eng, shape, per_cell, smax, seed=0, acc=None):
    acc = {} if acc is None else acc
    X = cplx(shape, seed)
    g = torch.Generator().manual_seed(seed + 1)
    n = X.numel() if per_cell else shape[0]
    sh = (torch.rand(n, generator=g, dtype=torch.float64) * 2 - 1) * smax
    sh = sh.float().reshape(shape if per_cell else (shape[0],))
    got = eng.spec_rotate(dev(X).clone(), dev(sh)).cpu()
    ref = s.rotate(X, sh if per_cell else sh.reshape(-1, *([1] * (len(shape) - 1))))
    r = ((got.to(torch.complex128) - ref).abs() / (U * X.abs().double().clamp_min(1e-30))).max().item()
    worst(acc, "rotate", r)
    assert r <= s.C_ROT, (shape, per_cell, smax, r)
    return acc


ROTATE_CASES = [((3, 2, 33, 70), False, 3.0), ((3, 2, 33, 70), True, 3.0), ((4, 1, 17, 65), True, 1e4),
                ((4, 1, 17, 65), False, 1e4), ((3, 1, 513, 400), False, 100.0), ((3, 1, 513, 400), True, 1e4)]


@pytest.mark.parametrize("shape,per_cell,smax", ROTATE_CASES)
def test_rotate_per_cell(eng, shape, per_cell, smax):
    """|s| up to 1e4 (sincosf's range reduction); 3 x 513 x 400 cells pass the 132 x 16-CTA grid cap."""
    check_rotate(eng, shape, per_cell, smax)


# --------------------------------------------------------------------------- mask_low_magnitudes
def check_mask_low(eng, X, cut, val, where, acc=None, seed=0, max_undecided=1e-3, must_decide=None):
    """In place, out of place and the backward against the float64 decision: decided unmasked cells bit for bit,
    decided masked cells within C_KEEP u |val| of val X / |X|, undecided cells either; the gradient likewise.  Returns
    (float64 masked, undecided)."""
    acc = {} if acc is None else acc
    cut = torch.as_tensor(cut, dtype=torch.float32).reshape(-1)
    masked, und = s.mask_low_decision(X, cut)
    if must_decide is not None:
        assert not bool(und[must_decide].any()), where
    assert und.float().mean().item() <= max_undecided, (where, und.float().mean().item())
    Xd = dev(X)
    got_in = eng.spec_mask_low(Xd.clone(), dev(cut), val).cpu()
    got, ws = eng.spec_mask_low_out(Xd, dev(cut), val)
    got = got.cpu()
    assert torch.equal(s.bits(got_in), s.bits(got)), where
    assert torch.equal(s.bits(Xd), s.bits(X)), where
    same = (s.bits(got) == s.bits(X)).all(-1)
    fill = s.mask_low_value(X, val)
    e = (got.to(torch.complex128) - fill).abs() / (U * max(abs(val), 1e-30))
    near = e <= s.C_KEEP if val != 0 else (got.real == 0) & (got.imag == 0)
    assert bool(same[~masked & ~und].all()), (where, "an unmasked cell changed")
    assert bool(near[masked & ~und].all()), (where, "a masked cell is off", e[masked & ~und].max().item())
    assert bool((same | near)[und].all()), where
    if val != 0 and bool((masked & ~und).any()):
        worst(acc, "keep", e[masked & ~und].max().item())
    # the backward, from the forward's maximum
    Gr = cplx(X.shape, seed + 11)
    gx = eng.spec_mask_low_backward(dev(Gr), Xd, dev(cut), val, ws).cpu()
    zero = (X.real == 0) & (X.imag == 0)
    gz = (gx.real == 0) & (gx.imag == 0)
    assert bool(gz[zero].all()), where
    pas = (s.bits(gx) == s.bits(Gr)).all(-1)
    if val == 0:
        ok_m = gz
    else:
        want = s.mask_low_grad(Gr, X, val)
        scale = U * abs(val) * Gr.abs().double() / X.abs().double()
        eg = (gx.to(torch.complex128) - want).abs() / scale
        ok_m = eg <= s.C_MLBWD
        sel = masked & ~und & ~zero
        if bool(sel.any()):
            worst(acc, "mask_low_bwd", eg[sel].max().item())
    assert bool(pas[~masked & ~und & ~zero].all()), (where, "an unmasked gradient changed")
    assert bool(ok_m[masked & ~und & ~zero].all()), (where, "a masked gradient is off")
    assert bool((pas | ok_m)[und & ~zero].all()), where
    return masked, und


def ramped(shape, seed, lo_db=-110.0, hi_db=10.0):
    """Random phases, magnitudes log-uniform in dB [lo_db, hi_db]."""
    g = torch.Generator().manual_seed(seed)
    db = lo_db + (hi_db - lo_db) * torch.rand(shape, generator=g, dtype=torch.float64)
    ph = (torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) * math.pi
    return (10 ** (db / 20) * torch.exp(1j * ph)).to(torch.complex64)


@pytest.mark.parametrize("val", [0.0, 0.5])
@pytest.mark.parametrize("shape", [(2, 1, 33, 70), (3, 2, 17, 65), (3, 1, 513, 400)])
def test_mask_low_random(eng, shape, val):
    """Random cells over 120 dB with per-item cut-offs; 3 x 513 x 400 passes the grid cap."""
    X = ramped(shape, 1 + shape[-1])
    cut = torch.linspace(-60.0, -20.0, shape[0])  # clear of the floor near -70 dB
    check_mask_low(eng, X, cut, val, (shape, val))


def margin_cells(shape, cut, seed):
    """Cells whose dB value is cut +- 0.5 and 2 decision margins, above a loud cell that fixes the floor 80 dB lower."""
    X = ramped(shape, seed, -60.0, -1.0)
    flat = X.reshape(-1)
    flat[0] = 1.0
    n = flat.numel()
    g = torch.Generator().manual_seed(seed + 3)
    k = torch.randperm(n - 1, generator=g)[: 4 * 64] + 1
    mult = torch.tensor([-2.0, -0.5, 0.5, 2.0], dtype=torch.float64).repeat_interleave(64)
    delta = s.db_margin(cut) + s.db_margin(-80.0)  # the cell's margin and the floor's (0 dB - 80)
    db = cut + mult * delta
    ph = (torch.rand(k.numel(), generator=g, dtype=torch.float64) * 2 - 1) * math.pi
    flat[k] = (10 ** (db / 20) * torch.exp(1j * ph)).to(torch.complex64)
    two = torch.zeros(n, dtype=torch.bool)
    two[k[mult.abs() == 2.0]] = True
    return X, two.reshape(shape)


@pytest.mark.parametrize("val", [0.0, 0.5])
def test_mask_low_near_the_cutoff(eng, val):
    """Cells 2 margins from the cut-off must be decided as in float64; cells 0.5 margin away may go either way."""
    cut = -30.0
    X, two = margin_cells((1, 1, 33, 70), cut, 5)
    check_mask_low(eng, X, [cut], val, ("margin", val), max_undecided=0.06, must_decide=two)


def test_mask_low_loud_item_sets_the_floor_of_a_quiet_one(eng):
    X = torch.cat([ramped((1, 1, 33, 70), 8, -20.0, 0.0), ramped((1, 1, 33, 70), 9, -110.0, -100.0)])
    m, _ = check_mask_low(eng, X, [-200.0, -90.0], 0.5, "floor")
    assert not bool(m[1].any())  # floored at -80 dB: not below -90
    m, _ = check_mask_low(eng, X, [-200.0, -70.0], 0.5, "floor")
    assert bool(m[1].all())


def test_mask_low_all_silent(eng):
    """Every cell at amin^2: -100 dB against the floor of -180 dB."""
    X = torch.zeros((2, 1, 17, 65), dtype=torch.complex64)
    X[1] = ramped((1, 1, 17, 65), 4, -160.0, -120.0)
    m, _ = check_mask_low(eng, X, [-99.0, -101.0], 0.5, "silent")
    assert bool(m[0].all()) and not bool(m[1].any())


@pytest.mark.parametrize("cut", [float("inf"), float("-inf")])
def test_mask_low_infinite_cutoffs(eng, cut):
    X = ramped((2, 1, 33, 70), 12)
    m, _ = check_mask_low(eng, X, [cut], 0.5, ("cut", cut))
    assert bool(m.all()) if cut > 0 else not bool(m.any())


# --------------------------------------------------------------------------- gate
def gate_signal(B, C, F, N, seed):
    """A noise spectrogram around -40 dB and a signal whose dB values spread 30 dB either side of it."""
    return ramped((B, C, F, N), seed, -75.0, -5.0)


def gate_noise(shape, seed):
    return cplx(shape, seed, 0.01)


def check_gate(eng, X, nz, n_std, amount, sf, st, where, acc=None, g=None, max_undecided=1e-3):
    """Stage by stage: the thresholds against float64, S = (1 - out / X) / amount inside the float64 bracket built from
    the kernel's own thresholds, the output against X (1 - amount S); the backward with g := X bit for bit against the
    forward, with a random g against the bracket.  Returns the kernel's thresholds."""
    acc = {} if acc is None else acc
    B, C, F, N = X.shape
    amount = torch.as_tensor(amount, dtype=torch.float32).reshape(-1).expand(B).contiguous()
    out, th = eng.spec_gate(dev(X), dev(nz), n_std, dev(amount), sf, st)
    out, th = out.cpu(), th.cpu()
    # 1. thresholds
    nzb = nz if nz.shape[:2] == (1, 1) else nz.expand(B, C, -1, -1)
    want = s.thresholds(nzb, n_std)
    assert torch.equal(torch.isnan(th), torch.isnan(want)), (where, "NaN thresholds differ")
    ok = ~torch.isnan(want)
    if bool(ok.any()):
        e = ((th.double() - want).abs() / (U * s.thresh_scale(nzb, n_std)))[ok]
        worst(acc, "thresh", e.max().item())
        assert e.max().item() <= s.C_TH, (where, e.max().item())
    # 2. the smoothed mask, inside its bracket
    lo, hi, und = s.gate_bracket(X, th, sf, st)
    assert und.float().mean().item() <= max_undecided, (where, und.float().mean().item())
    a = amount.double().reshape(B, 1, 1, 1).expand(B, C, F, N)
    Xd = X.to(torch.complex128)
    fin = torch.isfinite(Xd.real) & torch.isfinite(Xd.imag) & (Xd.abs() > 0)
    sel = fin & (a > 0)
    nf, nt = len(sf), len(st)
    if bool(sel.any()):
        S = ((1 - out.to(torch.complex128) / Xd).real / a)[sel]
        d = torch.maximum(lo[sel] - S, S - hi[sel]).clamp_min(0) / (U * s.s_scale(nf, nt, a[sel]))
        worst(acc, "S", d.max().item())
        assert d.max().item() <= s.C_S, (where, d.max().item())
    else:
        assert torch.equal(s.bits(out)[fin], s.bits(X)[fin]), where  # amount 0: the output is X
    # 3. the output (and the backward for a random g) against mul (1 - amount S)
    def excess(y, mul):
        mid = 1 - a * (lo + hi) / 2
        half = a * (hi - lo) / 2
        m = mul.to(torch.complex128)
        r = ((y.to(torch.complex128) - m * mid).abs() - m.abs() * half).clamp_min(0)
        return (r / (U * m.abs().clamp_min(1e-30) * (a * (nf + nt) + 3)))[fin]

    r = excess(out, X)
    worst(acc, "out", r.max().item())
    assert r.max().item() <= s.C_OUT, (where, r.max().item())
    gb = eng.spec_gate_backward(dev(X), dev(X), dev(th), dev(amount), sf, st).cpu()
    assert torch.equal(s.bits(gb), s.bits(out)), (where, "backward with g := X differs from the forward")
    g = cplx(X.shape, 99) if g is None else g
    gg = eng.spec_gate_backward(dev(g), dev(X), dev(th), dev(amount), sf, st).cpu()
    r = excess(gg, g)
    worst(acc, "out", r.max().item())
    assert r.max().item() <= s.C_OUT, (where, "backward", r.max().item())
    return th


def gate_case(eng, B, C, F, N, nz_shape, seed, n_std=1.0, amount=(1.0, 0.6), hf=1, ht=2, sf=None, st=None, acc=None):
    X = gate_signal(B, C, F, N, seed)
    nz = gate_noise(nz_shape, seed + 1)
    sf = _ramp(hf).tolist() if sf is None else sf
    st = _ramp(ht).tolist() if st is None else st
    return check_gate(eng, X, nz, n_std, list(amount)[:B] if len(amount) >= B else amount[0], sf, st,
                      (B, C, F, N, tuple(nz_shape), len(sf), len(st)), acc)


@pytest.mark.parametrize("F", F_EDGES)
def test_gate_tiles(eng, F):
    """1 to 17 tiles along time and 1 to 65 along frequency, with the default 3 x 5 smoothing (half-widths 2, 3)."""
    for N in N_EDGES:
        gate_case(eng, 2, 2, F, N, (1, 1, F, 50), F + N, hf=3, ht=5)


@pytest.mark.parametrize("hf", HALVES)
def test_gate_smoothing_widths(eng, hf):
    """SpectralGate(n_freq, n_time) for every pair of {0, 1, 3, 5, 8}: halos up to G_MAXH = 8 at the tile edges."""
    for ht in HALVES:
        for F, N in ((33, 130), (16, 64), (17, 65)):
            gate_case(eng, 2, 1, F, N, (1, 1, F, 50), 3 * hf + ht + F, hf=hf, ht=ht)


@pytest.mark.parametrize("F,N", [(33, 130), (17, 65), (1025, 257)])
def test_gate_asymmetric_smoothing_orientation(eng, F, N):
    """conv2d is a cross-correlation: asymmetric odd vectors tell it from a convolution."""
    gate_case(eng, 2, 2, F, N, (1, 1, F, 50), 21, sf=ASYM_F, st=ASYM_T)
    gate_case(eng, 2, 2, F, N, (1, 1, F, 50), 22, sf=ASYM_T, st=ASYM_F)


@pytest.mark.parametrize("nz_shape", [(1, 1), (3, 1), (1, 2), (3, 2)])
def test_gate_noise_shapes(eng, nz_shape):
    gate_case(eng, 3, 2, 33, 130, nz_shape + (33, 50), 31, amount=(1.0, 0.3, 0.8))


@pytest.mark.parametrize("nz_N", NZ_FRAMES)
def test_gate_noise_frames(eng, nz_N):
    """ceil(N / 32) values per lane; one frame gives NaN thresholds (torch.std) and gates nothing."""
    th = gate_case(eng, 2, 2, 33, 130, (2, 2, 33, nz_N), 40 + nz_N, n_std=1.5)
    assert bool(torch.isnan(th).all()) == (nz_N == 1)


@pytest.mark.parametrize("amount", [(0.0,), (1.0,), (0.25, 1.0)])
def test_gate_amounts(eng, amount):
    gate_case(eng, 2, 1, 33, 130, (1, 1, 33, 50), 50, amount=amount)


def test_gate_silent_noise_and_signal(eng):
    """Silent noise and a signal below 1e-4 both sit at -80 dB exactly: the strict < gates nothing."""
    X = ramped((2, 1, 33, 70), 60, -200.0, -90.0)
    nz = torch.zeros((1, 1, 33, 50), dtype=torch.complex64)
    out, th = eng.spec_gate(dev(X), dev(nz), 3.0, dev(torch.tensor([1.0, 1.0])), _ramp(3).tolist(), _ramp(5).tolist())
    assert bool((th.cpu() == -80.0).all())
    assert torch.equal(s.bits(out), s.bits(X))


# --------------------------------------------------------------------------- non-finite input
NONFINITE = [("signal", float("nan")), ("signal", float("inf")), ("signal", float("-inf")),
             ("noise", float("nan")), ("noise", float("inf")), ("noise", float("-inf"))]


def plant(X, cells, value, imag=False):
    X = X.clone()
    r = torch.view_as_real(X)
    for c in cells:
        r[c + (1 if imag else 0,)] = value
    return X


def check_gate_nonfinite(eng, where, value, acc=None):
    """NaN / inf cells against the reference's arithmetic in float64: the thresholds' NaN pattern, every finite cell
    inside its bracket, and every cell's factor the reference's.  A NaN cell is never below a threshold, an inf cell
    never either; a NaN or inf noise cell makes its bin's threshold NaN (mean of inf minus inf), and that bin gates
    nothing."""
    B, C, F, N = 2, 1, 33, 70
    X = gate_signal(B, C, F, N, 70)
    nz = gate_noise((1, 1, F, 40), 71)
    cells = [(0, 0, 7, 3), (1, 0, 20, 35), (1, 0, 0, 0), (0, 0, 32, 69)]
    if where == "signal":
        X = plant(X, cells, value)
        X = plant(X, [(0, 0, 12, 40)], value, imag=True)
    else:
        nz = plant(nz, [(0, 0, 7, 3), (0, 0, 20, 39)], value)
    sf, st = _ramp(3).tolist(), _ramp(5).tolist()
    amount = torch.tensor([0.5, 0.75])
    th = check_gate(eng, X, nz, 2.0, amount, sf, st, (where, value), acc)
    out = eng.spec_gate(dev(X), dev(nz), 2.0, dev(amount), sf, st)[0].cpu()
    # the reference's factor, from its own thresholds, applied part by part
    fac = s.reference_gate(X, nz, 2.0, amount, sf, st)
    lo, hi, _ = s.gate_bracket(X, th, sf, st)
    a = amount.double().reshape(B, 1, 1, 1)
    assert bool(((fac >= 1 - a * hi - 1e-12) & (fac <= 1 - a * lo + 1e-12)).all()), (where, value)
    want = torch.complex(X.real.double() * fac, X.imag.double() * fac)
    for part in (lambda t: t.real, lambda t: t.imag):
        w, o = part(want), part(out).double()
        assert torch.equal(torch.isnan(o), torch.isnan(w)), (where, value)
        assert torch.equal(torch.isinf(o) & (o > 0), torch.isinf(w) & (w > 0)), (where, value)
        assert torch.equal(torch.isinf(o) & (o < 0), torch.isinf(w) & (w < 0)), (where, value)
    if where == "noise":
        assert bool(torch.isnan(th[0, [7, 20]]).all()) and not bool(torch.isnan(th[0, :7]).any())


@pytest.mark.parametrize("where,value", NONFINITE)
def test_gate_nonfinite(eng, where, value):
    check_gate_nonfinite(eng, where, value)


MASK_LOW_NONFINITE = [float("nan"), -float("nan"), float("inf"), float("-inf")]


def check_mask_low_nonfinite(eng, value, imag):
    """One NaN (either sign bit) or inf part anywhere in the batch: log_spec.max() is NaN or +inf, so the floor is too
    and nothing is below any cut-off, +inf included."""
    X = ramped((2, 1, 33, 70), 80)
    X = plant(X, [(1, 0, 30, 60)], value, imag)
    for cut in ([-40.0, -40.0], [float("inf"), 0.0]):
        for val in (0.0, 0.5):
            got = eng.spec_mask_low(dev(X).clone(), dev(torch.tensor(cut)), val).cpu()
            assert torch.equal(s.bits(got), s.bits(X)), (value, imag, cut, val)
            out, ws = eng.spec_mask_low_out(dev(X), dev(torch.tensor(cut)), val)
            assert torch.equal(s.bits(out), s.bits(X)), (value, imag, cut, val)
            Gr = cplx(X.shape, 81)
            gx = eng.spec_mask_low_backward(dev(Gr), dev(X), dev(torch.tensor(cut)), val, ws).cpu()
            assert torch.equal(s.bits(gx), s.bits(Gr)), (value, imag, cut, val)
    masked, _ = s.mask_low_decision(X, torch.tensor([-40.0, -40.0]))
    assert not bool(masked.any())


@pytest.mark.parametrize("imag", [False, True])
@pytest.mark.parametrize("value", MASK_LOW_NONFINITE, ids=["nan", "-nan", "inf", "-inf"])
def test_mask_low_nonfinite(eng, value, imag):
    check_mask_low_nonfinite(eng, value, imag)


# --------------------------------------------------------------------------- limits
def stream_of(t):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream) if t.is_cuda else None


def check_refusals(eng):
    """Refused shapes return their error code before any launch (buffers of a few cells are never read)."""
    lib = eng.lib
    buf = torch.zeros(64, dtype=torch.complex64, device=DEV)
    fl = torch.zeros(64, dtype=torch.float32, device=DEV)
    p, q, st = ctypes.c_void_p(buf.data_ptr()), ctypes.c_void_p(fl.data_ptr()), stream_of(buf)
    ok3 = (ctypes.c_float * 3)(1.0, 1.0, 1.0)
    l19 = (ctypes.c_float * 19)(*([1.0] * 19))
    out = torch.zeros(64, dtype=torch.complex64, device=DEV)
    o = ctypes.c_void_p(out.data_ptr())
    n0 = lib.kernel_launches.value

    def gate(rows, n_f, n_t, sf, stv):
        return lib.b2a_spec_gate_f32(p, rows, 1, 1, p, 1, 4, 1.0, q, 1, sf, n_f, stv, n_t, o, q, st)

    def gate_bwd(rows, n_f, n_t, sf, stv):
        return lib.b2a_spec_gate_backward_f32(p, p, rows, 1, 1, q, 1, q, 1, sf, n_f, stv, n_t, o, st)

    assert gate(65536, 3, 3, ok3, ok3) == -1
    assert gate_bwd(65536, 3, 3, ok3, ok3) == -1
    assert gate(1, 19, 3, l19, ok3) == -2 and gate(1, 3, 19, ok3, l19) == -2
    assert gate_bwd(1, 19, 3, l19, ok3) == -2 and gate_bwd(1, 3, 19, ok3, l19) == -2
    lines = 2 ** 31
    assert lib.b2a_spec_band_mask_f32(p, lines, 1, 1, q, q, q, 1, 0, 0.0, 0.0, st) == -2
    assert lib.b2a_spec_band_mask_out_f32(p, o, lines, 1, 1, q, q, q, 1, 1, 0.0, 0.0, st) == -2
    assert lib.b2a_spec_band_mask_backward_f32(p, p, lines, 1, 1, q, q, q, 1, 0, o, st) == -2
    assert lib.kernel_launches.value == n0


def test_refusals_before_any_launch(eng):
    check_refusals(eng)


def test_gate_accepts_65535_rows(eng):
    X = gate_signal(65535, 1, 3, 5, 90)
    nz = gate_noise((1, 1, 3, 50), 91)
    check_gate(eng, X, nz, 1.0, 0.8, _ramp(1).tolist(), _ramp(2).tolist(), "65535 rows", max_undecided=2e-3)


def check_reruns(eng):
    X = dev(ramped((3, 2, 33, 130), 95))
    nz = dev(gate_noise((1, 1, 33, 50), 96))
    cut, amt = dev(torch.tensor([-60.0, -40.0, -20.0])), dev(torch.tensor([1.0, 0.5, 0.25]))
    sh = dev(torch.linspace(-50, 50, X.numel()).reshape(X.shape))
    v = dev(torch.linspace(0, 8000.0, 33))
    lo, hi = dev(torch.tensor([100.0, 2000.0, 0.0])), dev(torch.tensor([900.0, 2500.0, 8000.0]))
    runs = []
    for _ in range(2):
        r = [eng.spec_rotate(X.clone(), sh), eng.spec_mask_low(X.clone(), cut, 0.5), eng.spec_mask_low_out(X, cut, 0.5)[0],
             eng.spec_gate(X, nz, 1.0, amt, ASYM_F, ASYM_T)[0], eng.spec_band_mask_out(X, v, lo, hi, 0, 0.3)]
        runs.append([s.bits(t) for t in r])
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_reruns_bit_identical(eng):
    check_reruns(eng)


def big_case(eng, op):
    """One call past 2^31 cells (2 items of 1025 x 1 047 553), checked on a strided subset and the last row."""
    F, N = 1025, 1_047_553
    total = 2 * F * N
    assert total > 2 ** 31
    need = total * 8 + (2 << 30)
    if torch.cuda.mem_get_info()[0] < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory")
    X = torch.empty((2, 1, F, N), dtype=torch.complex64, device=DEV)
    torch.view_as_real(X).uniform_(-0.5, 0.5, generator=torch.Generator(DEV).manual_seed(7))
    flat = X.view(-1)
    flat[-1] = 40.0  # the loudest cell is the last one: the floor depends on the top index
    idx = torch.cat([torch.arange(0, total, 104_729, device=DEV), torch.arange(total - N, total, device=DEV)])
    x0 = flat[idx].cpu()
    if op == "rotate":
        sh = torch.tensor([0.75, -2.5])
        eng.spec_rotate(X, dev(sh))
        got = flat[idx].cpu()
        item = (idx.cpu() >= F * N).long()
        ref = s.rotate(x0, sh[item])
        r = ((got.to(torch.complex128) - ref).abs() / (U * x0.abs().double().clamp_min(1e-30))).max().item()
        assert r <= s.C_ROT, r
    else:
        cut = torch.tensor([-20.0, -6.0])
        eng.spec_mask_low(X, dev(cut), 0.5)
        got = flat[idx].cpu()
        item = (idx.cpu() >= F * N).long()
        p = x0.to(torch.complex128).abs() ** 2
        floor = 10 * math.log10(1600.0) - 80.0
        dbf = torch.maximum(10 * torch.log10(p.clamp_min(1e-10)), torch.tensor(floor))
        c = cut.double()[item]
        masked = dbf < c
        und = (dbf - c).abs() <= torch.from_numpy(2 * s.db_margin(dbf.numpy()))
        same = (s.bits(got) == s.bits(x0)).all(-1)
        near = (got.to(torch.complex128) - s.mask_low_value(x0, 0.5)).abs() <= s.C_KEEP * U * 0.5
        assert bool(same[~masked & ~und].all()) and bool(near[masked & ~und].all())
        assert bool(masked[item == 1].any()) and bool((~masked).any())
    del X, flat
    torch.cuda.empty_cache()


@pytest.mark.parametrize("op", ["rotate", "mask_low"])
def test_past_2_31_cells(eng, op):
    big_case(eng, op)
