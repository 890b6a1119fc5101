"""Gradients through resample, equalizer, convolve, apply_ir, ensure_max_of_audio, mix and the quantisers on the
CPU-simulated build of the kernels (tests/cusim): against torch.autograd over the reference's arithmetic in float64
(tests/effects_grad_cases.py), the adjoint identity of every route, the masked (bypass) forms, the no-gradient path's
launches, and the methods that still raise."""
import os
import subprocess
import sys

import pytest
import torch

import audiotools_b200.engine as engine_mod
from audiotools_b200 import AudioSignal
from tests import effects_grad_cases as ec
from tests.conftest import elementwise_ok, rel_err
from tests.cusim.sim_engine import sim_engine

TOL = 1e-4
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def sim_signals(monkeypatch):
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    yield sim_engine()


def _check(method, shape, seed, sr=44100, **kw):
    x = ec.x_of(shape, seed)
    y = ec.ours(method, sr, **kw)(x)
    g = ec.x_of(y.shape, seed + 1, 1.0)
    gx = ec.vjp(ec.ours(method, sr, **kw), x, g)
    want = ec.vjp(ec.ref(method, sr, **kw), x.double(), g)
    assert rel_err(gx, want) < TOL, (method, rel_err(gx, want))
    assert elementwise_ok(gx, want, frame_dim=-1)
    return gx, want


@pytest.mark.parametrize("old,new", ec.RESAMPLE_RATES)
@pytest.mark.parametrize("T", ec.RESAMPLE_LENGTHS)
def test_resample_grad_matches_autograd(sim_signals, old, new, T):
    """Both forward routes (polyphase; the decimating FIR when the reduced new rate is 1), down and up, with T below
    the filter's half width and below its length: the replicate fold lands in gx[0] and gx[T-1]."""
    _check("resample", (2, 2, T), T + old, sr=old, new_sr=new)


@pytest.mark.parametrize("old,new,T", [(16000, 44100, 1), (16000, 44100, 2), (11025, 96000, 700)])
def test_resample_grad_tiny_rows_and_large_new_rate(sim_signals, old, new, T):
    """T = 1 (every extended position folds into gx[0]) and T = 2 (no interior samples) when upsampling, and a reduced
    new rate (147 -> 1280) whose frames are staged in phase tiles."""
    _check("resample", (2, 2, T), T + old, sr=old, new_sr=new)
    eng = sim_signals
    _adjoint(lambda v: eng.resample(v, old, new), lambda g: eng.resample_backward(g, T, old, new),
             ec.x_of((1, 2, T), T), None, 1)


def test_grads_match_reference_golden(sim_signals):
    """Every case of tests/golden/make_golden_effects_grad.py against the REAL reference's gradients."""
    ec.check_golden(ec.load_golden(), "cpu")


def test_in_place_change_of_a_saved_ir_is_caught(sim_signals):
    ir = ec.synthetic_ir(2, 300, 1)
    xg = ec.x_of((2, 1, 1000), 2).requires_grad_()
    y = AudioSignal(xg, 44100).convolve(AudioSignal(ir, 44100)).audio_data
    ir.mul_(2.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        y.sum().backward()


@pytest.mark.parametrize("T", ec.EQ_LENGTHS)
@pytest.mark.parametrize("per_item", [False, True])
def test_equalizer_grad_matches_autograd(sim_signals, T, per_item):
    db = ec.db_curve(2 if per_item else 1, 6, T)
    _check("equalizer", (2, 2, T), T, db=db)


def test_single_band_equalizer_is_a_gain(sim_signals):
    _check("equalizer", (2, 1, 500), 3, db=torch.tensor([[2.0], [-3.0]]))


@pytest.mark.parametrize("L,T,B_ir,start", [(300, 2000, 2, True), (3000, 2000, 2, True), (300, 2000, 1, True),
                                            (300, 2000, 2, False)])
def test_convolve_grad_matches_autograd(sim_signals, L, T, B_ir, start):
    """An IR shorter than the signal, one longer (truncated), a batch-1 IR, and no roll to the peak."""
    _check("convolve", (2, 2, T), L + T, ir=ec.synthetic_ir(B_ir, L, L), start_at_max=start)


@pytest.mark.parametrize("L", [300, 3000])
def test_apply_ir_grad_matches_autograd(sim_signals, L):
    _check("apply_ir", (2, 2, 2000), L, ir=ec.synthetic_ir(2, L, L + 1))


def test_ensure_max_of_audio_grad(sim_signals):
    """One row above max (scaled: the peak's own gradient term), one below (identity)."""
    x = ec.x_of((2, 2, 1000), 5)
    x[0] *= 4
    x[1] *= 0.3
    g = ec.x_of(x.shape, 6, 1.0)
    gx = ec.vjp(ec.ours("ensure_max_of_audio", max=1.0), x, g)
    want = ec.vjp(ec.ref("ensure_max_of_audio", max=1.0), x.double(), g)
    assert rel_err(gx, want) < TOL and torch.equal(gx[1], g[1])


def test_mix_grads(sim_signals):
    """d/dself = identity; d/dother = the noise's loudness-normalisation gain (a constant, as in normalize), also
    through an equalised `other`."""
    x, n = ec.x_of((2, 1, 8000), 7), ec.x_of((2, 1, 8000), 8)
    xg, ng = x.clone().requires_grad_(), n.clone().requires_grad_()
    out = AudioSignal(xg, 16000).mix(AudioSignal(ng, 16000), snr=torch.tensor([10.0, 3.0]))
    g = ec.x_of(out.audio_data.shape, 9, 1.0)
    gx, gn = torch.autograd.grad((out.audio_data * g).sum(), (xg, ng))
    assert torch.equal(gx, g)
    with torch.no_grad():
        n2 = AudioSignal(n.clone(), 16000)
        ref = AudioSignal(x.clone(), 16000).mix(n2, snr=torch.tensor([10.0, 3.0])).audio_data
    gain = (ref - x)[:, 0, 100] / n[:, 0, 100]
    assert rel_err(gn, g * gain[:, None, None]) < 1e-5

    db = ec.db_curve(1, 6, 10)
    ng = n.clone().requires_grad_()
    out = AudioSignal(x.clone(), 16000).mix(AudioSignal(ng, 16000), snr=5.0, other_eq=db)
    (gn,) = torch.autograd.grad((out.audio_data * g).sum(), ng)
    assert gn.abs().sum() > 0 and torch.isfinite(gn).all()
    with pytest.raises(NotImplementedError, match="snr requires a gradient"):
        AudioSignal(xg, 16000).mix(AudioSignal(n, 16000), snr=torch.tensor(10.0, requires_grad=True))


@pytest.mark.parametrize("mulaw", [False, True])
def test_quantization_is_straight_through(sim_signals, mulaw):
    x = ec.x_of((2, 1, 500), 11)
    xg = x.clone().requires_grad_()
    s = AudioSignal(xg, 16000)
    out = (s.mulaw_quantization(32) if mulaw else s.quantization(32)).audio_data
    with torch.no_grad():
        s0 = AudioSignal(x.clone(), 16000)
        want = (s0.mulaw_quantization(32) if mulaw else s0.quantization(32)).audio_data
    assert torch.equal(out.detach(), want)
    g = ec.x_of(x.shape, 12, 1.0)
    (gx,) = torch.autograd.grad((out * g).sum(), xg)
    assert torch.equal(gx, g)


def _adjoint(A, AT, x, gshape, seed):
    y = A(x)
    g = ec.x_of(gshape or y.shape, seed, 1.0)
    gx = AT(g)
    lhs, rhs = (y.double() * g.double()).sum().item(), (x.double() * gx.double()).sum().item()
    scale = (y.double().abs() * g.double().abs()).sum().item()
    assert abs(lhs - rhs) <= 1e-5 * scale, (lhs, rhs)


@pytest.mark.parametrize("old,new", ec.RESAMPLE_RATES)
@pytest.mark.parametrize("T", [7, 1000])
def test_resample_adjoint_identity(sim_signals, old, new, T):
    eng = sim_signals
    _adjoint(lambda v: eng.resample(v, old, new), lambda g: eng.resample_backward(g, T, old, new),
             ec.x_of((1, 2, T), T), None, 1)


@pytest.mark.parametrize("per_item,bypass", [(False, None), (True, None), (True, [1, 0])])
def test_equalizer_adjoint_identity(sim_signals, per_item, bypass):
    eng = sim_signals
    db = ec.db_curve(2 if per_item else 1, 6, 3)
    _adjoint(lambda v: eng.equalizer(v, 44100, db, bypass=bypass),
             lambda g: eng.equalizer_backward(g, 44100, db, bypass=bypass), ec.x_of((2, 2, 900), 4), None, 2)


@pytest.mark.parametrize("B_ir,C_ir,roll,bypass", [(2, 1, True, None), (2, 1, False, None), (1, 1, True, None),
                                                   (2, 2, True, None), (2, 1, True, [0, 1]), (1, 1, True, [1, 0])])
def test_convolve_adjoint_identity(sim_signals, B_ir, C_ir, roll, bypass):
    """Per-item, shared (batch-1) and per-channel IRs, roll on / off, bypass flags."""
    eng = sim_signals
    ir = ec.synthetic_ir(B_ir, 700, 5, C=C_ir)
    _adjoint(lambda v: eng.circular_convolve(v, ir, roll_to_peak=roll, bypass=bypass),
             lambda g: eng.circular_convolve_backward(g, ir, roll_to_peak=roll, bypass=bypass),
             ec.x_of((2, 2, 1500), 6), None, 3)


def test_fir_pad_fold_short_rows(sim_signals):
    """The replicate fold for T < K and for per-filter offsets, against autograd through F.pad(mode="replicate")."""
    eng = sim_signals
    K = 41
    taps = ec.x_of((2, K), 1)
    left = torch.tensor([20, 7], dtype=torch.int32)
    for T in (1, 5, 30, 200):
        g = ec.x_of((2, T), T, 1.0)
        gx = eng.fir_pad_fold(g, taps, rows_per_filt=1, left=left, grad_x=torch.zeros(2, T))

        def ext(v, f):
            # the padded positions only: y[m] = sum_k h[k] xv[m + k - l] minus its zero-padded part
            lf = int(left[f])
            xv = torch.nn.functional.pad(v[None, None], (lf, K - 1 - lf), mode="replicate")[0, 0]
            xz = torch.nn.functional.pad(v, (lf, K - 1 - lf))
            h = taps[f].double()
            return torch.stack([(h * (xv[m:m + K] - xz[m:m + K])).sum() for m in range(T)])

        for f in range(2):
            want = ec.vjp(lambda v: ext(v, f), torch.zeros(T, dtype=torch.float64), g[f])
            assert rel_err(gx[f], want) < 1e-5, T


@pytest.mark.parametrize("method", ["equalizer", "apply_ir", "convolve"])
def test_bypass_items_get_the_identity_gradient(sim_signals, method):
    """_bypass inside a grad graph on a non-leaf signal: unselected items get exactly g, selected ones the gradient
    of the effect."""
    kw = {"equalizer": dict(db=ec.db_curve(2, 6, 1)), "apply_ir": dict(ir=ec.synthetic_ir(2, 300, 2)),
          "convolve": dict(ir=ec.synthetic_ir(2, 300, 3))}[method]
    bypass = torch.tensor([True, False])
    x = ec.x_of((2, 2, 1500), 13)
    g = ec.x_of(x.shape, 14, 1.0)
    gx = ec.vjp(lambda v: ec.ours(method, bypass=bypass, **kw)(v * 1.0), x, g)
    want = ec.vjp(lambda v: ec.bypassed(ec.ref(method, **kw), v, bypass), x.double(), g)
    assert torch.equal(gx[0], g[0])
    assert rel_err(gx[1], want[1]) < TOL


@pytest.mark.parametrize("name", ["Equalizer", "RoomImpulseResponse"])
@pytest.mark.parametrize("flags", [False, True])
def test_masked_transforms_in_a_grad_graph(sim_signals, name, flags):
    """The data transforms with prob 0.5 on a non-leaf signal: unselected items get exactly g, whichever path
    the transform takes (gather / scatter through torch indexing, or the kernels' bypass flags)."""
    from audiotools_b200.data import transforms as tfm

    B, sr = 5, 16000
    x = ec.x_of((B, 2, 4000), 15, 0.1)
    if name == "Equalizer":
        t = tfm.Equalizer(prob=0.5)
    else:
        irs = [AudioSignal(ec.synthetic_ir(1, 800, 20 + i), sr) for i in range(2)]
        t = tfm.RoomImpulseResponse(sources=irs, prob=0.5)
    if flags:
        t._mask_aware, t._bypass_ok = True, (lambda *a: True)
    xg = x.clone().requires_grad_()
    sig = AudioSignal(xg * 1.0, sr)
    kw = t.batch_instantiate(list(range(B)), AudioSignal(x.clone(), sr))
    mask = kw[t.name]["mask"]
    assert 0 < int(mask.sum()) < B
    out = t(sig, **kw).audio_data
    g = ec.x_of(out.shape, 16, 1.0)
    (gx,) = torch.autograd.grad((out * g).sum(), xg)
    for b in range(B):
        if not bool(mask[b]):
            assert torch.equal(gx[b], g[b]), b
        else:
            assert not torch.equal(gx[b], g[b]), b


def test_no_grad_path_is_unchanged(sim_signals, monkeypatch):
    """Without a gradient the effects never enter the new Functions and make the same launches, with the same
    outputs, in grad mode as under torch.no_grad()."""
    from audiotools_b200.core import grad as _grad

    def refuse(*a, **k):
        raise AssertionError("autograd Function used without a gradient")

    for f in (_grad.Resample, _grad.Equalizer, _grad.CircConv, _grad.PeakScale, _grad.Mix, _grad.StraightThrough):
        monkeypatch.setattr(f, "apply", refuse)
    eng = sim_signals
    x = ec.x_of((2, 1, 3000), 31)
    ir = ec.synthetic_ir(2, 400, 32)

    def run():
        n0 = eng.launches
        outs = [AudioSignal(x.clone(), 44100).resample(16000).audio_data,
                AudioSignal(x.clone(), 48000).resample(16000).audio_data,
                AudioSignal(x.clone(), 44100).equalizer(ec.db_curve(2, 6, 1)).audio_data,
                AudioSignal(x.clone(), 44100).convolve(AudioSignal(ir, 44100)).audio_data,
                AudioSignal(x.clone(), 44100).apply_ir(AudioSignal(ir, 44100)).audio_data,
                AudioSignal(x.clone() * 3, 44100).ensure_max_of_audio().audio_data,
                AudioSignal(x.clone(), 44100).mix(AudioSignal(x.flip(-1), 44100), snr=5.0).audio_data,
                AudioSignal(x.clone(), 44100).quantization(16).audio_data,
                AudioSignal(x.clone(), 44100).mulaw_quantization(16).audio_data]
        return eng.launches - n0, outs

    n_grad_mode, a = run()
    with torch.no_grad():
        n_no_grad, b = run()
    assert n_grad_mode == n_no_grad
    for u, v in zip(a, b):
        assert u.grad_fn is None and torch.equal(u, v)


def test_out_of_scope_still_raises(sim_signals):
    xg = ec.x_of((2, 1, 3000), 41).requires_grad_()
    with pytest.raises(NotImplementedError, match="sinc_filter.*requires a gradient.*mel_spectrogram"):
        AudioSignal(xg, 16000).low_pass(2000)
    with pytest.raises(NotImplementedError, match="requires a gradient"):
        AudioSignal(xg, 16000).mel_filterbank(4)
    with pytest.raises(NotImplementedError, match="requires a gradient"):
        AudioSignal(xg, 16000).clip_distortion(0.1)
    with pytest.raises(NotImplementedError, match="db requires a gradient"):
        AudioSignal(xg, 44100).equalizer(torch.zeros(1, 6, requires_grad=True))
    with pytest.raises(NotImplementedError, match="impulse response requires a gradient"):
        AudioSignal(xg, 44100).convolve(AudioSignal(ec.synthetic_ir(2, 100, 1).requires_grad_(), 44100))


_SHUFFLED = r"""
import sys, torch
sys.path.insert(0, sys.argv[1])
import audiotools_b200.engine as em
from tests import effects_grad_cases as ec
from tests.conftest import rel_err
from tests.cusim.sim_engine import sim_engine
em._ENGINE = sim_engine()
cases = [("resample", 44100, dict(new_sr=16000)), ("resample", 44100, dict(new_sr=22050)),
         ("resample", 16000, dict(new_sr=44100)), ("equalizer", 44100, dict(db=ec.db_curve(2, 6, 1))),
         ("convolve", 44100, dict(ir=ec.synthetic_ir(2, 300, 2))), ("apply_ir", 44100, dict(ir=ec.synthetic_ir(2, 300, 3))),
         ("ensure_max_of_audio", 44100, dict(max=0.5))]
for method, sr, kw in cases:
    x = ec.x_of((2, 2, 1200), 1)
    g = ec.x_of(ec.ours(method, sr, **kw)(x).shape, 2, 1.0)
    gx = ec.vjp(ec.ours(method, sr, **kw), x, g)
    want = ec.vjp(ec.ref(method, sr, **kw), x.double(), g)
    assert rel_err(gx, want) < 1e-4, (method, rel_err(gx, want))
print("ok")
"""


@pytest.mark.parametrize("seed", ["1", "2", "3"])
def test_effect_grad_kernels_under_shuffled_fiber_order(seed):
    """The simulator visits the CUDA threads of a block in a random order under CUSIM_SHUFFLE: a missing barrier that
    the fixed order happens to satisfy shows up as a wrong result.  (Read once per process: run in a child.)"""
    env = dict(os.environ, CUSIM_SHUFFLE=seed)
    r = subprocess.run([sys.executable, "-c", _SHUFFLED, REPO], env=env, cwd=REPO, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
