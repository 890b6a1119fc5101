"""metrics.LoudnessLoss and b2a_lufs_backward_f32 (DESIGN.md K21) on the H100 against the float64 oracle
(tests/loudness_grad64.py): the gradient per (row, 100 ms interval) at or below the sequential float32 cascade's error
or under a floor, at every rate, channel count and length edge; items clamped at -70, silent or non-finite; a deferred
gain; batch-versus-single bit identity; the loss equal to ``loudness()``'s numbers; launch counts; refusals; and an
end-to-end property (a per-item gain trained to -23 LUFS).  tests/test_sim_loudness_grad.py runs the same checks on the
CPU-simulated kernels, at smaller sizes."""
import numpy as np
import pytest
import torch

from audiotools_b200 import AudioSignal
from audiotools_b200.core import grad as _grad
from audiotools_b200.engine import get_engine
from audiotools_b200.metrics import LoudnessLoss
from tests import loudness_grad64 as lg

DEV = "cuda"
RATIO = 1.0      # the kernel's worst interval against the float32 baseline's
FLOOR = 128.0    # u = 2^-24 of the interval's RMS: passes whatever the baseline does

RATES = (16000, 22050, 44100, 48000, 11025)


def signals(rate, C, T, seed=0):
    """[4, C, T] float32: noise; noise whose second half is 30 dB down (under the relative gate); a 50 Hz sine with
    noise (the high-pass's band); noise with a 20 dB swell."""
    rng = np.random.default_rng(seed)
    t = np.arange(T) / rate
    x = np.empty((4, C, T))
    x[0] = 0.1 * rng.standard_normal((C, T))
    x[1] = 0.1 * rng.standard_normal((C, T)) * np.where(t < t[-1] / 2, 1.0, 0.03)
    x[2] = 0.3 * np.sin(2 * np.pi * 50 * t + rng.uniform(0, 6, (C, 1))) + 0.01 * rng.standard_normal((C, T))
    x[3] = 0.05 * rng.standard_normal((C, T)) * (1 + 9 * np.exp(-((t - t[-1] / 3) / 0.05) ** 2))
    return x.astype(np.float32)


def loss_grad(x, rate, target=-100.0, reduction="sum", gain=None):
    """(loss, grad x) through LoudnessLoss on DEV; ``gain`` [B]: a normalize-style gain deferred before the call."""
    xt = torch.from_numpy(x).to(DEV)
    sig = AudioSignal(xt, rate)
    if gain is not None:
        gt = torch.as_tensor(gain, dtype=torch.float32, device=DEV)
        if xt.is_cuda:
            with torch.no_grad():
                sig._defer_gain(gt)  # deferred; _materialized() applies it differentiably once x requires a gradient
        else:  # a CPU signal is scaled at once (no deferral): the same chain rule, through torch
            sig = AudioSignal(xt.requires_grad_(True) * gt[:, None, None], rate)
    xt.requires_grad_(True)
    loss = LoudnessLoss(reduction=reduction)(sig, target)
    loss.sum().backward()
    return loss.detach(), xt.grad.cpu().numpy()


def check_accuracy(rate, C, T, seed=0):
    x = signals(rate, C, T, seed)
    Tp = lg.padded_length(T, rate)
    _, g = loss_grad(x, rate)  # target -100: the loss is sum(loud + 100), dL/dloud = 1
    fw = lg.forward64(x, rate, Tp)
    assert (fw["lufs"] > -70).all()
    ref = lg.grad64(x, rate, Tp, fw=fw)
    base = lg.baseline32(x, rate, Tp, fw=fw)
    skip = lg.near_gate_mask(fw, T, rate)
    e, eb = lg.interval_error(g, ref, rate, skip), lg.interval_error(base, ref, rate, skip)
    assert np.isfinite(g).all()
    assert (e <= np.maximum(RATIO * eb, FLOOR)).all(), (e, eb)
    return e, eb


@pytest.mark.gpu
@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("C", [1, 2, 5])
def test_gradient_against_float64(rate, C):
    check_accuracy(rate, C, int(1.3 * rate) + 77)  # not a multiple of the stride


@pytest.mark.gpu
@pytest.mark.parametrize("rate", RATES)
def test_short_rows_are_zero_extended(rate):
    check_accuracy(rate, 2, int(0.3 * rate) + 5)  # T < 0.5 s: the adjoint runs over the zero extension too


def check_tail_under_relative_gate(rate):
    fw = lg.forward64(signals(rate, 1, 2 * rate), rate)
    keep = fw["keep"][1]
    assert keep[:5].all() and not keep[-5:].any()  # item 1's tail is gated out: m[t] = 0 there
    check_accuracy(rate, 1, 2 * rate)


@pytest.mark.gpu
def test_tail_under_relative_gate():
    check_tail_under_relative_gate(44100)


def check_silent_clamped_and_nan(rate):
    T = rate
    x = signals(rate, 2, T)
    x[0] = 0.0                                                            # silent: lufs = -inf
    x[1] = 1e-5 * np.random.default_rng(1).standard_normal((2, T))        # about -90 LUFS: clamped at -70
    x[2, 1, T // 3] = np.nan
    loss, g = loss_grad(x, rate)
    fw = lg.forward64(np.nan_to_num(x), rate)
    assert fw["lufs"][1] < -70
    assert (g[0] == 0).all() and (g[1] == 0).all()
    assert np.isnan(g[2]).all()
    _, g3 = loss_grad(x[3:], rate)
    np.testing.assert_array_equal(g[3], g3[0])  # the other items are unaffected


@pytest.mark.gpu
def test_silent_clamped_and_nan_items():
    check_silent_clamped_and_nan(16000)


def check_deferred_gain(rate):
    T = rate + 333
    x = signals(rate, 2, T)
    gain = np.array([0.5, 2.0, 1.25, 0.1], np.float32)
    _, g = loss_grad(x, rate, gain=gain)
    xs = (x * gain[:, None, None]).astype(np.float32)
    fw = lg.forward64(xs, rate)
    ref = lg.grad64(xs, rate, fw=fw) * gain[:, None, None]
    base = lg.baseline32(xs, rate, fw=fw) * gain[:, None, None]
    skip = lg.near_gate_mask(fw, T, rate)
    e, eb = lg.interval_error(g, ref, rate, skip), lg.interval_error(base, ref, rate, skip)
    assert (e <= np.maximum(RATIO * eb, FLOOR)).all(), (e, eb)
    # the engine's own gain argument gives the same gradient up to the rounding of gain into the weight
    eng = get_engine()
    xt = torch.from_numpy(x).to(DEV)
    gt = torch.from_numpy(gain).to(DEV)
    out = eng.lufs(eng.gain(xt, gt), rate, want_blocks=True)
    gx = eng.lufs_backward(torch.ones(4, device=DEV), xt, rate, out["blocks"], out["lufs"], gain=gt).cpu().numpy()
    e2 = lg.interval_error(gx, ref, rate, skip)
    assert (e2 <= np.maximum(RATIO * eb, FLOOR)).all(), (e2, eb)


@pytest.mark.gpu
def test_deferred_normalize_gain():
    check_deferred_gain(44100)


def check_batch_and_value(rate):
    T = int(0.7 * rate)
    x = signals(rate, 2, T)
    loss, g = loss_grad(x, rate, reduction="none")
    for b in range(x.shape[0]):
        _, gb = loss_grad(x[b:b + 1], rate)
        np.testing.assert_array_equal(g[b], gb[0])
    # the value: loudness() bit for bit, and |loud(est) - loud(ref)| in float32
    est = AudioSignal(torch.from_numpy(x).to(DEV), rate)
    ref = AudioSignal(torch.from_numpy(x[::-1].copy() * np.float32(0.3)).to(DEV), rate)
    xt = torch.from_numpy(x).to(DEV).requires_grad_(True)
    loud = _grad.Loudness.apply(xt, None, rate, est._padded_length())
    assert torch.equal(loud.detach(), est.loudness())
    want = (est.loudness() - ref.loudness()).abs()
    got = LoudnessLoss(reduction="none")(AudioSignal(xt, rate), ref)
    assert got.dtype == torch.float32 and torch.equal(got.detach(), want)
    assert est._loudness is not None  # est.loudness() above filled its own cache; the loss reads none
    fresh = AudioSignal(torch.from_numpy(x).to(DEV), rate)
    LoudnessLoss()(fresh, -23.0)
    assert fresh._loudness is None
    t = torch.tensor([-20.0, -21.0, -22.0, -23.0], device=DEV)
    got = LoudnessLoss(reduction="sum")(fresh, t)
    want = (fresh.loudness().double() - t.double()).abs().sum().float()
    assert torch.equal(got, want)


@pytest.mark.gpu
def test_batch_single_and_value():
    check_batch_and_value(48000)


def check_launches(rate):
    eng = get_engine()
    x = torch.from_numpy(signals(rate, 2, rate)).to(DEV)
    n0 = eng.launches
    AudioSignal(x, rate).loudness()
    n_loud = eng.launches - n0
    n0 = eng.launches
    LoudnessLoss()(AudioSignal(x, rate), -23.0)
    assert eng.launches - n0 == n_loud == 2
    xg = x.clone().requires_grad_(True)
    n0 = eng.launches
    with torch.no_grad():
        LoudnessLoss()(AudioSignal(xg, rate), -23.0)
    assert eng.launches - n0 == n_loud
    n0 = eng.launches
    loss = LoudnessLoss()(AudioSignal(xg, rate), -23.0)
    assert eng.launches - n0 == n_loud
    n0 = eng.launches
    loss.backward()
    assert eng.launches - n0 == 7  # b2a.h: one gate kernel, two three-launch K-weighting passes


@pytest.mark.gpu
def test_launch_counts():
    check_launches(16000)


def check_refusals(rate):
    x = torch.from_numpy(signals(rate, 2, rate)).to(DEV).requires_grad_(True)
    est = AudioSignal(x, rate)
    with pytest.raises(NotImplementedError):
        LoudnessLoss()(est, AudioSignal(x * 0.5, rate))
    with pytest.raises(NotImplementedError):
        LoudnessLoss()(est, torch.tensor([-23.0], device=DEV, requires_grad=True))
    with pytest.raises(ValueError):
        LoudnessLoss()(est, AudioSignal(x.detach(), rate * 2))
    with pytest.raises(ValueError):
        LoudnessLoss()(est, AudioSignal(x.detach()[:2], rate))
    with pytest.raises(ValueError):
        LoudnessLoss()(est, [-23.0, -20.0])
    with pytest.raises(ValueError):
        LoudnessLoss()(AudioSignal(torch.zeros(1, 6, rate, device=DEV, requires_grad=True), rate), -23.0)


@pytest.mark.gpu
def test_refusals():
    check_refusals(16000)


@pytest.mark.gpu
def test_bench_batch_strided_items():
    """The bench batch (64 x 2 x 10 s at 44.1 kHz); every 9th item against float64."""
    rate, T = 44100, 441000
    rng = np.random.default_rng(3)
    x = (0.1 * rng.standard_normal((64, 2, T)) * rng.uniform(0.05, 1.0, (64, 1, 1))).astype(np.float32)
    x[::5, :, T // 2:] *= 0.02
    _, g = loss_grad(x, rate)
    idx = np.arange(0, 64, 9)
    fw = lg.forward64(x[idx], rate)
    ref = lg.grad64(x[idx], rate, fw=fw)
    base = lg.baseline32(x[idx], rate, fw=fw)
    skip = lg.near_gate_mask(fw, T, rate)
    e, eb = lg.interval_error(g[idx], ref, rate, skip), lg.interval_error(base, ref, rate, skip)
    assert (e <= np.maximum(RATIO * eb, FLOOR)).all(), (e, eb)


@pytest.mark.gpu
def test_adam_trains_a_gain_to_the_target():
    rate = 44100
    x = torch.from_numpy(signals(rate, 2, 2 * rate)).to(DEV)
    g = torch.nn.Parameter(torch.ones(4, device=DEV))
    opt = torch.optim.Adam([g], lr=0.05)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, 0.985)
    loss_fn = LoudnessLoss()
    for _ in range(400):
        opt.zero_grad()
        loss = loss_fn(AudioSignal(x * g[:, None, None], rate), -23.0)
        loss.backward()
        opt.step()
        sched.step()
    with torch.no_grad():
        loud = AudioSignal(x * g[:, None, None], rate).loudness()
    assert (loud + 23.0).abs().max().item() < 0.05, loud
