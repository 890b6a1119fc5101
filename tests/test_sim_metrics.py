"""audiotools_b200.metrics on the CPU-simulated build of the kernels (tests/cusim): the fused spectral losses of
csrc/loss.cu against the real reference's goldens and float64, the selection between the fused and the composed path,
and the exact properties (loss(x, x) = 0, bit-identical reruns, no gradient buffers without a gradient, deferred gains,
stft_data untouched)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import audiotools_b200.engine as engine_mod
from audiotools_b200 import AudioSignal, STFTParams, metrics
from audiotools_b200.engine import Engine
from tests import metrics_cases as mc
from tests.conftest import rel_err
from tests.cusim.sim_engine import sim_engine

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden")
SR = 16000


@pytest.fixture
def sim(monkeypatch):
    monkeypatch.setattr(engine_mod, "_ENGINE", sim_engine())
    yield sim_engine()


def _x(shape, seed):
    return 0.5 * torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def test_metrics_match_reference_golden(sim):
    """Every case of make_golden_metrics (log-only mel with fmin / fmax, 3-scale sqrt_hann STFT loss, match_stride with
    replicate / constant padding on 2-channel signals, PhaseLoss, L1Loss, SISDRLoss per reduction) within 1e-4."""
    golden = np.load(os.path.join(GOLDEN, "reference_golden_metrics.npz"))
    mc.check_metrics_golden(golden, "cpu")


def test_default_losses_match_reference_golden(sim):
    """The default mel, 7-scale mel and default STFT losses against make_golden_grad's values and gradients; the STFT
    loss's gradient by the rule of tests/grad_cases.check_golden (ours <= max(1e-4, 1.25 x the reference's FP32 error
    against float64))."""
    golden = np.load(os.path.join(GOLDEN, "reference_golden_grad.npz"))
    errs = mc.grad_golden_errors(golden, "cpu")
    assert all(v[0] < 1e-4 for v in errs.values()), errs
    assert errs["loss_mel"][1] < 1e-4 and errs["loss_mel7"][1] < 1e-4, errs
    ours, w = mc.stft_golden_oracle_err("cpu")
    ref_err = rel_err(torch.from_numpy(golden["loss_stft_grad"]), w)
    assert ours <= max(1e-4, 1.25 * ref_err), (ours, ref_err)


# (window, hop, mel = (sr, n_mels, fmin, fmax), match_stride, padding, window type, loss options): both MEL modes, every
# padding mode, match_stride, an odd hop and non-default weights (also per cell in tests/test_sim_loss_accuracy.py)
ENGINE_GEOMETRIES = [
    (256, 64, None, False, "reflect", "hann", {}),
    (128, 32, (SR, 20, 0.0, None), True, "constant", "hann", {}),
    (64, 13, None, False, "replicate", "hann", dict(pow=1.0, clamp_eps=1e-4)),          # odd hop
    (512, 128, (SR, 40, 100.0, 6000.0), False, "reflect", "sqrt_hann", dict(log_weight=0.5, mag_weight=2.0)),
    (2048, 512, (SR, 80, 0.0, None), True, "replicate", "hann", dict(mag_weight=0.0)),
]


@pytest.mark.parametrize("wl,hop,mel,ms,pt,wt,kw", ENGINE_GEOMETRIES)
def test_engine_loss_and_both_gradients_match_float64(sim, wl, hop, mel, ms, pt, wt, kw):
    """Engine.spectral_loss + the STFT adjoint against torch.autograd in float64, for x and y, both MEL modes, every
    padding mode, match_stride, an odd hop and non-default weights."""
    eng = sim
    T = 3000
    x, y = _x((2, 2, T), wl), _x((2, 2, T), wl + 1)
    right_pad, pad = (-T % hop, (wl - hop) // 2) if ms else (0, 0)
    w = AudioSignal.get_window(wt, wl, "cpu")
    tables = None
    if mel is not None:
        tables = AudioSignal._mel_tables(mel[0], wl, mel[1], mel[2], mel[3], torch.device("cpu"))
    drop = 2 if ms else 0
    loss, gX, gY = eng.spectral_loss(x, y, wl, hop, w, pad, right_pad, pt, drop, tables, want_grad_x=True,
                                     want_grad_y=True, **kw)
    gx = eng.stft_backward(gX, T, wl, hop, w, pad, right_pad, pt, drop)
    gy = eng.stft_backward(gY, T, wl, hop, w, pad, right_pad, pt, drop)
    xd, yd = x.double().requires_grad_(), y.double().requires_grad_()
    want = mc.scale_loss64(xd, yd, wl, hop, mel, ms, pt, wt, **kw)
    wx, wy = torch.autograd.grad(want, (xd, yd))
    xf, yf = x.clone().requires_grad_(), y.clone().requires_grad_()
    tx, ty = torch.autograd.grad(mc.scale_loss64(xf, yf, wl, hop, mel, ms, pt, wt, **kw), (xf, yf))
    assert abs(loss.item() - want.item()) <= 1e-5 * abs(want.item())
    assert rel_err(gx, wx) <= max(1e-4, 1.25 * rel_err(tx, wx)), (rel_err(gx, wx), rel_err(tx, wx))
    assert rel_err(gy, wy) <= max(1e-4, 1.25 * rel_err(ty, wy)), (rel_err(gy, wy), rel_err(ty, wy))


def _defaults():
    return [metrics.MelSpectrogramLoss(), metrics.MultiScaleSTFTLoss(),
            metrics.MelSpectrogramLoss([5, 10], [64, 128], mag_weight=0.0, pow=1.0, mel_fmin=[0.0] * 2,
                                       mel_fmax=[None] * 2)]


def test_fused_path_is_taken(sim, monkeypatch):
    """With the composed path's pieces patched to raise, the losses still run forward and backward."""
    def boom(*a, **k):
        raise AssertionError("composed path")

    for name in ("spectral", "mel_backward"):
        monkeypatch.setattr(Engine, name, boom)
    monkeypatch.setattr(torch, "stft", boom)
    monkeypatch.setattr(torch, "log10", boom)
    x, y = _x((2, 1, 4000), 0), _x((2, 1, 4000), 1)
    for mod in _defaults():
        xg = x.clone().requires_grad_()
        (gx,) = torch.autograd.grad(mod(AudioSignal(xg, SR), AudioSignal(y, SR)), xg)
        assert torch.isfinite(gx).all() and gx.abs().sum() > 0


@pytest.mark.parametrize("case", ["sisdr_loss_fn", "window_4096", "window_32", "sum_reduction", "other_sample_rate"])
def test_other_inputs_take_the_composed_path(sim, monkeypatch, case):
    """A loss_fn other than mean L1, a window outside [64, 2048] or mismatched signals run the reference's arithmetic
    through the differentiable AudioSignal methods, never the fused kernel; the result equals that arithmetic."""
    def boom(*a, **k):
        raise AssertionError("fused path")

    monkeypatch.setattr(Engine, "spectral_loss", boom)
    x, y = _x((1, 1, 9000), 2), _x((1, 1, 9000), 3)
    loss_fn, wls, sr_y = torch.nn.L1Loss(), [512], SR
    if case == "sisdr_loss_fn":
        loss_fn = metrics.SISDRLoss()
    elif case == "window_4096":
        wls = [4096]
    elif case == "window_32":
        wls = [32]
    elif case == "sum_reduction":
        loss_fn = torch.nn.L1Loss(reduction="sum")
    else:
        sr_y = SR // 2
    for mod in (metrics.MultiScaleSTFTLoss(wls, loss_fn=loss_fn), metrics.MelSpectrogramLoss([20], wls, loss_fn=loss_fn)):
        xg = x.clone().requires_grad_()
        loss = mod(AudioSignal(xg, SR), AudioSignal(y, sr_y))
        (gx,) = torch.autograd.grad(loss, xg)
        xr = x.clone().requires_grad_()
        sx, sy = AudioSignal(xr, SR), AudioSignal(y, sr_y)
        wl = wls[0]
        if isinstance(mod, metrics.MultiScaleSTFTLoss):
            a, b = sx.stft(wl, wl // 4).abs(), sy.stft(wl, wl // 4).abs()
        else:
            a, b = sx.mel_spectrogram(20, window_length=wl, hop_length=wl // 4), sy.mel_spectrogram(
                20, window_length=wl, hop_length=wl // 4)
        want = loss_fn(a.clamp(1e-5).pow(2).log10(), b.clamp(1e-5).pow(2).log10()) + loss_fn(a, b)
        (wx,) = torch.autograd.grad(want, xr)
        assert torch.equal(loss.detach(), want.detach()) and torch.equal(gx, wx)


def test_exact_properties(sim, monkeypatch):
    """loss(x, x.clone()) is exactly 0 with a zero gradient; reruns are bit-identical; stft_data is left alone."""
    x, y = _x((2, 2, 5000), 4), _x((2, 2, 5000), 5)
    for mod in _defaults():
        xg = x.clone().requires_grad_()
        sx, sy = AudioSignal(xg, SR), AudioSignal(x.clone(), SR)
        loss = mod(sx, sy)
        (gx,) = torch.autograd.grad(loss, xg)
        assert loss.item() == 0.0 and torch.count_nonzero(gx) == 0
        runs = []
        for _ in range(2):
            xg = x.clone().requires_grad_()
            sx, sy = AudioSignal(xg, SR), AudioSignal(y.clone(), SR)
            sentinel = torch.zeros(1, dtype=torch.complex64)
            sx.stft_data = sentinel
            loss = mod(sx, sy)
            (gx,) = torch.autograd.grad(loss, xg)
            assert sx.stft_data is sentinel and sy.stft_data is None
            runs.append((loss.detach(), gx))
        assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


def test_no_grad_allocates_no_gradient_and_defers_gain(sim, monkeypatch):
    """Under no_grad the kernel is asked for the loss alone; a gain deferred under no_grad gives the result of
    applying it explicitly."""
    seen = []
    orig = Engine.spectral_loss

    def spy(self, *a, **k):
        out = orig(self, *a, **k)
        seen.append((k.get("want_grad_x", False), k.get("want_grad_y", False), out[1], out[2]))
        return out

    monkeypatch.setattr(Engine, "spectral_loss", spy)
    x, y = _x((2, 1, 5000), 6), _x((2, 1, 5000), 7)
    db = torch.tensor([-6.0, 3.0])
    for mod in _defaults():
        seen.clear()
        with torch.no_grad():
            sx = AudioSignal(x.clone(), SR)
            sx.volume_change(db)  # (a CPU tensor is scaled at once; the H100 test covers a deferred gain)
            a = mod(sx, AudioSignal(y.clone(), SR))
            b = mod(AudioSignal(x * 10 ** (db[:, None, None] / 20), SR), AudioSignal(y.clone(), SR))
        assert seen and all(s == (False, False, None, None) for s in seen)
        assert abs(a.item() - b.item()) <= 1e-6 * abs(b.item())


def test_stft_params_decide_match_stride_and_padding(sim):
    """The constructor's match_stride is stored, unused: the signals' stft_params decide (as in the reference)."""
    x, y = _x((1, 2, 4000), 8), _x((1, 2, 4000), 9)
    sp = STFTParams(512, 128, "hann", True, "constant")
    a = metrics.MultiScaleSTFTLoss([512], match_stride=False)(AudioSignal(x, SR, stft_params=sp),
                                                               AudioSignal(y, SR, stft_params=sp))
    b = metrics.MultiScaleSTFTLoss([512], match_stride=True)(AudioSignal(x, SR, stft_params=sp),
                                                              AudioSignal(y, SR, stft_params=sp))
    want = mc.scale_loss64(x.double(), y.double(), 512, 128, ms=True, pt="constant")
    assert a.item() == b.item() and abs(a.item() - want.item()) <= 1e-5 * want.item()


_SHUFFLED = r"""
import sys, torch
sys.path.insert(0, sys.argv[1])
import audiotools_b200.engine as em
from audiotools_b200 import AudioSignal
from tests import metrics_cases as mc
from tests.conftest import rel_err
from tests.cusim.sim_engine import sim_engine
em._ENGINE = sim_engine()
eng = em._ENGINE
T = 2500
for wl, hop, mel in [(256, 64, None), (128, 32, (16000, 20, 0.0, None)), (1024, 256, (16000, 40, 0.0, None))]:
    x = torch.randn(1, 2, T, generator=torch.Generator().manual_seed(wl))
    y = torch.randn(1, 2, T, generator=torch.Generator().manual_seed(wl + 1))
    w = AudioSignal.get_window("hann", wl, "cpu")
    tables = AudioSignal._mel_tables(mel[0], wl, mel[1], mel[2], mel[3], torch.device("cpu")) if mel else None
    loss, gX, gY = eng.spectral_loss(x, y, wl, hop, w, mel=tables, want_grad_x=True, want_grad_y=True)
    gx, gy = eng.stft_backward(gX, T, wl, hop, w), eng.stft_backward(gY, T, wl, hop, w)
    xd, yd = x.double().requires_grad_(), y.double().requires_grad_()
    want = mc.scale_loss64(xd, yd, wl, hop, mel)
    wx, wy = torch.autograd.grad(want, (xd, yd))
    assert abs(loss.item() - want.item()) <= 1e-5 * abs(want.item()), wl
    assert rel_err(gx, wx) < 1e-3 and rel_err(gy, wy) < 1e-3, (wl, rel_err(gx, wx), rel_err(gy, wy))
print("ok")
"""


def test_loss_kernel_under_shuffled_fiber_order():
    """The simulator visits the CUDA threads of a block in a random order under CUSIM_SHUFFLE: a missing barrier or
    __syncwarp that the fixed order happens to satisfy shows up as a wrong result.  (Read once per process: a child.)"""
    env = dict(os.environ, CUSIM_SHUFFLE="1")
    r = subprocess.run([sys.executable, "-c", _SHUFFLED, REPO], env=env, cwd=REPO, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
