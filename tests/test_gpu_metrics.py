"""audiotools_b200.metrics on the H100: the fused spectral losses of csrc/loss.cu against the real reference's goldens
and float64 at 16 x 1 ch x 1 s, the fused path with the composed path's pieces forbidden, and the exact properties."""
import os

import numpy as np
import pytest
import torch

from audiotools_b200 import AudioSignal, metrics
from audiotools_b200.engine import Engine
from tests import grad_cases as gc
from tests import metrics_cases as mc
from tests.conftest import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SR = 44100


def _pair(B=16, C=1, T=SR, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (0.1 * torch.randn(B, C, T, generator=g)).to(DEV), (0.1 * torch.randn(B, C, T, generator=g)).to(DEV)


def _defaults():
    seven = dict(n_mels=gc.MEL_LOSS_7SCALE["n_mels"], window_lengths=gc.MEL_LOSS_7SCALE["window_lengths"],
                 mag_weight=0.0, pow=1.0, mel_fmin=[0.0] * 7, mel_fmax=[None] * 7)
    return {"mel": metrics.MelSpectrogramLoss(), "mel7": metrics.MelSpectrogramLoss(**seven),
            "stft": metrics.MultiScaleSTFTLoss()}


def test_metrics_match_reference_golden():
    mc.check_metrics_golden(np.load(os.path.join(GOLDEN, "reference_golden_metrics.npz")), DEV)


def test_default_losses_match_reference_golden():
    golden = np.load(os.path.join(GOLDEN, "reference_golden_grad.npz"))
    errs = mc.grad_golden_errors(golden, DEV)
    assert all(v[0] < 1e-4 for v in errs.values()), errs
    assert errs["loss_mel"][1] < 1e-4 and errs["loss_mel7"][1] < 1e-4, errs
    ours, w = mc.stft_golden_oracle_err(DEV)
    ref_err = rel_err(torch.from_numpy(golden["loss_stft_grad"]), w)
    assert ours <= max(1e-4, 1.25 * ref_err), (ours, ref_err)


def test_default_losses_against_float64_at_training_shape():
    """16 x 1 ch x 1 s: loss within 1e-5 of float64, dL/dx (and dL/dy) within max(1e-4, 1.25 x torch FP32's error),
    with torch.stft / torch.log10 / the composed path's kernels forbidden for the fused run."""
    x, y = _pair()
    mods = _defaults()
    xd, yd = x.double().requires_grad_(), y.double().requires_grad_()
    xf, yf = x.clone().requires_grad_(), y.clone().requires_grad_()
    want = dict(zip(["mel", "mel7", "stft"], gc.oracle_losses(xd, yd, SR)))
    f32 = dict(zip(["mel", "mel7", "stft"], gc.oracle_losses(xf, yf, SR)))
    for name, mod in mods.items():
        wx, wy = torch.autograd.grad(want[name], (xd, yd))
        tx, ty = torch.autograd.grad(f32[name], (xf, yf))
        xg, yg = x.clone().requires_grad_(), y.clone().requires_grad_()
        with _forbidden(name != "mel7"):  # the 7-scale loss's 32-sample scale runs the composed path
            loss = mod(AudioSignal(xg, SR), AudioSignal(yg, SR))
            gx, gy = torch.autograd.grad(loss, (xg, yg))
        assert abs(loss.item() - want[name].item()) <= 1e-5 * abs(want[name].item()), name
        ex, ey = rel_err(tx, wx), rel_err(ty, wy)
        if name == "mel7":
            # the 7-scale loss has cells whose L1 sign FP32 cannot resolve (tests/grad_cases.fp32_resolution_keep);
            # the fused kernel computes the whole loss, so it is held to the composed path's error on the same cells
            xc, yc = x.clone().requires_grad_(), y.clone().requires_grad_()
            cx, cy = torch.autograd.grad(gc.signal_losses(xc, yc, SR)[1], (xc, yc))
            ex, ey = max(ex, rel_err(cx, wx)), max(ey, rel_err(cy, wy))
        assert rel_err(gx, wx) <= max(1e-4, 1.25 * ex), (name, rel_err(gx, wx), ex)
        assert rel_err(gy, wy) <= max(1e-4, 1.25 * ey), (name, rel_err(gy, wy), ey)


class _forbidden:
    """The composed path's pieces raise inside the block (when ``on``)."""

    def __init__(self, on=True):
        self.on = on

    def __enter__(self):
        def boom(*a, **k):
            raise AssertionError("composed path")

        self.saved = [(Engine, "spectral", Engine.spectral), (Engine, "mel_backward", Engine.mel_backward),
                      (torch, "stft", torch.stft), (torch, "log10", torch.log10)] if self.on else []
        for obj, name, _ in self.saved:
            setattr(obj, name, boom)

    def __exit__(self, *exc):
        for obj, name, fn in self.saved:
            setattr(obj, name, fn)


def test_composed_path_for_other_inputs():
    """SISDRLoss as loss_fn and a 4096 window run the reference's arithmetic, with the same result."""
    x, y = _pair(4, 1, 20000, 3)
    for mod, wl, loss_fn in [(metrics.MultiScaleSTFTLoss([4096]), 4096, torch.nn.L1Loss()),
                             (metrics.MultiScaleSTFTLoss([512], loss_fn=metrics.SISDRLoss()), 512, metrics.SISDRLoss())]:
        xg = x.clone().requires_grad_()
        loss = mod(AudioSignal(xg, SR), AudioSignal(y, SR))
        (gx,) = torch.autograd.grad(loss, xg)
        xr = x.clone().requires_grad_()
        a, b = AudioSignal(xr, SR).stft(wl, wl // 4).abs(), AudioSignal(y, SR).stft(wl, wl // 4).abs()
        want = loss_fn(a.clamp(1e-5).pow(2).log10(), b.clamp(1e-5).pow(2).log10()) + loss_fn(a, b)
        (wx,) = torch.autograd.grad(want, xr)
        assert torch.equal(loss.detach(), want.detach()) and torch.equal(gx, wx)


def test_exact_properties_on_device():
    """loss(x, x) = 0 with zero gradient, bit-identical reruns, stft_data untouched, deferred gain under no_grad."""
    x, y = _pair(4, 2, 30000, 5)
    for name, mod in _defaults().items():
        xg = x.clone().requires_grad_()
        loss = mod(AudioSignal(xg, SR), AudioSignal(x.clone(), SR))
        (gx,) = torch.autograd.grad(loss, xg)
        assert loss.item() == 0.0 and torch.count_nonzero(gx) == 0, name
        runs = []
        for _ in range(2):
            xg = x.clone().requires_grad_()
            sx, sy = AudioSignal(xg, SR), AudioSignal(y.clone(), SR)
            loss = mod(sx, sy)
            (gx,) = torch.autograd.grad(loss, xg)
            assert sx.stft_data is None and sy.stft_data is None
            runs.append((loss.detach(), gx))
        assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1]), name
        db = torch.tensor([-6.0, 3.0, 0.5, -1.0], device=DEV)
        with torch.no_grad():
            sx = AudioSignal(x.clone(), SR)
            sx.volume_change(db)
            a = mod(sx, AudioSignal(y.clone(), SR))
            b = mod(AudioSignal(x * 10 ** (db[:, None, None] / 20), SR), AudioSignal(y.clone(), SR))
        assert abs(a.item() - b.item()) <= 1e-6 * abs(b.item()), name


def test_no_grad_allocates_no_gradient(monkeypatch):
    seen = []
    orig = Engine.spectral_loss

    def spy(self, *a, **k):
        out = orig(self, *a, **k)
        seen.append(out[1] is None and out[2] is None)
        return out

    monkeypatch.setattr(Engine, "spectral_loss", spy)
    x, y = _pair(64, 2, 10 * SR, 9)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(DEV)
    torch.cuda.reset_peak_memory_stats(DEV)
    with torch.no_grad():  # (the 7-scale loss's 32-sample scale runs the composed path, which materialises the STFT)
        for name in ("mel", "stft"):
            _defaults()[name](AudioSignal(x, SR), AudioSignal(y, SR))
    torch.cuda.synchronize()
    assert seen and all(seen)
    # no STFT-sized buffer (905 MB at this shape) was allocated
    assert torch.cuda.max_memory_allocated(DEV) - base < 64 * 2**20
