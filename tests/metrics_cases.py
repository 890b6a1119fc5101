"""Shared by the metrics tests (simulator and GPU): the real reference's goldens recomputed through
``audiotools_b200.metrics``, and float64 restatements of one loss scale for the engine-level checks."""
import numpy as np
import torch

from audiotools_b200 import AudioSignal, STFTParams, metrics
from tests import grad_cases as gc
from tests.conftest import rel_err


def golden_metric_errors(golden, device):
    """{case: (relative error of the value, relative error of dL/dx)} of every case of make_golden_metrics against the
    real reference, and of the three losses of make_golden_grad (``loss_mel``, ``loss_mel7``, ``loss_stft``)."""
    from tests.golden import make_golden_grad as mg
    from tests.golden import make_golden_metrics as mm

    x, y = mg.make_input().to(device), mg.make_input(1).to(device)
    keep = mg.keep_index(mg.T, 2048)
    errs = {}
    for key in mm.CASES:
        xg = x.clone().requires_grad_()
        sx, sy = mm.signals(AudioSignal, STFTParams, key, xg, y.clone())
        loss = mm.module(metrics.spectral, metrics.distance, key)(sx, sy)
        (gx,) = torch.autograd.grad(loss.sum(), xg)
        want = torch.from_numpy(np.asarray(golden[key]))
        errs[key] = (rel_err(loss.detach().double().cpu().reshape(want.shape), want),
                     rel_err(gx[mg.ROWS][..., keep].cpu(), torch.from_numpy(golden[key + "_grad"])))
    return errs


def _stft_case_oracle(key, device):
    """float64 dL/dx (golden rows / samples) of a MultiScaleSTFTLoss case of make_golden_metrics."""
    from tests.golden import make_golden_grad as mg
    from tests.golden import make_golden_metrics as mm

    x, y = mg.make_input().to(device).double().requires_grad_(), mg.make_input(1).to(device).double()
    _, kw, sp = mm.CASES[key]
    ms, pt = (sp["match_stride"], sp["padding_type"]) if sp else (False, "reflect")
    wt = kw.get("window_type") or "hann"
    loss = sum(scale_loss64(x, y, wl, wl // 4, None, ms, pt, wt, log_weight=kw.get("log_weight", 1.0))
               for wl in kw["window_lengths"])
    (w,) = torch.autograd.grad(loss, x)
    return w[mg.ROWS][..., mg.keep_index(mg.T, 2048)].cpu()


def check_metrics_golden(golden, device, tol=1e-4):
    """Every make_golden_metrics case within ``tol`` of the real reference, except:
      - the MultiScaleSTFTLoss gradients: log10 of single bins is ill-conditioned where |X| is small, and the reference's
        own FP32 gradient is ~1e-4..1e-3 from float64; there ours must be at most 1.25x the reference's distance to
        float64 (the rule of tests/grad_cases.check_golden);
      - PhaseLoss: the reference's wrap (``diff[diff > pi] -= -2 pi``) jumps by 4 pi where a phase difference crosses
        pi, so FP32 phase errors of a few cells flip their term; value and gradient within 0.1 (torch's FP32 path
        over the same inputs differs from float64 by the same order)."""
    from tests.golden import make_golden_metrics as mm

    errs = golden_metric_errors(golden, device)
    bad = {}
    for key, (ev, eg) in errs.items():
        if key == "phase":
            ok = ev < 0.1 and eg < 0.1
        elif mm.CASES[key][0] == "MultiScaleSTFTLoss":
            w = _stft_case_oracle(key, device)
            from tests.golden import make_golden_grad as mg

            x, y = mg.make_input().to(device), mg.make_input(1).to(device)
            xg = x.clone().requires_grad_()
            sx, sy = mm.signals(AudioSignal, STFTParams, key, xg, y.clone())
            (g,) = torch.autograd.grad(mm.module(metrics.spectral, metrics.distance, key)(sx, sy), xg)
            ours = rel_err(g[mg.ROWS][..., mg.keep_index(mg.T, 2048)].cpu(), w)
            ref = rel_err(torch.from_numpy(golden[key + "_grad"]), w)
            ok = ev < tol and ours <= max(tol, 1.25 * ref)
            errs[key] = (ev, eg, ours, ref)
        else:
            ok = ev < tol and eg < tol
        if not ok:
            bad[key] = errs[key]
    assert not bad, bad
    return errs


def grad_golden_errors(golden_grad, device):
    """The three losses of make_golden_grad through the metrics modules: {key: (value error, dL/dx error)}."""
    from tests.golden import make_golden_grad as mg

    x, y = mg.make_input().to(device), mg.make_input(1).to(device)
    keep = mg.keep_index(mg.T, 2048)
    mods = {"loss_mel": metrics.MelSpectrogramLoss(), "loss_stft": metrics.MultiScaleSTFTLoss(),
            "loss_mel7": metrics.MelSpectrogramLoss(**mg.LOSS_7SCALE)}
    errs = {}
    for key, mod in mods.items():
        xg = x.clone().requires_grad_()
        loss = mod(AudioSignal(xg, mg.SR), AudioSignal(y.clone(), mg.SR))
        (gx,) = torch.autograd.grad(loss, xg)
        want = float(golden_grad[key])
        errs[key] = (abs(loss.item() - want) / abs(want),
                     rel_err(gx[mg.ROWS][..., keep].cpu(), torch.from_numpy(golden_grad[key + "_grad"])))
    return errs


def stft_golden_oracle_err(device, key="loss_stft"):
    """(ours, the reference's own FP32) distance to float64 of the default MultiScaleSTFTLoss gradient on the golden
    inputs: the rule for that gradient is ours <= max(1e-4, 1.25 x the reference's)."""
    from tests.golden import make_golden_grad as mg

    x, y = mg.make_input().to(device), mg.make_input(1).to(device)
    keep = mg.keep_index(mg.T, 2048)
    xd = x.double().requires_grad_()
    (w,) = torch.autograd.grad(gc.oracle_losses(xd, y.double(), mg.SR)[2], xd)
    w = w[mg.ROWS][..., keep].cpu()
    xg = x.clone().requires_grad_()
    (g,) = torch.autograd.grad(metrics.MultiScaleSTFTLoss()(AudioSignal(xg, mg.SR), AudioSignal(y.clone(), mg.SR)), xg)
    return rel_err(g[mg.ROWS][..., keep].cpu(), w), w


def scale_loss64(x, y, wl, hop, mel=None, ms=False, pt="reflect", window_type="hann", clamp_eps=1e-5, pow=2.0,
                 log_weight=1.0, mag_weight=1.0):
    """One scale of the reference's L1 loss in x's precision through torch.stft; mel = (sr, n_mels, fmin, fmax)."""
    def mag(t):
        X = gc.stft64(t, wl, hop, window_type, ms, pt).abs()
        if mel is None:
            return X
        sr, nm, fmin, fmax = mel
        fb = torch.from_numpy(np.asarray(AudioSignal.get_mel_filters(sr, wl, nm, fmin, fmax), dtype=np.float64))
        return (X.transpose(2, -1) @ fb.to(t.device, t.dtype).T).transpose(-1, 2)

    xm, ym = mag(x), mag(y)
    lg = lambda v: v.clamp(clamp_eps).pow(pow).log10()  # noqa: E731
    return (log_weight * torch.nn.functional.l1_loss(lg(xm), lg(ym))
            + mag_weight * torch.nn.functional.l1_loss(xm, ym))
