"""Shared checks of the spectral masks' and the spectral gate's gradients against the REAL reference's
(tests/golden/make_golden_specaug_grad.py), used by the simulator and the GPU tests."""
import os

import numpy as np
import torch

import audiotools_b200
from tests.conftest import rel_err
from tests.golden import make_golden_specaug_grad as mg

# per cell, relative to the RMS of the cell's frame of the upstream gradient G (val = 0, val = 0.25 band masks, the gate).
# G's frame, not dL/dX's: the gate's 1 - amount * S cancels where S is near 1, in the reference's FP32 as in this
# package's, so there the error is a fraction of |G|, not of the (small) gradient.
SPEC_TOL = 1e-6
WAVE_TOL = 1e-4  # end to end, relative to the largest gradient


def load_golden():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                                "reference_golden_specaug_grad.npz"))


def frame_rms(g):
    """RMS over the frequency axis of each frame of a [B, C, F, N] complex tensor."""
    return g.abs().pow(2).mean(dim=-2, keepdim=True).sqrt()


def gate_smoothed(mask, amount):
    """amount * the reference's zero-padded 2-D smoothing of a boolean mask, float64 (spectral_gate.py:107-121)."""
    from audiotools_b200.ml.layers import SpectralGate

    k = SpectralGate().smoothing_filter.double()
    B, C, F, N = mask.shape
    S = torch.nn.functional.conv2d(mask.double().reshape(B * C, 1, F, N), k,
                                   padding=(k.shape[-2] // 2, k.shape[-1] // 2)).reshape(B, C, F, N)
    return S * torch.as_tensor(amount, dtype=torch.float64).reshape(-1, 1, 1, 1)


def low_val_float64(X, G, mask, val):
    """dL/dX of mask_low_magnitudes restated in float64 with the reference's mask: where masked, val exp(1j angle X)."""
    Xd = X.to(torch.complex128).requires_grad_()
    y = torch.where(mask, val * torch.exp(1j * torch.angle(Xd)), Xd.abs() * torch.exp(1j * torch.angle(Xd)))
    (g,) = torch.autograd.grad((torch.view_as_real(y) * torch.view_as_real(G.to(torch.complex128))).sum(), Xd)
    return g


def check_spec_case(golden, key, device):
    """One spectral-domain case: mask decisions equal the reference's, the gradient per cell within SPEC_TOL of the
    frame RMS; mask_low's val != 0 masked cells against float64 (returns (ours, reference's FP32) max error there,
    relative to the largest float64 gradient of those cells, else None)."""
    _, method, args = mg.CASES[key]
    seed = int(golden[f"{key}_seed"])
    y, g, X = mg.run_case(audiotools_b200, key, device, seed=seed)
    y, g, X = y.cpu(), g.cpu(), X.cpu()
    want = torch.from_numpy(golden[f"{key}_grad"])
    mask = torch.from_numpy(golden[f"{key}_mask"])
    if method == "gate":
        # 1 - out / X = amount * S: a flipped decision moves S by at least one smoothing weight (>= 1e-2)
        nz = X != 0
        S = (1 - y[nz] / X[nz]).real.double()
        assert (S - gate_smoothed(mask, args["amount"])[nz]).abs().max() < 1e-4, key
    else:
        val = args["val"]
        assert torch.equal(y != X, mask & ~((X == 0) & (val == 0))), key
    G = mg.cotangent(y.shape, 7000 + sorted(mg.CASES).index(key), complex_=True)
    tol = SPEC_TOL * frame_rms(G)
    exact = ~mask if method == "mask_low_magnitudes" and args["val"] != 0 else torch.ones_like(mask)
    assert bool(((g - want).abs() <= tol)[exact].all()), (key, (g - want).abs().max().item())
    if not bool(exact.all()):
        g64 = low_val_float64(X, G, mask, args["val"])
        sel = mask & (X != 0)
        scale = g64[sel].abs().max()
        ours = ((g.to(torch.complex128) - g64)[sel].abs().max() / scale).item()
        ref = ((want.to(torch.complex128) - g64)[sel].abs().max() / scale).item()
        assert ours <= 2 * ref, (key, ours, ref)
        assert bool((g[mask & (X == 0)] == 0).all())
        return ours, ref
    return None


def check_wave_case(golden, key, device):
    seed = int(golden[f"{key}_seed"])
    _, gx, _ = mg.run_case(audiotools_b200, key, device, seed=seed)
    want = torch.from_numpy(golden[f"{key}_grad"])
    err = rel_err(gx.cpu(), want)
    assert err < WAVE_TOL, (key, err)
    return err


def spec_keys():
    return [k for k, v in mg.CASES.items() if v[0] == "spec"]


def wave_keys():
    return [k for k, v in mg.CASES.items() if v[0] == "wave"]
