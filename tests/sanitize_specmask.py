"""Small driver for compute-sanitizer runs (memcheck / racecheck / synccheck) over csrc/specmask.cu through the engine:
the band masks on both axes at both block sizes, rotate and mask_low past the grid-stride cap, and the gate forward and
backward with the largest halos (half-width 8 on both axes, and 0) at shapes one cell on either side of the
16 x 64 tiles of ``gate_apply_kernel``, whose two barriers separate staging, the time pass and the frequency pass.
`compute-sanitizer --tool racecheck python tests/sanitize_specmask.py`"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as graft  # noqa: E402

graft.build()
from audiotools_b200.engine import get_engine  # noqa: E402
from audiotools_b200.ml.layers.spectral_gate import _ramp  # noqa: E402

dev = "cuda:0"
eng = get_engine()
gen = torch.Generator().manual_seed(0)


def cplx(*shape):
    return torch.complex(torch.randn(shape, generator=gen), torch.randn(shape, generator=gen)).to(dev)


out = []
for F, N in ((17, 255), (16, 257), (1, 1)):
    X, G = cplx(2, 2, F, N), cplx(2, 2, F, N)
    lo, hi = torch.tensor([0.1, 0.3], device=dev), torch.tensor([0.6, 0.9], device=dev)
    for axis, n in ((0, F), (1, N)):
        v = torch.linspace(0, 1, n, device=dev)
        out.append(float(eng.spec_band_mask(X.clone(), v, lo, hi, axis, 0.5).abs().sum()))
        out.append(float(eng.spec_band_mask_out(X, v, lo, hi, axis, 0.5).abs().sum()))
        out.append(float(eng.spec_band_mask_backward(G, X, v, lo, hi, axis).abs().sum()))
X, G = cplx(3, 1, 513, 400), cplx(3, 1, 513, 400)
cut = torch.tensor([-10.0, 0.0, 5.0], device=dev)
out.append(float(eng.spec_rotate(X.clone(), torch.tensor([0.5, 1.0, -2.0], device=dev)).abs().sum()))
out.append(float(eng.spec_mask_low(X.clone(), cut, 0.5).abs().sum()))
y, ws = eng.spec_mask_low_out(X, cut, 0.5)
out += [float(y.abs().sum()), float(eng.spec_mask_low_backward(G, X, cut, 0.5, ws).abs().sum())]
amount = torch.tensor([1.0, 0.5], device=dev)
for F, N in ((15, 63), (17, 65), (33, 129)):
    X, G = 0.02 * cplx(2, 2, F, N), cplx(2, 2, F, N)
    nz = 0.01 * cplx(1, 1, F, 50)
    for h in (8, 0):
        sf, st = _ramp(h).tolist(), _ramp(h).tolist()
        y, th = eng.spec_gate(X, nz, 1.0, amount, sf, st)
        out += [float(y.abs().sum()), float(eng.spec_gate_backward(G, X, th, amount, sf, st).abs().sum())]
torch.cuda.synchronize()
print("ok", [round(v, 3) for v in out])
