"""Second-order sections of the RBJ Audio EQ Cookbook (R. Bristow-Johnson), designed in float64 on the parameters'
device: one biquad per item and per band, as ``sos`` rows ``b0 b1 b2 a0 a1 a2`` for ``AudioSignal.sos_filter``.

With w0 = 2 pi freq / sr, A = 10^(gain_db / 40) and alpha = sin w0 / (2 Q):

  peaking      b = 1 + alpha A, -2 cos w0, 1 - alpha A           a = 1 + alpha / A, -2 cos w0, 1 - alpha / A
  low_shelf    b = A ((A+1) - (A-1) cos w0 + 2 sqrt(A) alpha), 2 A ((A-1) - (A+1) cos w0),
                   A ((A+1) - (A-1) cos w0 - 2 sqrt(A) alpha)
               a = (A+1) + (A-1) cos w0 + 2 sqrt(A) alpha, -2 ((A-1) + (A+1) cos w0), (A+1) + (A-1) cos w0 - 2 sqrt(A) alpha
  high_shelf   the low shelf with the signs of the (A-1) cos w0 terms and of b1 / a1's (A-1) turned around
  low_pass     b = (1 - cos w0) / 2, 1 - cos w0, (1 - cos w0) / 2   a = 1 + alpha, -2 cos w0, 1 - alpha
  high_pass    b = (1 + cos w0) / 2, -(1 + cos w0), (1 + cos w0) / 2
  band_pass    b = alpha, 0, -alpha  (0 dB peak)
  notch        b = 1, -2 cos w0, 1
  all_pass     b = 1 - alpha, -2 cos w0, 1 + alpha
(the last five share a = 1 + alpha, -2 cos w0, 1 - alpha).  ``gain_db`` is used by ``peaking`` and the shelves only.
"""
import numpy as np
import torch

from . import util

KINDS = ("peaking", "low_shelf", "high_shelf", "low_pass", "high_pass", "band_pass", "notch", "all_pass")


def _host(v):
    return util.host_view(v) if torch.is_tensor(v) else v


def check(kinds, freq, q, sample_rate: float):
    """Refuse an unknown kind, a frequency outside (0, sr/2) or a Q that is not positive, on host values: a parameter
    table with a host mirror (``util.prepare_batch``) costs no device synchronisation."""
    for k in kinds:
        if k not in KINDS:
            raise ValueError(f"parametric_eq: unknown kind {k!r}; one of {', '.join(KINDS)}")
    f = np.asarray(torch.as_tensor(_host(freq)).double().cpu())
    qq = np.asarray(torch.as_tensor(_host(q)).double().cpu())
    if not ((f > 0) & (f < sample_rate / 2)).all():
        raise ValueError(f"parametric_eq: every freq must lie in (0, {sample_rate / 2}) Hz, got {f.min()} .. {f.max()}")
    if not (qq > 0).all():
        raise ValueError(f"parametric_eq: q must be positive, got {qq.min()}")


def design(kinds, freq, gain_db, q, sample_rate: float, batch_size: int, device) -> torch.Tensor:
    """-> sos [batch_size, n_bands, 6] float64 on ``device``.  ``kinds``: n_bands strings; ``freq``, ``gain_db`` and
    ``q``: numbers, [n_bands] or [batch_size, n_bands]."""
    n = len(kinds)

    def table(v):
        t = torch.as_tensor(np.asarray(v, dtype=np.float64)) if not torch.is_tensor(v) else v.to(torch.float64)
        t = t.to(device, non_blocking=True)  # a host table is uploaded without waiting for the device
        if t.ndim < 2:
            t = t.reshape(1, -1)
        return t.expand(batch_size, n)

    f, g, qq = table(freq), table(gain_db), table(q)
    w0 = 2 * np.pi * f / float(sample_rate)
    cw, alpha = torch.cos(w0), torch.sin(w0) / (2 * qq)
    A = torch.pow(10.0, g / 40)
    sA = torch.sqrt(A)
    one = torch.ones_like(cw)
    rows = []
    for i, k in enumerate(kinds):
        c, al, a, s = cw[:, i], alpha[:, i], A[:, i], sA[:, i]
        o = one[:, i]
        if k == "peaking":
            r = (o + al * a, -2 * c, o - al * a, o + al / a, -2 * c, o - al / a)
        elif k in ("low_shelf", "high_shelf"):
            sg = 1 if k == "low_shelf" else -1
            r = (a * ((a + 1) - sg * (a - 1) * c + 2 * s * al), sg * 2 * a * ((a - 1) - sg * (a + 1) * c),
                 a * ((a + 1) - sg * (a - 1) * c - 2 * s * al), (a + 1) + sg * (a - 1) * c + 2 * s * al,
                 -sg * 2 * ((a - 1) + sg * (a + 1) * c), (a + 1) + sg * (a - 1) * c - 2 * s * al)
        else:
            den = (o + al, -2 * c, o - al)
            num = {"low_pass": ((o - c) / 2, o - c, (o - c) / 2),
                   "high_pass": ((o + c) / 2, -(o + c), (o + c) / 2),
                   "band_pass": (al, 0 * o, -al),
                   "notch": (o, -2 * c, o),
                   "all_pass": (o - al, -2 * c, o + al)}[k]
            r = num + den
        rows.append(torch.stack(r, dim=-1))
    return torch.stack(rows, dim=1)
