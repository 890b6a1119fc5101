"""``scipy.signal.sosfilt`` with initial state and ``scipy.signal.sosfiltfilt`` for a batch on the GPU (csrc/iir.cu,
DESIGN.md K19), with scipy's argument order and return conventions.

* ``sosfilt(sos, x, zi=None)``: ``y``, or ``(y, zf)`` when ``zi`` is given.  ``zi`` has scipy's layout for x
  [B, C, T], ``[S, B, C, 2]``; ``zf`` is float64 in the same layout, so a long row can be filtered in segments by
  passing each ``zf`` as the next ``zi``.
* ``sosfiltfilt(sos, x, padtype="odd", padlen=None)``: zero-phase filtering, method "pad".

``x`` is [B, C, T] float32 on the GPU; ``sos`` is [S, 6] or [B, S, 6] (1 <= S <= 8), each row divided by its a0 and
rounded to float32 once.  An item with a section whose poles are not strictly inside the unit circle is all NaN.
``sosfiltfilt`` and ``sosfilt`` without ``zi`` are differentiable with respect to ``x``; ``sos`` is a constant.
``sosfilt`` with ``zi`` has no backward: an ``x`` or a ``zi`` that requires a gradient raises ``NotImplementedError``.
"""
from . import grad as _grad


def _engine():
    from ..engine import get_engine

    return get_engine()


def sosfilt(sos, x, zi=None):
    """``scipy.signal.sosfilt(sos, x, axis=-1, zi=zi)`` for x [B, C, T]."""
    _grad.refuse_param_grad("sosfilt", "sos", sos)
    eng = _engine()
    if zi is None:
        if _grad.wants_grad(x):
            return _grad.SOSFilter.apply(x, eng.sos_coefficients(sos, x.shape[0], x.device), None)
        return eng.sos_filter(x, sos)
    return eng.sos_filter_zi(x, sos, zi)


def sosfiltfilt(sos, x, padtype="odd", padlen=None):
    """``scipy.signal.sosfiltfilt(sos, x, axis=-1, padtype=padtype, padlen=padlen)`` for x [B, C, T].  With
    ``padlen=None`` each item's padding follows scipy's rule for its own sections; the length is checked against the
    largest such value, 3 (2S + 1), so that no value is read back from the GPU: unlike scipy, rows of at most 51
    samples are refused when the sections would allow a shorter padding."""
    _grad.refuse_param_grad("sosfiltfilt", "sos", sos)
    if _grad.wants_grad(x):
        return _grad.SOSFiltFilt.apply(x, sos, None, padtype, padlen)
    return _engine().sos_filtfilt(x, sos, padtype, padlen)
