"""The per-item element-wise effects of csrc/effects.cu on the H100 (``-m gpu``): gain, clamp_items, mix (with and
without a gain), limit_peak, row_absmax and linear quantize, bit for bit against a float32 NumPy restatement, on both
branches of their walk: float4 on 16-byte-aligned rows of a multiple of 4 samples, scalar on views offset by one float
and on lengths of 1, 2 and 3 mod 4.  tests/test_sim_elementwise.py runs the same checks on the CPU simulator."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
LENGTHS = (1, 2, 3, 4, 5, 6, 7, 4096, 4099)


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


def place(x: np.ndarray, off: int) -> torch.Tensor:
    """x on DEV as a view ``off`` floats into a 16-byte-aligned buffer."""
    buf = torch.zeros(x.size + 4, device=DEV)
    v = buf[off:off + x.size].view(x.shape)
    v.copy_(torch.from_numpy(x))
    assert v.data_ptr() % 16 == 4 * off
    return v


def same_bits(t: torch.Tensor, ref: np.ndarray) -> bool:
    a = t.detach().cpu().numpy()
    return a.shape == ref.shape and np.array_equal(a.view(np.int32), ref.astype(np.float32).view(np.int32))


def check_elementwise(eng, T: int, off: int):
    rng = np.random.default_rng(4 * T + off)
    f32 = np.float32
    x = (rng.standard_normal((3, 2, T)) * np.array([0.05, 0.5, 2.0])[:, None, None]).astype(f32)
    o = rng.standard_normal((3, 2, T)).astype(f32)
    g = np.array([0.5, 2.0, -1.25], f32)
    lo, hi = np.array([-0.5, -1.0, -0.1], f32), np.array([0.5, 1.0, 0.2], f32)
    q = np.array([8, 256, 3], f32)
    xd, od = place(x, off), place(o, off)
    dev = lambda a: torch.from_numpy(a).to(DEV)  # noqa: E731
    item = lambda a: a[:, None, None]  # noqa: E731

    assert same_bits(eng.gain(xd, dev(g)), x * item(g))
    assert same_bits(eng.gain(place(x, 0), dev(g), out=place(np.zeros_like(x), off)), x * item(g))
    assert same_bits(eng.clamp_items(xd, dev(lo), dev(hi)), np.minimum(np.maximum(x, item(lo)), item(hi)))
    assert same_bits(eng.mix(xd, od, dev(g)), x + o * item(g))  # float32: the product is rounded before the sum
    assert same_bits(eng.mix(xd, od), x + o)
    peak = np.abs(x).max(-1, keepdims=True)
    assert same_bits(eng.row_absmax(xd), peak)
    lim = f32(0.7)
    scale = np.where(peak > lim, lim / peak, f32(1)).astype(f32)
    assert same_bits(eng.limit_peak(xd, float(lim)), x * scale)
    # linear quantisation, operation by operation (ref:audiotools/core/effects.py:481-491)
    y = np.floor(((x + f32(1)) / f32(2)) * item(q)) / item(q)
    y = f32(2) * y + f32(-1)
    assert same_bits(eng.quantize(xd, dev(q)), x - (x - y))


@pytest.mark.parametrize("off", [0, 1])
@pytest.mark.parametrize("T", LENGTHS)
def test_elementwise_against_float32(eng, T, off):
    check_elementwise(eng, T, off)
