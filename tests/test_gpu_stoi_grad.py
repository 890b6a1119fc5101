"""metrics.quality.STOILoss on the H100 (the STOI backward of csrc/stoi.cu): the loss equals -stoi() for every golden
case, the gradient matches autograd through the float64 restatement (tests/stoi_grad_cases.py) for every case in both
modes, its properties and plumbing, bit-identical reruns, and a full-size 64 x 2ch x 10 s batch at 44.1 kHz against the
restatement on a strided subset of items."""
import numpy as np
import pytest
import torch

from audiotools_b200 import metrics
from tests import stoi_grad_cases as sg
from tests.golden import make_golden_quality as mg

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("key", sorted(mg.CASES))
def test_loss_is_minus_stoi(key):
    sg.check_value(key, DEV)


@pytest.mark.parametrize("extended", [False, True])
@pytest.mark.parametrize("key", sorted(mg.CASES))
def test_gradient_matches_float64(key, extended):
    sg.check_gradient(key, extended, DEV)


@pytest.mark.parametrize("extended", [False, True])
def test_gradient_properties(extended):
    sg.check_properties(DEV, extended)


def test_plumbing():
    sg.check_plumbing(DEV)


def test_reruns_are_bit_identical():
    est, ref, sr = mg.case_signals("stereo44100")
    for ext in (False, True):
        a = sg.kernel_grad(est, ref, sr, ext, DEV)[1]
        b = sg.kernel_grad(est, ref, sr, ext, DEV)[1]
        assert torch.equal(a, b)


def test_full_size_batch_matches_float64():
    B, C, sr = 64, 2, 44100
    T = 10 * sr
    clips = np.stack([np.stack([mg.speech(sr, T, 8 * i + c, ((2.0 + 0.3 * i, 3.0 + 0.3 * i),)) for c in range(C)])
                      for i in range(8)])
    ref = np.tile(clips, (B // 8, 1, 1))
    g = np.random.default_rng(0)
    gains = np.float32(10.0) ** (g.uniform(-2, 0.5, size=(B, 1, 1)).astype(np.float32))
    est = (ref + gains * np.float32(0.3) * g.standard_normal(ref.shape, dtype=np.float32)).astype(np.float32)
    for ext in (False, True):
        loss, gk = sg.kernel_grad(est, ref, sr, ext, DEV)
        assert torch.equal(gk, sg.kernel_grad(est, ref, sr, ext, DEV)[1])
        for b in range(0, B, 21):  # items 0, 21, 42, 63
            g64 = -sg.grad64(est[b:b + 1], ref[b:b + 1], sr, ext, DEV)[0]
            gb = gk[b].double()
            assert float(torch.linalg.norm(gb - g64) / torch.linalg.norm(g64)) <= sg.GLOBAL_TOL, (b, ext)
            assert float((gb - g64).abs().max()) <= sg.ROW_TOL * float(g64.abs().max()), (b, ext)
