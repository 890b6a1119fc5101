"""The checks of tests/test_gpu_elementwise.py on the CPU-simulated build of the kernels (tests/cusim): the per-item
element-wise effects bit for bit against a float32 NumPy restatement, on both branches of their walk."""
import pytest

import tests.test_gpu_elementwise as G
from tests.cusim.sim_engine import sim_engine


@pytest.fixture
def eng(monkeypatch):
    monkeypatch.setattr(G, "DEV", "cpu")
    return sim_engine()


@pytest.mark.parametrize("off", [0, 1])
@pytest.mark.parametrize("T", G.LENGTHS)
def test_elementwise_against_float32(eng, T, off):
    G.check_elementwise(eng, T, off)
