"""``Engine.loudness_stats`` / ``AudioSignal.loudness_stats`` on the H100 (``-m gpu``): EBU R128 statistics
(csrc/lufs.cu ``loudness_stats_kernel`` behind the shared K-weighting pass).

* I is bit-identical to ``Engine.lufs``, and a statistics call leaves ``Engine.lufs`` bit-identical after it;
* the momentary and short-term series agree with a float64 restatement (tests/loudness_stats64.py) within the
  per-block K-weighting budget of tests/timedomain64.py;
* the gating and the nearest-rank selection are exact: the LRA fields equal a float64 recomputation from the kernel's
  own short-term series (ties, n = 1, nothing above -70, items under 3 s, silent and loud items in one batch, a row of
  >= 100 k blocks whose selection runs from the workspace);
* EBU Tech 3342 cases 1-4 (LRA 10, 5, 20, 15 LU) at 48 kHz within 0.01 LU.
tests/test_sim_loudness_stats.py runs the same checks at smaller sizes on the CPU simulator."""
import math

import numpy as np
import pytest
import torch

import tests.test_gpu_timedomain_accuracy as TDA
from tests import loudness_stats64 as ls
from tests import timedomain64 as td

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


def _np(t):
    return t.detach().cpu().double().numpy()


def _batch(sr, T, C, names, seed=0):
    sig = TDA.kw_signals(sr, T, seed)
    return np.stack([np.stack([sig[n] * (1.0 - 0.1 * c) for c in range(C)]) for n in names]).astype(np.float32)


# --------------------------------------------------------------------------- bit identity with Engine.lufs
def check_integrated_identity(eng, sr, C, T, Tp=None):
    x = torch.from_numpy(_batch(sr, T, C, ["noise", "sin30+noise", "noise_1e-6"])).to(DEV)
    x = torch.cat([x, torch.zeros_like(x[:1])])  # a silent item: -inf
    before = eng.lufs(x, sr, padded_length=Tp, want_blocks=True)
    for series in (False, True):
        st = eng.loudness_stats(x, sr, padded_length=Tp, want_series=series)
        assert torch.equal(st["I"], before["lufs"]), (sr, C, T, series)
        after = eng.lufs(x, sr, padded_length=Tp, want_blocks=True)
        assert torch.equal(after["lufs"], before["lufs"]) and torch.equal(after["blocks"], before["blocks"])
    assert st["I"][-1].item() == -math.inf and st["I Threshold"][-1].item() == -math.inf


@pytest.mark.parametrize("sr,C,T", [(16000, 1, 16000 * 5 + 77), (44100, 2, 441000), (48000, 5, 48000 * 4),
                                    (11025, 2, 11025 * 7 + 3), (22050, 1, 22050 * 2)])
def test_integrated_is_bit_identical(eng, sr, C, T):
    check_integrated_identity(eng, sr, C, T)


def test_integrated_is_bit_identical_padded(eng):
    check_integrated_identity(eng, 44100, 2, 30000, Tp=44100 * 4)


# --------------------------------------------------------------------------- series against float64
def check_series(eng, sr, C, T, names):
    x = _batch(sr, T, C, names)
    out = eng.loudness_stats(torch.from_numpy(x).to(DEV), sr, want_series=True)
    m, s = _np(out["momentary"]), _np(out["short_term"])
    m64, s64 = ls.momentary64(x, sr), ls.short_term64(x, sr)
    assert m.shape == m64.shape and s.shape == s64.shape == (len(names), ls.num_short_term(T, sr))
    assert s.shape[1] > 0
    for b, name in enumerate(names):
        rel = td.kweight_budget(sr, name) * td.U  # relative energy error per block
        # momentary: float32 z (one more rounding) and a float32 result; short-term: a float32 result
        tm = ls.DB_PER_REL * (rel + td.U) + ls.ulp32(m64[b])
        ts = ls.DB_PER_REL * rel + ls.ulp32(s64[b])
        assert np.all(np.abs(m[b] - m64[b]) <= tm), (sr, C, name, np.abs(m[b] - m64[b]).max())
        assert np.all(np.abs(s[b] - s64[b]) <= ts), (sr, C, name, np.abs(s[b] - s64[b]).max())
    return out


@pytest.mark.parametrize("C", [1, 2, 5])
@pytest.mark.parametrize("sr", [16000, 44100, 48000])
def test_series_against_float64(eng, sr, C):
    check_series(eng, sr, C, int(4.5 * sr), ["noise", "sin30+noise", "sin20+noise"])


# --------------------------------------------------------------------------- gating and ranks, exactly
def check_lra_exact(out):
    """The LRA fields of every item equal lra64 of the item's own short-term series; returns the kept counts."""
    S = _np(out["short_term"])
    ns = []
    for b in range(S.shape[0]):
        want = ls.lra64(S[b])
        for k in ("LRA", "LRA Low", "LRA High"):
            assert out[k][b].item() == want[k], (b, k, out[k][b].item(), want[k])
        # the threshold is float64 arithmetic rounded to a float32 output: 1e-6 LU on top of that rounding
        got_thr, want_thr = out["LRA Threshold"][b].item(), want["LRA Threshold"]
        assert (got_thr == want_thr == -math.inf) or abs(got_thr - want_thr) <= 1e-6 + 0.5 * ls.ulp32(want_thr), (
            b, got_thr, want_thr)
        ns.append(want["n"])
    return ns


def gating_cases(sr):
    """[B, 2, T] float32 and names: level steps (ties on every plateau), a noisy level ramp (no ties), every block
    below -70, silence."""
    T = int(12 * sr)
    t = np.arange(T) / sr
    g = np.random.default_rng(sr)
    sine = np.sin(2 * np.pi * 1000.0 * t)
    items = {"steps": np.where(t < 4, 0.01, np.where(t < 8, 0.3, 0.05)) * sine,
             "ramp": (10.0 ** (-3 + 2.9 * t / t[-1])) * g.standard_normal(T),
             "below_-70": 1e-5 * g.standard_normal(T),
             "silence": np.zeros(T)}
    x = np.stack([np.stack([v, 0.9 * v]) for v in items.values()]).astype(np.float32)
    return x, list(items)


def check_gating(eng, sr):
    """Loud, stepped, quiet and silent items in one batch, each checked on its own series; then n = 1."""
    x, names = gating_cases(sr)
    out = eng.loudness_stats(torch.from_numpy(x).to(DEV), sr, want_series=True)
    ns = dict(zip(names, check_lra_exact(out)))
    steps = _np(out["short_term"])[names.index("steps")]
    assert steps.size - len(np.unique(steps)) >= 5  # the plateaus tie
    assert ns["steps"] > 10 and ns["ramp"] > 10
    assert ns["below_-70"] == ns["silence"] == 0
    for name in ("below_-70", "silence"):
        b = names.index(name)
        assert out["LRA"][b].item() == 0.0
        assert all(out[k][b].item() == -math.inf for k in ("LRA Threshold", "LRA Low", "LRA High"))
    assert out["I"][names.index("silence")].item() == -math.inf
    # exactly one short-term block: n = 1, Low = High, LRA = 0
    T = 30 * td.kweight_geometry(sr, sr)[1]
    one = eng.loudness_stats(torch.from_numpy(_batch(sr, T, 2, ["noise"])).to(DEV), sr, want_series=True)
    assert one["short_term"].shape == (1, 1) and check_lra_exact(one) == [1]
    assert one["LRA"].item() == 0.0 and one["LRA Low"].item() == one["LRA High"].item() == one["short_term"].item()
    return out


@pytest.mark.parametrize("sr", [16000, 48000])
def test_gating_and_ranks_exact(eng, sr):
    check_gating(eng, sr)


def check_short_items(eng, sr):
    """Items under 3 s: n_st = 0, LRA = 0, the rest -inf, I still the integrated loudness; under 0.5 s the engine
    reads the zero extension like loudness()."""
    for T, Tp in ((int(2.9 * sr), None), (int(0.3 * sr), int(0.5 * sr))):
        x = torch.from_numpy(_batch(sr, T, 2, ["noise", "sin30+noise"])).to(DEV)
        out = eng.loudness_stats(x, sr, padded_length=Tp, want_series=True)
        assert out["short_term"].shape == (2, 0)
        assert torch.equal(out["I"], eng.lufs(x, sr, padded_length=Tp)["lufs"])
        assert (out["LRA"] == 0).all() and torch.isinf(out["LRA Low"]).all() and torch.isinf(out["LRA High"]).all()
        assert torch.isinf(out["LRA Threshold"]).all() and torch.isfinite(out["I Threshold"]).all()


def test_short_items(eng):
    check_short_items(eng, 44100)


def test_long_row_selection_from_workspace(eng):
    """A row of > 100 k short-term blocks (2.8 h at 8 kHz): the keys do not fit in shared memory and the selection
    runs from the workspace, still exact."""
    sr = 8000
    T = 800 * 100_100 + 30 * 800
    g = torch.Generator(device=DEV).manual_seed(3)
    env = 10.0 ** (-2.5 + 2.0 * torch.sin(torch.arange(T, device=DEV, dtype=torch.float64) * (2 * math.pi / (sr * 977))))
    x = (env * torch.randn(T, device=DEV, generator=g, dtype=torch.float64)).float().reshape(1, 1, T)
    del env
    out = eng.loudness_stats(x, sr, want_series=True)
    assert out["short_term"].shape[1] > 100_000
    ns = check_lra_exact(out)
    assert ns[0] > 8192


# --------------------------------------------------------------------------- EBU Tech 3342
def check_ebu3342(eng, case, sr, seg_s):
    x, want = ls.ebu3342(case, sr, seg_s)
    out = eng.loudness_stats(torch.from_numpy(x).to(DEV), sr, want_series=True)
    check_lra_exact(out)
    got = out["LRA"].item()
    assert abs(got - want) <= 0.01, (case, sr, got, want)


@pytest.mark.parametrize("case", [1, 2, 3, 4])
def test_ebu3342_loudness_range(eng, case):
    check_ebu3342(eng, case, 48000, 20.0)


# --------------------------------------------------------------------------- the AudioSignal method
def check_signal_method(sr):
    """Keys, shapes, series, the deferred normalize() gain, no cache touched, other filter classes raise."""
    from audiotools_b200 import AudioSignal
    from audiotools_b200.engine import get_engine

    eng = get_engine()
    x = torch.from_numpy(_batch(sr, int(3.5 * sr), 2, ["noise", "sin30+noise"]))
    sig = AudioSignal(x.clone(), sr).to(DEV)
    st = sig.loudness_stats()
    assert list(st) == ["I", "I Threshold", "LRA", "LRA Threshold", "LRA Low", "LRA High"]
    assert all(v.shape == (2,) and v.dtype == torch.float32 and v.device == sig.device for v in st.values())
    assert sig._loudness is None  # loudness() was not filled
    spec = sig.stft()
    st2 = sig.loudness_stats(series=True)
    assert sig.stft_data is spec and sig._loudness is None
    assert st2["momentary"].shape == (2, eng.lib.b2a_lufs_num_blocks(x.shape[-1], float(sr), 0.4))
    assert st2["short_term"].shape == (2, ls.num_short_term(x.shape[-1], sr))
    for k in st:
        assert torch.equal(st[k], st2[k])
    assert torch.equal(torch.maximum(st["I"], torch.tensor(-70.0, device=sig.device)), sig.loudness())
    # the deferred gain of normalize() is applied first
    sig = AudioSignal(x.clone(), sr).to(DEV)
    sig.normalize(-30.0)
    got = sig.loudness_stats()["I"]
    assert torch.allclose(got, torch.full_like(got, -30.0), atol=1e-3), got
    with pytest.raises(NotImplementedError):
        sig.loudness_stats(filter_class="Fenton/Lee 1")


def test_signal_method(eng):
    check_signal_method(44100)
