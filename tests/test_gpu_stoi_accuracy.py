"""STOI and its backward on the H100 (``-m gpu``), per stage against float64 (tests/stoi64.py): the resampler per
sample at every supported kind of rate (8 kHz upsamples; 12345 and 7999 Hz have 178 853 and 724 387 taps) and around
its 1024-output tiles, the mask per frame around its 256-frame scan chunks, every band envelope at M around the
32-frame tiles and the short-item rule, the score at J * 15 around 256 and J around multiples of 8, and each backward
stage from the kernel's own input to it; end to end against the numpy restatement of pystoi; non-finite inputs;
exact batch, rerun and scaling properties; and a reference row past flat index 2^31.
tests/probes/stoi_accuracy_probe.py prints the table of DESIGN.md "STOI accuracy"."""
import warnings

import numpy as np
import pytest
import torch

from audiotools_b200 import AudioSignal, metrics
from tests import stoi64 as s
from tests import stoi_grad_cases as sg
from tests import stoi_oracle as so

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
KINDS = ["speech", "noise", "tone6", "tone7", "tone218", "tone219", "deep", "silence", "alternate", "burst"]
# kinds whose score is well conditioned: a tone or a band 100 dB down leaves band envelopes 70 to 100 dB under the
# frame's norm, whose float32 relative error (~1e-4, within C_B) moves the score by more than 1e-5; those kinds are
# held per stage
E2E = np.array([k not in ("tone6", "tone7", "tone218", "tone219", "deep") for k in KINDS])


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


def check_case(eng, est, ref, sr, where, backward=True, oracle=True, acc=None, e2e=None):
    """Both modes: every forward stage, the score of the items in ``e2e`` (default all) against the numpy restatement
    of pystoi within 1e-5 (NaN where it is NaN), the kept counts of all, and every backward stage for a random upstream
    gradient."""
    acc = {} if acc is None else acc
    B = est.shape[0]
    e2e = np.ones(B, bool) if e2e is None else e2e
    for ext in (False, True):
        f = s.Forward(eng, est, ref, sr, ext, DEV)
        s.check_forward(f, est, ref, (where, ext), acc)
        if oracle:
            want, kept, _ = so.batch_stoi(est, ref, sr, ext)
            assert np.array_equal(np.isnan(f.score), np.isnan(want)), (where, ext, f.score, want)
            ok = ~np.isnan(want) & e2e
            assert np.abs(f.score[ok] - want[ok]).max(initial=0) < 1e-5, (where, ext, f.score, want)
            assert np.array_equal(f.kept_out, kept), (where, ext, f.kept_out, kept)
        if backward:
            g = np.random.default_rng(B).uniform(-2, 2, B)
            s.check_backward(f, s.Backward(eng, f, g, DEV), (where, ext), acc)
    return acc


def length_for(sr, n10):
    """The shortest input length T at sr whose 10 kHz row has at least n10 samples (exactly n10 when sr >= 10 kHz;
    an upsampling rate skips some lengths)."""
    up, down = s.Engine.stoi_ratio(sr)
    T = ((n10 - 1) * down) // up + 1
    assert -(-T * up // down) >= n10 and (up < down or -(-T * up // down) == n10 or -(-(T - 1) * up // down) < n10)
    return T


# --------------------------------------------------------------------------- every rate, every signal kind
def check_rate(eng, sr, seconds, acc=None):
    C = {8000: 5, 44100: 2, 12345: 2}.get(sr, 1 + (sr // 1000) % 2)
    T = int(seconds * sr) + sr % 7
    est, ref = s.batch(KINDS, sr, T, C, seed=sr)
    return check_case(eng, est, ref, sr, ("rate", sr, C, T), acc=acc, e2e=E2E)


@pytest.mark.parametrize("sr", s.RATES + [7999])
def test_every_stage_at_every_rate(eng, sr):
    check_rate(eng, sr, 2.0)


# --------------------------------------------------------------------------- resampler tiles
N10_EDGES = [257, 385, 1023, 1024, 1025, 2047, 2048, 2049]


def check_resampler_tiles(eng, sr, acc=None):
    acc = {} if acc is None else acc
    for n10 in N10_EDGES:
        T = length_for(sr, n10)
        est, ref = s.batch(["noise", "speech"], sr, T, 2, seed=n10)
        check_case(eng, est, ref, sr, ("tiles", sr, n10), acc=acc)
    return acc


@pytest.mark.parametrize("sr", [8000, 10000, 12345, 44100, 192000, 7999])
def test_resampler_tiles(eng, sr):
    check_resampler_tiles(eng, sr)


def check_input_tiles(eng, sr, acc=None):
    """The transposed FIR's 1024-input tiles: T = 1024 k - 1, 1024 k, 1024 k + 1."""
    acc = {} if acc is None else acc
    k = -(-int(0.5 * sr) // 1024)
    for T in (1024 * k - 1, 1024 * k, 1024 * k + 1):
        est, ref = s.batch(["speech", "noise"], sr, T, 2, seed=T)
        check_case(eng, est, ref, sr, ("input tiles", sr, T), oracle=False, acc=acc)
    return acc


@pytest.mark.parametrize("sr", [8000, 16000, 44100])
def test_gradient_input_tiles(eng, sr):
    check_input_tiles(eng, sr)


# --------------------------------------------------------------------------- mask scan chunks
def mask_patterns(n_fr):
    """10 kHz clean rows with n_fr frames: first frame dropped, last frame dropped, every other frame kept."""
    n10 = s.n10_for(n_fr)
    rows = []
    if n_fr >= 6:
        rows.append(s.bursts_10k(n10, [(2, n_fr - 2)], 1))             # frame 0 dropped
        rows.append(s.bursts_10k(n10, [(0, n_fr - 4)], 2))             # the last frames dropped
        rows.append(s.bursts_10k(n10, [(a, -1) for a in range(2, n_fr, 2)], 3))  # alternating
    rows.append(0.1 * s._noise(n10, 4).astype(np.float32))          # all kept
    return np.stack(rows)[:, None, :]


def check_mask_chunks(eng, n_fr, acc=None):
    """Per stage; end to end except for the alternating row, whose lone clicks leave most band envelopes so far under
    the frame's norm that the float32 spectra move its score (near 0) by ~1e-4."""
    ref = mask_patterns(n_fr)
    est = (ref + np.float32(0.01) * s._noise(ref.size, 5).reshape(ref.shape)).astype(np.float32)
    e2e = np.array([True, True, False, True]) if n_fr >= 6 else None
    return check_case(eng, est, ref, 10000, ("mask", n_fr), acc=acc, e2e=e2e)


@pytest.mark.parametrize("n_fr", [1, 2, 255, 256, 257, 512, 513])
def test_mask_scan_chunks(eng, n_fr):
    check_mask_chunks(eng, n_fr)


# --------------------------------------------------------------------------- band tiles, short-item rule, score
# M around the 32-frame band tiles and the 30-frame short-item rule; J * 15 around 256 (J = 17, 18); J around
# multiples of 8 (J = 7, 9, 63, 65) in the extended score's warp-per-segment loop; and a long row
M_EDGES = [0, 1, 29, 30, 31, 32, 33, 36, 38, 46, 47, 63, 64, 65, 92, 94, 1200]


def check_m(eng, M, acc=None):
    n_fr = max(M + 12, 24)
    n10 = s.n10_for(n_fr)
    rows = [s.bursts_10k(n10, s.spans_for(M, n_fr), 10 + M),
            s.bursts_10k(n10, s.spans_for(M, n_fr, gap=True), 11 + M)]
    rows += [s.bursts_10k(n10, s.spans_for(M, n_fr, gap=k % 2 == 1), 12 + k, tone=k) for k in (6, 7, 218, 219)]
    ref = np.stack(rows)[:, None, :]
    est = (ref + np.float32(0.02) * s._noise(ref.size, M).reshape(ref.shape)).astype(np.float32)
    f = s.Forward(eng, est, ref, 10000, False, DEV)
    assert (f.M == M).all(), (M, f.M)
    return check_case(eng, est, ref, 10000, ("M", M), acc=acc)


@pytest.mark.parametrize("M", M_EDGES)
def test_band_tiles_and_score_shapes(eng, M):
    check_m(eng, M)


# --------------------------------------------------------------------------- non-finite inputs
def nonfinite_batch(sr, bad, value):
    """Three speech items of 1.6 s at sr; item 1's estimate or reference has one `value` sample at T / 2."""
    from tests.golden import make_golden_quality as mg

    T = int(1.6 * sr)
    ref = np.stack([mg.speech(sr, T, 40 + i)[None] for i in range(3)])
    est = np.stack([mg.with_snr(ref[i], 5.0, 50 + i) for i in range(3)])
    (est if bad == "est" else ref)[1, 0, T // 2] = value
    return est, ref


NONFINITE = [(10000, "est", np.nan), (16000, "est", np.inf), (16000, "ref", np.nan), (16000, "ref", np.inf),
             (44100, "est", -np.inf), (8000, "ref", np.nan)]


def check_nonfinite(eng, sr, bad, value):
    """What the restatement of pystoi returns: NaN in both modes for a non-finite estimate (the clean items' kept
    counts unchanged), 1e-5 with one warning and no kept frame for a non-finite reference.  The other items are
    bit-identical to a batch without the bad item, and so are their gradient rows; a bad reference's gradient row is
    0, a bad estimate's is non-finite wherever autograd through the float64 restatement is."""
    est, ref = nonfinite_batch(sr, bad, value)
    good = [0, 2]
    for ext in (False, True):
        want, kept, _ = so.batch_stoi(est, ref, sr, ext)
        e, r = (AudioSignal(torch.from_numpy(v.copy()).to(DEV), sr) for v in (est, ref))
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            v = metrics.quality.stoi(e, r, ext).numpy()
        n_warn = len([x for x in w if "Returning 1e-5" in str(x.message)])
        _, kk, short = eng.stoi(e.audio_data, r.audio_data, sr, ext)
        kk, short = kk.cpu().numpy(), short.cpu().numpy()
        assert np.array_equal(kk, kept), (sr, bad, ext, kk, kept)
        if bad == "est":
            assert np.isnan(want[1]) and np.isnan(v[1]) and n_warn == 0 and not short.any(), (sr, ext, v)
        else:
            assert want[1] == 1e-5 and v[1] == 1e-5 and kk[1] == 0 and n_warn == 1 and short[1], (sr, ext, v, n_warn)
        clean = eng.stoi(torch.from_numpy(est[good]).to(DEV), torch.from_numpy(ref[good]).to(DEV), sr, ext)[0]
        assert torch.equal(torch.from_numpy(v[good]), clean.cpu()), (sr, bad, ext)
        assert np.abs(v[good] - want[good]).max() < 1e-5
        # the loss's gradient
        loss, g = sg.kernel_grad(est, ref, sr, ext, DEV)
        assert torch.equal(loss[good], (-clean).float())
        _, g_clean = sg.kernel_grad(est[good], ref[good], sr, ext, DEV)
        assert torch.equal(g[good], g_clean), (sr, bad, ext)
        if bad == "ref":
            assert torch.equal(g[1], torch.zeros_like(g[1]))
        else:
            g64 = sg.grad64(est[1:2], ref[1:2], sr, ext)[0].numpy()
            gk = g[1].cpu().numpy()
            assert (~np.isfinite(g64)).any()
            assert (~np.isfinite(gk[~np.isfinite(g64)])).all(), (sr, ext, int((~np.isfinite(g64)).sum()),
                                                                   int((~np.isfinite(gk)).sum()))


@pytest.mark.parametrize("sr,bad,value", NONFINITE)
def test_nonfinite_inputs(eng, sr, bad, value):
    check_nonfinite(eng, sr, bad, value)


# --------------------------------------------------------------------------- exact properties
def mixed_m_batch(Ms, seed=0):
    n_fr = max(Ms) + 12
    n10 = s.n10_for(n_fr)
    ref = np.stack([s.bursts_10k(n10, s.spans_for(M, n_fr, gap=i % 2 == 1), seed + i) for i, M in enumerate(Ms)])
    ref = ref[:, None, :]
    est = (ref + np.float32(0.02) * s._noise(ref.size, seed).reshape(ref.shape)).astype(np.float32)
    return est, ref


def check_batch_rows(eng, Ms):
    """Every item of a batch that mixes M = 0 .. max(Ms) equals its single-item call, score and gradient row, bit for
    bit; reruns are identical."""
    est, ref = mixed_m_batch(Ms)
    for ext in (False, True):
        f = s.Forward(eng, est, ref, 10000, ext, DEV)
        assert np.array_equal(f.M, Ms)
        loss, g = sg.kernel_grad(est, ref, 10000, ext, DEV)
        loss2, g2 = sg.kernel_grad(est, ref, 10000, ext, DEV)
        assert torch.equal(loss, loss2) and torch.equal(g, g2)
        for b in range(len(Ms)):
            one = eng.stoi(torch.from_numpy(est[b:b + 1]).to(DEV), torch.from_numpy(ref[b:b + 1]).to(DEV), 10000,
                           ext)[0]
            assert one.item() == f.score[b], (Ms[b], ext)
            _, gb = sg.kernel_grad(est[b:b + 1], ref[b:b + 1], 10000, ext, DEV)
            assert torch.equal(gb[0], g[b]), (Ms[b], ext)


def test_batch_rows_equal_single_items(eng):
    check_batch_rows(eng, [0, 1, 29, 30, 31, 200, 2000, 47])


def check_power_of_two_scaling(eng, sr, T):
    """Scaling either signal by a power of two scales its 10 kHz rows and envelopes exactly and leaves the kept
    lists unchanged, bit for bit; the score moves only through the EPS pystoi adds to its norms, which does not scale
    (<= 1e-12; 8e-14 seen on a tone)."""
    est, ref = s.batch(["speech", "alternate", "tone7"], sr, T, 2, seed=7)
    for ext in (False, True):
        base = s.Forward(eng, est, ref, sr, ext, DEV)
        for ke, kr in ((3, 0), (0, -5), (-7, 9)):
            f = s.Forward(eng, est * np.float32(2.0 ** ke), ref * np.float32(2.0 ** kr), sr, ext, DEV)
            assert all(np.array_equal(a, b) for a, b in zip(f.kept, base.kept))
            assert np.array_equal(f.sig10[0], base.sig10[0] * np.float32(2.0 ** ke))
            assert np.array_equal(f.sig10[1], base.sig10[1] * np.float32(2.0 ** kr))
            for b in range(est.shape[0]):
                M = int(base.M[b])
                assert np.array_equal(f.tob[0, b, :, :M], base.tob[0, b, :, :M] * np.float32(2.0 ** ke))
                assert np.array_equal(f.tob[1, b, :, :M], base.tob[1, b, :, :M] * np.float32(2.0 ** kr))
            assert np.abs(f.score - base.score).max() <= 1e-12, (ke, kr, ext, f.score - base.score)


def test_power_of_two_scaling(eng):
    for sr in (10000, 44100):
        check_power_of_two_scaling(eng, sr, int(1.5 * sr))


# --------------------------------------------------------------------------- flat index past 2^31
def test_reference_rows_past_flat_index_2_31(eng):
    """B = 4 at 10 kHz with T = 3.1e8: the reference rows of sig10 start at flat index 4 T; item 2's row crosses 2^31
    and item 3's lies past it.  Their sig10 (bit for bit: 10 kHz is the mono mix), kept lists and a strided subset of
    their envelopes against float64.  (The backward's scratch at this size is over 40 GB and is not run.)"""
    B, T = 4, 310_000_000
    assert (B + 2) * T < 2 ** 31 < (B + 3) * T
    gen = torch.Generator(device=DEV).manual_seed(0)
    blk = 64 * s.HOP
    env = (torch.arange(T, device=DEV) // blk % 5 != 0).float()  # one silent block in five
    ref = torch.randn(B, 1, T, device=DEV, generator=gen) * 0.1 * env
    est = ref + 0.01 * torch.randn(B, 1, T, device=DEV, generator=gen)
    _, kept, _, ws = eng.stoi(est, ref, 10000, False, return_workspace=True)
    L = s.Layout(B, T, 1, 1)
    assert ws.numel() == L.bytes
    del est
    for b in (2, 3):
        check_long_item(ws, L, b, ref[b, 0].cpu().numpy(), kept[b].item())


def check_long_item(ws, L, b, x, kept_b):
    B = L.B
    x10 = s._view(ws, (B + b) * L.n10 * 4, L.n10, torch.float32, (L.n10,)).cpu().numpy()
    assert np.array_equal(x10, x)
    cnt = s._view(ws, L.off_count, B, torch.int32, (B,)).cpu().numpy()
    kl = s._view(ws, L.off_kept + b * L.n_fr * 4, L.n_fr, torch.int32, (L.n_fr,)).cpu().numpy()[:cnt[b]]
    e64 = np.concatenate([s.energies64(x10[i * s.HOP:(i + 4097) * s.HOP + s.FRAME], min(4096, L.n_fr - i))
                          for i in range(0, L.n_fr, 4096)])
    d = e64.max() - so.DYN_RANGE - e64
    assert np.abs(d).min() > s.THRESH_DB
    assert np.array_equal(kl, np.nonzero(d < 0)[0]) and kept_b == cnt[b]
    M = int(cnt[b]) - 1
    tob_off = L.off_tob + ((B + b) * s.NBAND) * L.n_fr * 4
    tob = s._view(ws, tob_off, s.NBAND * L.n_fr, torch.float32, (s.NBAND, L.n_fr)).cpu().numpy()
    for i in list(range(0, M, 99_991)) + [M - 1]:
        lo = max(i - 1, 0)
        fr = s.stoi_frames64(x10, kl[lo:i + 3])[i - lo:i - lo + 1]
        t64, _, nX = s.tob64(fr)
        assert np.abs(tob[:, i] - t64[:, 0]).max() <= s.C_B * s.U * nX[0], i
