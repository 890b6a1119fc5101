"""The fused spectral losses (``spectral_loss_kernel<LOG2N, MEL>``, csrc/loss.cu) on the H100 (``-m gpu``), per cell
against float64 (tests/loss64.py): dL/dX and dL/dY as the kernel writes them ([rows, F, frames], before the STFT
adjoint) and each loss term, for every window 64 ... 2048 in both modes, at the edges of the tiling (a last tile with
0, 1 or FR - 1 live frames beyond full tiles, one-frame and sub-window lengths, a batch with more tiles than the
persistent grid has CTAs), every padding mode and match_stride, three windows, pow 2 / 1 / 0.5, a clamp level that
clamps about half of the cells, each term alone, 1 mel / a default-like count / the largest accepted count, and the
signals of tests/spectral64.py plus silent stretches, silent rows and x == y rows.  Each error is held to the model's
budget and to 2x torch's FP32 arithmetic (torch.stft on cuFFT, the same loss) on the same input; then the exact
properties the kernel's design gives, bit for bit.  tests/probes/loss_accuracy_probe.py prints the table of
DESIGN.md "Loss accuracy"."""
import pytest
import torch

from tests import loss64 as L
from tests import spectral64 as s64

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
WINDOWS = [64, 128, 256, 512, 1024, 2048]
FR = {64: 256, 128: 128, 256: 64, 512: 32, 1024: 16, 2048: 8}  # WPlan<LOG2N>::FR: frames per tile
# the simulator's run (tests/test_sim_loss_accuracy.py) caps the row length and picks four rows per case
MAX_T = None
SIM_KINDS = None


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


def _T(nf, hop, n):
    """A length with nf frames under centred framing (no extra padding)."""
    return max((nf - 1) * hop + hop // 2, n // 2 + 1)


def _mel(eng, n, hop, j):
    """j = 0: 1 mel; 1: a default-like count with fmin / fmax set; 2: the largest count accepted for the window and
    hop."""
    if j == 0:
        return (16000, 1, 0.0, None)
    if j == 1:
        return (16000, 40, 20.0, 7600.0) if n == 64 else (44100, 150, 30.0, 16000.0) if n >= 1024 else \
            (16000, 80, 20.0, 7600.0)
    return (44100, L.max_mels(eng, n, hop), 0.0, None)


def _half_eps(x, n, hop, w, geo, mel):
    """A clamp level that clamps about half of the cells of the first row."""
    r = L.reference(x[:1], x[:1], n, hop, w, geo, L.mel_tables(mel, n, x.device)[0] if mel else None)
    v = r["vx"]
    return float(v[v > 0].median())


def cases(eng, n, mel_mode):
    """(name, kinds, T, hop, window, pad mode, match_stride, mel, options) of one window and mode: every row kind on
    the H100, four per case on the simulator."""
    fr, q = FR[n], n // 4
    odd = q + 1
    kinds_of = (lambda i: SIM_KINDS[i % len(SIM_KINDS)]) if SIM_KINDS else (lambda i: L.KINDS)
    out = [
        ("full tiles", 0, q, "hann", "reflect", False, fr, 1, dict()),
        ("1 live frame", 1, odd, "sqrt_hann", "constant", False, fr + 1, 0, dict(pow=1.0, mag_weight=0.0)),
        ("FR-1 live", 2, n, "random", "replicate", False, 2 * fr - 1, 2, dict(pow=0.5, clamp_eps="half",
                                                                               log_weight=0.5, mag_weight=2.0)),
        ("match_stride", 3, q, "hann", "reflect", True, fr + 3, 1, dict(clamp_eps="half", log_weight=0.0)),
        ("replicate ms", 4, odd, "random", "replicate", True, 3 * fr // 2, 2, dict(pow=1.0)),
        ("constant ms", 5, q, "sqrt_hann", "constant", True, fr - 1, 0, dict(pow=0.5)),
        # the shortest lengths: one frame (hop = n, T = n/2 + 1; constant match_stride at T = 1) and T < n_fft
        ("one frame", 6, n, "hann", "reflect", False, 1, 2, dict()),
        ("one frame T=1", 7, q, "hann", "constant", True, 1, 0, dict()),
        ("T<n replicate", 8, q, "hann", "replicate", False, 0, 1, dict(pow=1.0)),
        ("T<n constant", 9, odd, "random", "constant", False, 0, 2, dict(log_weight=0.0)),
    ]
    res = []
    for name, i, hop, wname, pt, ms, nf, j, opt in out:
        T = {"one frame": n // 2 + 1, "one frame T=1": 1, "T<n replicate": n // 2 + 3, "T<n constant": n - 5}.get(
            name, _T(nf, hop, n))
        if MAX_T is not None and T > MAX_T:  # the simulator: a shorter hop keeps the frame count
            hop = max(1, (MAX_T - n) // nf) | (hop & 1)
            T = _T(nf, hop, n)
        res.append((name, kinds_of(i), T, hop, wname, pt, ms, _mel(eng, n, hop, j) if mel_mode else None, opt))
    return res


def run_case(eng, n, case, dev):
    name, kinds, T, hop, wname, pt, ms, mel, opt = case
    x, y = L.batch(n, hop, T, kinds)
    x, y = x.to(dev), y.to(dev)
    w = s64.windows(n, dev)[wname]
    right_pad, pad = s64.padding(T, n, hop, ms)
    geo = (pad, right_pad, pt, 2 if ms else 0)
    opt = dict(opt)
    if opt.get("clamp_eps") == "half":
        opt["clamp_eps"] = _half_eps(x, n, hop, w, geo, mel)
    return L.check(eng, x, y, n, hop, w, geo, mel, kinds=kinds, **opt)


@pytest.mark.parametrize("mode", ["stft", "mel"])
@pytest.mark.parametrize("n_fft", WINDOWS)
def test_cells_and_terms_against_float64(eng, n_fft, mode):
    """Every case of ``cases``: each kept cell of dL/dX and dL/dY within the model's budget and 2x torch's FP32 error,
    each term's value within its budget and 2x torch's, the dropped share of noise cells <= 1 %, every dropped cell
    matching a branch float64 gives, and x == y rows with a gradient of exactly 0."""
    for case in cases(eng, n_fft, mode == "mel"):
        out = run_case(eng, n_fft, case, DEV)
        L.assert_within(out, mode, (n_fft, mode) + case[:1] + case[2:4])


@pytest.mark.parametrize("mode", ["stft", "mel"])
@pytest.mark.parametrize("n_fft", WINDOWS)
def test_long_rows_and_empty_bands(eng, n_fft, mode):
    """Rows of 3 s at hop n/4 (noise, and noise with a silent stretch); the mel mode at 16 kHz with empty and one-bin
    bands (512 with 160 mels, 64 with 40)."""
    hop = n_fft // 4
    T = 3 * 44100
    mel = None
    if mode == "mel":
        mel = {512: (16000, 160, 0.0, None), 64: (16000, 40, 0.0, None)}.get(n_fft, (16000, 80, 0.0, 8000.0))
    kinds = ("noise", "gap", "noise_1e-3")
    x, y = L.batch(n_fft, hop, T, kinds)
    w = s64.windows(n_fft, DEV)["hann"]
    out = L.check(eng, x.to(DEV), y.to(DEV), n_fft, hop, w, mel=mel, kinds=kinds)
    L.assert_within(out, mode, (n_fft, mode, "3 s"))
    if mel is not None and n_fft in (512, 64):
        lo, hi = L.mel_tables(mel, n_fft, "cpu")[1:]
        assert int(((hi - lo) <= 1).sum()) > 0


@pytest.mark.parametrize("mode", ["stft", "mel"])
@pytest.mark.parametrize("n_fft", WINDOWS)
def test_persistent_grid_loops_over_tiles(eng, n_fft, mode):
    """rows x n_tiles > 8 x SMs: every CTA of the persistent grid walks several tiles; the per-cell budget on a strided
    subset of the rows."""
    hop = n_fft // 4
    T = 44100
    nf = 1 + T // hop
    tiles = -(-nf // FR[n_fft])
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows = -(-(8 * sms + 1) // tiles)
    rows = 1 << (rows - 1).bit_length()
    assert rows * tiles > 8 * sms
    g = torch.Generator().manual_seed(n_fft)
    x = torch.randn(rows, 1, T, generator=g).to(DEV)
    y = torch.randn(rows, 1, T, generator=g).to(DEV)
    w = s64.windows(n_fft, DEV)["hann"]
    mel = (44100, 40 if n_fft == 64 else 80, 0.0, None) if mode == "mel" else None
    sub = slice(3, rows, max(1, rows // 8))
    out = L.check(eng, x, y, n_fft, hop, w, mel=mel, rows=sub, kinds=["noise"] * rows)
    L.assert_within(out, mode, (n_fft, mode, rows, tiles))


# --------------------------------------------------------------------------- exact properties, bit for bit
def _setup(eng, n, mel_mode, rows=2, T=None, seed=0, dev=None):
    dev = dev or DEV
    hop = n // 4
    T = T or _T(2 * FR[n] + 3, hop, n)
    if MAX_T is not None:
        T = min(T, MAX_T)
    g = torch.Generator().manual_seed(seed + n)
    x = torch.randn(rows, 1, T, generator=g).to(dev)
    y = torch.randn(rows, 1, T, generator=g).to(dev)
    tab = L.mel_tables((16000, 40, 0.0, None), n, dev) if mel_mode else None
    return x, y, hop, s64.windows(n, dev)["hann"], tab


@pytest.mark.parametrize("mode", ["stft", "mel"])
@pytest.mark.parametrize("n_fft", WINDOWS)
def test_swap_symmetry(eng, n_fft, mode):
    """loss(x, y) == loss(y, x) and dL/dY(x, y) == dL/dX(y, x): the two FFTs run the same instruction sequence and the
    terms are symmetric under negation.  The only direct check of the third-FFT dL/dY path."""
    x, y, hop, w, tab = _setup(eng, n_fft, mode == "mel")
    for kw in (dict(), dict(pow=0.5, log_weight=0.5, mag_weight=2.0)):
        a = eng.spectral_loss(x, y, n_fft, hop, w, mel=tab, want_grad_x=True, want_grad_y=True, **kw)
        b = eng.spectral_loss(y, x, n_fft, hop, w, mel=tab, want_grad_x=True, want_grad_y=True, **kw)
        assert torch.equal(a[0], b[0]), (n_fft, mode, kw)
        assert torch.equal(a[2], b[1]) and torch.equal(a[1], b[2]), (n_fft, mode, kw)


@pytest.mark.parametrize("mode", ["stft", "mel"])
@pytest.mark.parametrize("n_fft", WINDOWS)
def test_rows_are_independent(eng, n_fft, mode, R=8):
    """In a launch of R = 2^m distinct rows, row r's gradients are 2^-m x those of row r alone (numel scales by 2^m,
    so the weights / numel scale exactly)."""
    x, y, hop, w, tab = _setup(eng, n_fft, mode == "mel", rows=R)
    _, gX, gY = eng.spectral_loss(x, y, n_fft, hop, w, mel=tab, want_grad_x=True, want_grad_y=True)
    for r in range(R):
        _, ax, ay = eng.spectral_loss(x[r:r + 1], y[r:r + 1], n_fft, hop, w, mel=tab, want_grad_x=True,
                                      want_grad_y=True)
        assert torch.equal(gX[r:r + 1], ax / R) and torch.equal(gY[r:r + 1], ay / R), (n_fft, mode, r)


@pytest.mark.parametrize("mode", ["stft", "mel"])
@pytest.mark.parametrize("n_fft", WINDOWS)
def test_tile_phase_is_exact(eng, n_fft, mode):
    """x and y both delayed by s hop (s not a multiple of FR) in the same length: the interior frames' gradients are
    equal and shifted by s frames, though each frame sits in another slot of another tile."""
    x, y, hop, w, tab = _setup(eng, n_fft, mode == "mel", rows=1)
    T = x.shape[-1]
    _, gX, gY = eng.spectral_loss(x, y, n_fft, hop, w, mel=tab, want_grad_x=True, want_grad_y=True)
    N = gX.shape[-1]
    edge = n_fft // hop
    for s in (1, FR[n_fft] - 1, FR[n_fft] + 3):
        if N - 2 * edge - s < 2:
            continue
        xs = torch.cat([torch.randn(1, 1, s * hop, device=x.device), x[..., :T - s * hop]], -1)
        ys = torch.cat([torch.randn(1, 1, s * hop, device=x.device), y[..., :T - s * hop]], -1)
        _, bX, bY = eng.spectral_loss(xs, ys, n_fft, hop, w, mel=tab, want_grad_x=True, want_grad_y=True)
        keep = slice(edge, N - edge - s)
        sh = slice(edge + s, N - edge)
        assert torch.equal(bX[..., sh], gX[..., keep]) and torch.equal(bY[..., sh], gY[..., keep]), (n_fft, mode, s)


@pytest.mark.parametrize("mode", ["stft", "mel"])
@pytest.mark.parametrize("n_fft", WINDOWS)
def test_requests_are_independent(eng, n_fft, mode):
    """The loss is the same with no gradient, dL/dX only, dL/dY only or both; each gradient is the same whether or not
    the other is asked."""
    x, y, hop, w, tab = _setup(eng, n_fft, mode == "mel")
    l0, _, _ = eng.spectral_loss(x, y, n_fft, hop, w, mel=tab)
    l1, gx1, _ = eng.spectral_loss(x, y, n_fft, hop, w, mel=tab, want_grad_x=True)
    l2, _, gy2 = eng.spectral_loss(x, y, n_fft, hop, w, mel=tab, want_grad_y=True)
    l3, gx3, gy3 = eng.spectral_loss(x, y, n_fft, hop, w, mel=tab, want_grad_x=True, want_grad_y=True)
    assert torch.equal(l0, l1) and torch.equal(l0, l2) and torch.equal(l0, l3), (n_fft, mode)
    assert torch.equal(gx1, gx3) and torch.equal(gy2, gy3), (n_fft, mode)


@pytest.mark.parametrize("mode", ["stft", "mel"])
@pytest.mark.parametrize("n_fft", WINDOWS)
def test_magnitude_only_scaling_is_exact(eng, n_fft, mode):
    """log_weight = 0: L(2^k x, 2^k y) = 2^k L(x, y) and dL/dX, dL/dY unchanged, for k in [-20, 20] (the FFT, |X| and
    the mel scale exactly; the magnitude term's derivative is a sign)."""
    x, y, hop, w, tab = _setup(eng, n_fft, mode == "mel")
    kw = dict(mel=tab, log_weight=0.0, want_grad_x=True, want_grad_y=True)
    l0, gx0, gy0 = eng.spectral_loss(x, y, n_fft, hop, w, **kw)
    for k in (-20, -7, -1, 1, 5, 20):
        s = 2.0 ** k
        lk, gxk, gyk = eng.spectral_loss(x * s, y * s, n_fft, hop, w, **kw)
        assert torch.equal(lk, l0 * s) and torch.equal(gxk, gx0) and torch.equal(gyk, gy0), (n_fft, mode, k)
