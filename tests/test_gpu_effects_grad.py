"""Gradients through the time-domain effects on the H100 (``-m gpu``): resample, equalizer, convolve, apply_ir,
ensure_max_of_audio against torch.autograd over the reference's arithmetic in float64 on the same GPU
(tests/effects_grad_cases.py), full-size cases, bit-identical reruns, no torch convolution / FFT call on either pass,
and the reference's own list of methods that must carry a gradient (ref:tests/core/test_grad.py)."""
import pytest
import torch

from tests import effects_grad_cases as ec
from tests.conftest import elementwise_ok, rel_err

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TOL = 1e-4


@pytest.fixture(scope="module")
def at():
    import __graft_entry__ as graft

    graft.build()
    import audiotools_b200

    return audiotools_b200


def _x(shape, seed, scale=0.5):
    return ec.x_of(shape, seed, scale).to(DEV)


def _ir(B, L, seed, C=1):
    return ec.synthetic_ir(B, L, seed, C=C).to(DEV)


class _NoTorchConv:
    """F.conv1d / F.conv_transpose1d / torch.fft.* raise inside the block: neither pass may delegate to them."""

    FFT = ("rfft", "irfft", "fft", "ifft")

    def __enter__(self):
        F = torch.nn.functional
        self.saved = (F.conv1d, F.conv_transpose1d, {n: getattr(torch.fft, n) for n in self.FFT})

        def forbidden(*a, **k):
            raise AssertionError("torch convolution / FFT called")

        F.conv1d = F.conv_transpose1d = forbidden
        for n in self.FFT:
            setattr(torch.fft, n, forbidden)

    def __exit__(self, *exc):
        F = torch.nn.functional
        F.conv1d, F.conv_transpose1d, fft = self.saved
        for n, f in fft.items():
            setattr(torch.fft, n, f)


def _cases():
    out = [("resample", old, dict(new_sr=new), T) for old, new in ec.RESAMPLE_RATES for T in ec.RESAMPLE_LENGTHS]
    out += [("equalizer", 44100, dict(db=ec.db_curve(n, 6, T)), T) for T in ec.EQ_LENGTHS for n in (1, 2)]
    out += [("convolve", 44100, dict(ir=_ir(b, L, L), start_at_max=s), 2000)
            for L, b, s in [(300, 2, True), (3000, 2, True), (300, 1, True), (300, 2, False)]]
    out += [("apply_ir", 44100, dict(ir=_ir(2, L, L + 1)), 2000) for L in (300, 3000)]
    out += [("ensure_max_of_audio", 44100, dict(max=0.5), 1000)]
    return out


def test_effect_grads_match_autograd(at):
    for method, sr, kw, T in _cases():
        x = _x((2, 2, T), T + sr)
        with _NoTorchConv():
            y = ec.ours(method, sr, **kw)(x)
            g = _x(y.shape, T + 1, 1.0)
            gx = ec.vjp(ec.ours(method, sr, **kw), x, g)
        want = ec.vjp(ec.ref(method, sr, **kw), x.double(), g)
        assert rel_err(gx, want) < TOL, (method, sr, T, rel_err(gx, want))
        if method == "resample":
            # the taps are designed on the device (float32 torch trig there): up to 5e-6 from the CPU design, and the
            # forward uses the same taps, so the per-cell check runs against float64 autograd with those taps
            want = ec.vjp(lambda v: _resample64(v, sr, kw["new_sr"]), x.double(), g)
        assert elementwise_ok(gx.cpu(), want.cpu(), frame_dim=-1), (method, sr, T)


def test_grads_match_reference_golden(at):
    """Every case of tests/golden/make_golden_effects_grad.py (incl. apply_ir with drr + ir_eq and with
    use_original_phase, mix with other_eq) against the REAL reference's gradients, on the H100."""
    ec.check_golden(ec.load_golden(), DEV)


def test_resample_tiny_rows_and_large_new_rate(at):
    """T = 1 and T = 2 when upsampling (the edge kernel alone), and 11025 -> 96000 (reduced 147 -> 1280: phase tiles),
    against float64 autograd with the engine's taps."""
    for old, new, T in [(16000, 44100, 1), (16000, 44100, 2), (11025, 96000, 700)]:
        x = _x((2, 2, T), T)
        y = ec.ours("resample", old, new_sr=new)(x)
        g = _x(y.shape, T + 1, 1.0)
        gx = ec.vjp(ec.ours("resample", old, new_sr=new), x, g)
        want = ec.vjp(lambda v: _resample64(v, old, new), x.double(), g)
        assert rel_err(gx, want) < TOL and elementwise_ok(gx.cpu(), want.cpu(), frame_dim=-1), (old, new, T)


def _resample64(x, old_sr, new_sr):
    """julius.resample_frac's arithmetic in float64 with the engine's own (device-designed) taps."""
    from audiotools_b200.engine import get_engine

    kt, width, old, new = get_engine()._resample_kernel(old_sr, new_sr, x.device)
    T = x.shape[-1]
    v = torch.nn.functional.pad(x.reshape(-1, 1, T), (width, width + old), mode="replicate")
    ys = torch.nn.functional.conv1d(v, kt.t().double()[:, None, :], stride=old)
    return ys.transpose(1, 2).reshape(*x.shape[:-1], -1)[..., : new * T // old]


@pytest.mark.parametrize("method", ["resample", "equalizer", "apply_ir"])
def test_full_size_against_float64_on_a_row_subset(at, method):
    """64 items x 2 channels x 10 s at 44.1 kHz (the benchmark's shape); the float64 reference on every 8th item."""
    B, T, sr = 64, 441000, 44100
    x = _x((B, 2, T), 1, 0.1)
    kw = {"resample": dict(new_sr=16000), "equalizer": dict(db=ec.db_curve(B, 6, 2).to(DEV)),
          "apply_ir": dict(ir=_ir(B, sr, 3))}[method]
    y = ec.ours(method, sr, **kw)(x)
    g = _x(y.shape, 4, 1.0)
    gx = ec.vjp(ec.ours(method, sr, **kw), x, g)
    sub = slice(None, None, 8)
    kws = {k: (v[sub] if torch.is_tensor(v) and v.shape[0] == B else v) for k, v in kw.items()}
    want = ec.vjp(ec.ref(method, sr, **kws), x[sub].double(), g[sub])
    assert rel_err(gx[sub], want) < TOL, rel_err(gx[sub], want)


def test_bit_identical_reruns(at):
    for method, sr, kw in [("resample", 44100, dict(new_sr=16000)), ("resample", 44100, dict(new_sr=22050)),
                           ("equalizer", 44100, dict(db=ec.db_curve(4, 6, 1))),
                           ("apply_ir", 44100, dict(ir=_ir(4, 4410, 2)))]:
        x = _x((4, 2, 44100), 5, 0.2)
        y = ec.ours(method, sr, **kw)(x)
        g = _x(y.shape, 6, 1.0)
        a = ec.vjp(ec.ours(method, sr, **kw), x, g)
        b = ec.vjp(ec.ours(method, sr, **kw), x, g)
        assert torch.equal(a, b), method


def test_reference_audio_grad_method_list(at):
    """ref:tests/core/test_grad.py::test_audio_grad replayed on this AudioSignal: the methods this package
    differentiates produce a gradient; those without a backward raise NotImplementedError instead of returning a
    detached result."""
    from audiotools_b200 import AudioSignal

    sr = 44100
    base = _x((1, 1, sr), 7, 0.1)
    ir = AudioSignal(_ir(1, 4410, 8), sr)
    with_grad = [
        ("mix", {"other": AudioSignal(_x((1, 1, sr), 9, 0.1), sr), "snr": 0}),
        ("convolve", {"other": ir}),
        ("apply_ir", {"ir": ir, "drr": 0.1, "ir_eq": torch.randn(6, generator=torch.Generator().manual_seed(0))}),
        ("ensure_max_of_audio", {}),
        ("normalize", {}),
        ("volume_change", {"db": 1}),
        ("equalizer", {"db": torch.randn(6, generator=torch.Generator().manual_seed(1))}),
        ("quantization", {"quantization_channels": 8}),
        ("mulaw_quantization", {"quantization_channels": 8}),
        ("resample", {"sample_rate": 16000}),
    ]
    for name, kw in with_grad:
        x = base.clone().requires_grad_()
        sig = AudioSignal(x, sr)
        out = getattr(sig.clone(), name)(**kw)
        out.audio_data.sum().backward()
        assert x.grad is not None and torch.isfinite(x.grad).all(), name
    for name, kw in [("low_pass", {"cutoffs": 1000}), ("high_pass", {"cutoffs": 1000}),
                     ("clip_distortion", {"clip_percentile": 0.5})]:
        x = base.clone().requires_grad_()
        with pytest.raises(NotImplementedError):
            getattr(AudioSignal(x, sr).clone(), name)(**kw)
