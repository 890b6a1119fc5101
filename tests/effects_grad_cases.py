"""Shared cases of the time-domain effects' gradients (resample, equalizer, convolve, apply_ir, ensure_max_of_audio,
mix, quantization): the reference's arithmetic restated in float64 torch (oracle/ restatements of julius and of
ref:audiotools/core/effects.py), differentiated by torch.autograd, and the same computation through this package's
AudioSignal.  Used by the simulator and the GPU tests."""
import torch

from audiotools_b200 import AudioSignal
from oracle import signal_path as sp

RESAMPLE_RATES = [(44100, 16000), (44100, 22050), (48000, 16000), (16000, 44100)]
# T < width (44.1k -> 16k: width 70; 16k -> 44.1k: 26), T < K, and a few thousand samples
RESAMPLE_LENGTHS = [5, 60, 300, 3001]
EQ_LENGTHS = [200, 4000]  # 6 bands at 44.1 kHz: 641 taps (T < K and T > K)


def x_of(shape, seed, scale=0.5):
    return scale * torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def synthetic_ir(B, L, seed, C=1):
    """A direct peak plus exponentially decaying noise, [B, C, L]."""
    gen = torch.Generator().manual_seed(seed)
    t = torch.arange(L, dtype=torch.float32)
    ir = 0.3 * torch.randn(B, C, L, generator=gen) * torch.exp(-t / (0.2 * L))
    peak = torch.randint(0, max(1, L // 8), (B,), generator=gen)
    for b in range(B):
        ir[b, :, peak[b]] += 1.0
    return ir


def db_curve(B, n_bands, seed):
    return 6.0 * (torch.rand(B, n_bands, generator=torch.Generator().manual_seed(seed)) - 0.5)


def vjp(fn, x, g):
    """dL/dx of L = <fn(x), g> through torch.autograd, x float32 or float64."""
    xg = x.clone().requires_grad_()
    (gx,) = torch.autograd.grad((fn(xg) * g.to(xg.dtype)).sum(), xg)
    return gx


# ---- the product, as a function of the waveform ------------------------------------------------------------------
def ours(method, sr=44100, **kw):
    def run(x):
        s = AudioSignal(x, sr)
        if method == "resample":
            return s.resample(kw["new_sr"]).audio_data
        if method == "equalizer":
            return s.equalizer(kw["db"], _bypass=kw.get("bypass")).audio_data
        if method == "convolve":
            return s.convolve(AudioSignal(kw["ir"], sr), start_at_max=kw.get("start_at_max", True),
                              _bypass=kw.get("bypass")).audio_data
        if method == "apply_ir":
            return s.apply_ir(AudioSignal(kw["ir"], sr), _bypass=kw.get("bypass")).audio_data
        if method == "ensure_max_of_audio":
            return s.ensure_max_of_audio(kw.get("max", 1.0)).audio_data
        raise ValueError(method)

    return run


# ---- the reference's arithmetic in float64 -----------------------------------------------------------------------
def ref(method, sr=44100, **kw):
    def run(x):
        if method == "resample":
            return sp.resample(x, sr, kw["new_sr"])
        if method == "equalizer":
            return sp.equalizer(x, sr, kw["db"].to(x.device).double())
        if method == "convolve":
            return sp.convolve(x, kw["ir"].to(x), start_at_max=kw.get("start_at_max", True))
        if method == "apply_ir":
            return apply_ir64(x, kw["ir"].to(x))
        if method == "ensure_max_of_audio":
            return sp.ensure_max_of_audio(x, kw.get("max", 1.0))
        raise ValueError(method)

    return run


def apply_ir64(x, ir):
    """ref:audiotools/core/effects.py:125-179 without drr / ir_eq (those change the IR, a constant here)."""
    max_spk = x.abs().max(dim=-1, keepdim=True).values
    y = sp.convolve(x, ir)
    max_t = y.abs().max(dim=-1, keepdim=True).values
    return y * (max_spk.clamp(1e-8) / max_t.clamp(1e-8))


def bypassed(fn, x, bypass):
    """fn on the items bypass does not select, x on the others."""
    y = fn(x)
    keep = torch.as_tensor(bypass).bool().reshape(-1, 1, 1)
    return torch.where(keep, x, y)


def golden_errors(golden, device):
    """key -> (rel_err, elementwise_ok) of this package's gradient against the real reference's for every case of
    tests/golden/make_golden_effects_grad.py (same calls, inputs, parameters and cotangents)."""
    import numpy as np

    from tests.conftest import elementwise_ok, rel_err
    from tests.golden import make_golden_effects_grad as mg

    assert abs(float(golden["input_sum_abs"]) - mg.make_input().double().abs().sum().item()) < 1e-9 * float(
        golden["input_sum_abs"])
    errs = {}
    for key in mg.CASES:
        y, grads = mg.run_case(AudioSignal, key, device)
        assert y.shape[-1] == int(golden[key + "_out_len"]), key
        for name, gx in grads.items():
            got = gx.cpu()[..., mg.keep_index(gx.shape[-1])]
            want = torch.from_numpy(np.asarray(golden[f"{key}_grad_{name}"]))
            errs[f"{key}_grad_{name}"] = (rel_err(got, want), elementwise_ok(got, want, frame_dim=-1))
    return errs


# apply_ir with use_original_phase runs through angle(X), whose derivative is 1/|X|: FP32 spectra are ill-conditioned
# there.  Against float64 on the golden's input the reference's own FP32 gradient is 2.2e-4 away, this package's 7.8e-4.
GOLDEN_TOL = {"apply_ir_original_phase_grad_x": 2e-3}


def load_golden():
    import os

    import numpy as np

    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                                "reference_golden_effects_grad.npz"))


def check_golden(golden, device, tol=1e-4):
    """Every golden case within ``tol`` globally and per cell.  On a GPU the resample cases are held to the global
    tolerance only: the engine designs the resample taps with torch on the device, up to 5.2e-6 from the CPU design the
    reference uses, and the forward runs on those same taps (the per-cell check of the backward kernel on the GPU runs
    against float64 with the device's taps, tests/test_gpu_effects_grad.py)."""
    errs = golden_errors(golden, device)
    on_gpu = str(device).startswith("cuda")
    bad = {k: v for k, v in errs.items()
           if not (v[0] < GOLDEN_TOL.get(k, tol)
                   and (v[1] or k in GOLDEN_TOL or (on_gpu and k.startswith("resample_"))))}
    assert not bad, bad
    return errs
