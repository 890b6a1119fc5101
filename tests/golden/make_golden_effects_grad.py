"""Golden gradients of the REAL reference's time-domain effects (its AudioSignal differentiates through torch and the
julius restatements installed as shims), produced like ``make_golden_grad.py`` (run here only):
``python tests/golden/make_golden_effects_grad.py`` -> ``reference_golden_effects_grad.npz``
(ref:audiotools/core/audio_signal.py:716-736 resample; ref:audiotools/core/effects.py:27-64 mix, :66-123 convolve,
:125-179 apply_ir, :181-198 ensure_max_of_audio, :405-433 equalizer, :463-523 quantization / mulaw_quantization).

``run_case`` is shared with the tests: it takes the AudioSignal class to run (the reference's here, this package's in
the tests), so both sides execute the same calls on the same seeded inputs, IRs, curves and cotangents.  An input
gradient keeps its first and last EDGE samples in full (the replicate folds of the resampler and the equaliser's
641-tap filter live there) and every SAMPLE_STRIDE-th sample in between (``keep_index``); both items and both
channels are kept."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)

SR = 44100
T = 6000
EDGE = 700  # >= every case's width + old (44.1k -> 16k: 511) and the equaliser's 641 taps
SAMPLE_STRIDE = 7

# key -> (method, input sample rate, arguments); the arguments' tensors come from `params`
CASES = {
    "resample_44k1_16k": ("resample", 44100, {"sample_rate": 16000}),
    "resample_44k1_22k05": ("resample", 44100, {"sample_rate": 22050}),  # reduced new rate 1: the decimating route
    "resample_48k_16k": ("resample", 48000, {"sample_rate": 16000}),
    "resample_16k_44k1": ("resample", 16000, {"sample_rate": 44100}),
    "equalizer_shared": ("equalizer", SR, {"db": "db_shared"}),
    "equalizer_per_item": ("equalizer", SR, {"db": "db_items"}),
    "convolve_short_ir": ("convolve", SR, {"other": "ir_short"}),
    "convolve_long_ir": ("convolve", SR, {"other": "ir_long"}),
    "convolve_batch1_ir": ("convolve", SR, {"other": "ir_batch1"}),
    "convolve_no_roll": ("convolve", SR, {"other": "ir_short", "start_at_max": False}),
    "apply_ir_drr_eq": ("apply_ir", SR, {"ir": "ir_short", "drr": "drr", "ir_eq": "db_items"}),
    "apply_ir_original_phase": ("apply_ir", SR, {"ir": "ir_short", "use_original_phase": True}),
    "ensure_max_of_audio": ("ensure_max_of_audio", SR, {"max": 1.0}),
    "mix_other_eq": ("mix", SR, {"other": "noise", "snr": "snr", "other_eq": "db_shared"}),
    "quantization": ("quantization", SR, {"quantization_channels": 16}),
    "mulaw_quantization": ("mulaw_quantization", SR, {"quantization_channels": 16}),
}


def make_input(seed=0) -> torch.Tensor:
    """[2, 2, T] float32: a chirp plus seeded noise.  Item 0 peaks above 1 (ensure_max_of_audio scales it), item 1
    stays below (identity)."""
    g = torch.Generator().manual_seed(5500 + seed)
    t = torch.arange(T, dtype=torch.float64) / SR
    chirp = 0.3 * torch.sin(2 * np.pi * (100.0 * t + 0.5 * 20000.0 * t * t))
    x = chirp + 0.1 * torch.randn(2, 2, T, generator=g, dtype=torch.float64)
    return (x * torch.tensor([3.0, 0.5], dtype=torch.float64)[:, None, None]).float()


def synthetic_ir(B, L, seed) -> torch.Tensor:
    """[B, 1, L]: a direct peak (at a seeded delay) plus exponentially decaying seeded noise."""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(L, dtype=torch.float32)
    ir = 0.3 * torch.randn(B, 1, L, generator=g) * torch.exp(-t / 800.0)
    for b in range(B):
        ir[b, 0, int(torch.randint(5, 60, (1,), generator=g))] += 1.0
    return ir


def params() -> dict:
    g = torch.Generator().manual_seed(77)
    return {
        "db_shared": 6.0 * (torch.rand(1, 6, generator=g) - 0.5),
        "db_items": 6.0 * (torch.rand(2, 6, generator=g) - 0.5),
        "ir_short": synthetic_ir(2, 1500, 1),
        "ir_long": synthetic_ir(2, T + 2000, 2),  # longer than the signal: truncated
        "ir_batch1": synthetic_ir(1, 1500, 3),
        "drr": torch.tensor([5.0, 15.0]),
        "snr": torch.tensor([10.0, 3.0]),
        "noise": make_input(1) * 0.2,
    }


def cotangent(shape, seed) -> torch.Tensor:
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def keep_index(length: int, edge: int = EDGE) -> np.ndarray:
    """The samples an input gradient keeps: [0, edge), [length - edge, length) and a stride in between."""
    edge = min(edge, length)
    mid = np.arange(edge, max(edge, length - edge), SAMPLE_STRIDE)
    return np.unique(np.concatenate([np.arange(edge), mid, np.arange(length - edge, length)]))


def run_case(AudioSignal, key, device="cpu"):
    """(output, {input name: dL/dinput}) of L = <output, cotangent> for one case, with ``AudioSignal`` the class to
    run.  Gradients are taken with respect to the waveform (and, for mix, to the other signal's waveform)."""
    method, sr, args = CASES[key]
    p = params()
    x = make_input().to(device).requires_grad_()
    leaves = {"x": x}
    kw = {}
    for name, v in args.items():
        if isinstance(v, str):
            v = p[v].to(device)
            if name in ("other", "ir"):
                if v.shape[-1] == T and v.shape[0] == 2 and v.shape[1] == 2:  # a second signal: differentiate it too
                    v = v.clone().requires_grad_()
                    leaves["other"] = v
                v = AudioSignal(v, sr)
        kw[name] = v
    out = getattr(AudioSignal(x * 1.0, sr), method)(**kw).audio_data
    ct = cotangent(out.shape, 9000 + sorted(CASES).index(key)).to(device)
    names = sorted(leaves)
    grads = torch.autograd.grad((out * ct).sum(), [leaves[n] for n in names])
    return out.detach(), dict(zip(names, grads))


def main():
    from tests.golden.make_golden import import_reference

    at = import_reference()
    x = make_input()
    out = {"input_sum_abs": np.float64(x.double().abs().sum()),
           "params_sum_abs": np.float64(sum(v.double().abs().sum() for v in params().values()))}
    for key in CASES:
        y, grads = run_case(at.AudioSignal, key)
        out[key + "_out_len"] = np.int64(y.shape[-1])
        for name, gx in grads.items():
            out[f"{key}_grad_{name}"] = gx.numpy()[..., keep_index(gx.shape[-1])]
    path = os.path.join(HERE, "reference_golden_effects_grad.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
