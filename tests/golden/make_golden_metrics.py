"""Golden values and input gradients of the REAL reference's metrics (ref:audiotools/metrics/spectral.py and
distance.py), produced like ``make_golden_grad.py`` (same inputs, same shims; run here only):
``python tests/golden/make_golden_metrics.py`` -> ``reference_golden_metrics.npz``.
Each case stores the loss value (``<key>``) and dL/dx of the estimate (``<key>_grad``, rows ``ROWS`` and samples
``keep_index(T, 2048)`` of make_golden_grad).  The signals of a case are built by ``signals(AudioSignal, key)`` so that
the tests rebuild them through this package's AudioSignal the same way."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)

from tests.golden.make_golden_grad import ROWS, SR, T, keep_index, make_input  # noqa: E402

# key -> (module name, constructor kwargs, stft_params of both signals as a dict or None)
CASES = {
    "mel_log_only": ("MelSpectrogramLoss", dict(n_mels=[64, 32], window_lengths=[1024, 256], mag_weight=0.0, pow=1.0,
                                                clamp_eps=1e-4, mel_fmin=[50.0, 100.0], mel_fmax=[16000.0, 8000.0]),
                     None),
    "stft_3scale_sqrt": ("MultiScaleSTFTLoss", dict(window_lengths=[1024, 256, 64], log_weight=0.5,
                                                    window_type="sqrt_hann"), None),
    "mel_ms_replicate": ("MelSpectrogramLoss", dict(), dict(window_length=2048, hop_length=512, window_type="hann",
                                                            match_stride=True, padding_type="replicate")),
    "stft_ms_constant": ("MultiScaleSTFTLoss", dict(window_lengths=[512, 128]),
                         dict(window_length=512, hop_length=128, window_type="hann", match_stride=True,
                              padding_type="constant")),
    "phase": ("PhaseLoss", dict(), None),
    "l1": ("L1Loss", dict(), None),
    "sisdr": ("SISDRLoss", dict(), None),
    "sisdr_sum_noscale": ("SISDRLoss", dict(scaling=False, reduction="sum", zero_mean=False), None),
    "sisdr_none_clip": ("SISDRLoss", dict(reduction="none", clip_min=-20.0), None),
}


def signals(AudioSignal, STFTParams, key, x, y):
    sp = CASES[key][2]
    kw = {} if sp is None else {"stft_params": STFTParams(**sp)}
    return AudioSignal(x, SR, **kw), AudioSignal(y, SR, **kw)


def module(metrics_spectral, metrics_distance, key):
    name, kwargs, _ = CASES[key]
    mod = getattr(metrics_spectral, name, None) or getattr(metrics_distance, name)
    return mod(**kwargs)


def main():
    from tests.golden.make_golden import import_reference

    at = import_reference()
    from audiotools.metrics import distance, spectral

    x = make_input()
    y = make_input(1)
    out = {"input_sum_abs": np.float64(x.double().abs().sum()), "target_sum_abs": np.float64(y.double().abs().sum())}
    for key in CASES:
        xg = x.clone().requires_grad_()
        sx, sy = signals(at.AudioSignal, at.STFTParams, key, xg, y.clone())
        loss = module(spectral, distance, key)(sx, sy)
        (gx,) = torch.autograd.grad(loss.sum(), xg)
        out[key] = loss.detach().double().numpy()
        out[key + "_grad"] = gx[ROWS].numpy()[..., keep_index(T, 2048)]
    path = os.path.join(HERE, "reference_golden_metrics.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
