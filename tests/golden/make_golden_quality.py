"""Golden STOI / extended STOI values of the REAL reference's ``metrics.quality.stoi`` (ref:audiotools/metrics/
quality.py:11-57), run over ``tests/stoi_oracle.py`` (the float64 restatement of pystoi) in place of the pystoi package:
``python tests/golden/make_golden_quality.py`` -> ``reference_golden_quality.npz`` (run here only).

Each case is a batch built by ``case_signals(key)`` from seeds (synthetic speech-like signals: a gliding harmonic
source under a syllable-rate envelope, with a broadband floor), so the tests rebuild the same inputs.  Stored per case
and mode: the scores (``<key>_std`` / ``<key>_ext``), the kept-frame counts and STFT frame counts of the silence removal
(``<key>_kept`` / ``<key>_M``) and the inputs' sums of |x| (``<key>_sum``: a check that the rebuilt inputs are the
ones the golden saw).  The generator refuses a case where a frame energy lies within 1e-3 dB of the 40 dB threshold,
so float32 arithmetic cannot flip a keep decision."""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)

from tests import stoi_oracle as so  # noqa: E402


def speech(sr, T, seed, gaps=()):
    """[T] float32 speech-like signal: harmonics of a gliding 100-160 Hz source under a syllable-rate envelope, a
    -50 dB broadband floor; digital silence over the (start, end) second ranges in ``gaps``."""
    r = np.random.default_rng(seed)
    t = np.arange(T) / sr
    f0 = r.uniform(100, 160) + 25 * np.sin(2 * np.pi * r.uniform(0.5, 1.0) * t)
    ph = 2 * np.pi * np.cumsum(f0) / sr
    env = 0.2 + np.clip(np.sin(2 * np.pi * r.uniform(2.5, 4.0) * t + r.uniform(0, 6)), 0, None)
    nyq = min(sr / 2, 5000.0)
    x = sum(np.sin(h * ph + r.uniform(0, 6)) / h for h in range(1, int(nyq / 170)))
    x = 0.1 * x * env + 3e-4 * r.standard_normal(T)
    for a, b in gaps:
        x[int(a * sr):int(b * sr)] = 0.0
    return x.astype(np.float32)


def noise(shape, seed):
    return np.random.default_rng(seed).standard_normal(shape).astype(np.float32)


def with_snr(x, snr_db, seed):
    n = noise(x.shape, seed)
    g = np.sqrt((x.astype(np.float64) ** 2).sum() / (n.astype(np.float64) ** 2).sum() / 10 ** (snr_db / 10))
    return (x + g * n).astype(np.float32)


# key -> sample rate, seconds, channels, items; item = (estimate kind, argument, gaps of the clean signal)
CASES = {
    "sr10000": (10000, 1.6, 1, [("snr", 5.0, ()), ("scale", 0.5, ())]),
    "sr16000": (16000, 1.6, 1, [("snr", 10.0, ()), ("scale", 3.0, ())]),
    "sr22050": (22050, 1.6, 1, [("snr", 0.0, ()), ("identity", None, ())]),
    "sr44100": (44100, 1.6, 1, [("snr", 5.0, ()), ("scale", 0.25, ())]),
    "sr48000": (48000, 1.6, 1, [("snr", -5.0, ()), ("identity", None, ())]),
    "stereo44100": (44100, 1.6, 2, [("snr", 3.0, ()), ("snr", 15.0, ())]),
    "snr16000": (16000, 1.6, 1, [("snr", 30.0, ()), ("snr", 10.0, ()), ("snr", 0.0, ()), ("snr", -10.0, ())]),
    "gaps16000": (16000, 2.4, 1, [("snr", 5.0, ((0.3, 0.7), (1.2, 1.5))), ("identity", None, ((0.0, 0.5),))]),
    "short16000": (16000, 1.6, 1, [("snr", 5.0, ((0.0, 1.25),)), ("snr", 5.0, ())]),
}


def case_signals(key):
    """(estimates, references) [B, C, T] float32 and the sample rate of a case."""
    sr, sec, C, items = CASES[key]
    T = int(sr * sec)
    seed = sum(ord(c) for c in key) * 1000
    refs, ests = [], []
    for i, (kind, arg, gaps) in enumerate(items):
        ref = np.stack([speech(sr, T, seed + 10 * i + c, gaps) for c in range(C)])
        if kind == "snr":
            est = with_snr(ref, arg, seed + 10 * i + 7)
        elif kind == "scale":
            est = (ref * np.float32(arg)).astype(np.float32)
        else:
            est = ref.copy()
        refs.append(ref)
        ests.append(est)
    return np.stack(ests), np.stack(refs), sr


def check_margins(est, ref, sr):
    """Every frame energy of the clean signal at least 1e-3 dB away from the 40 dB keep threshold."""
    x = ref.mean(axis=1, dtype=np.float32)
    up, down = so.FS // np.gcd(so.FS, sr), sr // np.gcd(so.FS, sr)
    for i in range(x.shape[0]):
        xi = so.resample_oct(x[i], so.FS, sr) if sr != so.FS else x[i]
        _, _, _, e = so.remove_silent_frames(xi, xi)
        margin = np.abs(e.max() - so.DYN_RANGE - e).min()
        assert margin > 1e-3, (sr, up, down, i, margin)


def main():
    from tests.golden.make_golden import import_reference

    import_reference()
    sys.modules["pystoi"] = types.ModuleType("pystoi")
    sys.modules["pystoi"].stoi = so.stoi
    import torch
    from audiotools import AudioSignal
    from audiotools.metrics import quality

    out = {}
    for key in CASES:
        est, ref, sr = case_signals(key)
        check_margins(est, ref, sr)
        out[key + "_sum"] = np.array([np.abs(est).astype(np.float64).sum(), np.abs(ref).astype(np.float64).sum()])
        for mode, ext in (("std", False), ("ext", True)):
            v = quality.stoi(AudioSignal(torch.from_numpy(est), sr), AudioSignal(torch.from_numpy(ref), sr), ext)
            assert v.dtype == torch.float64 and v.shape == (est.shape[0],)
            out[f"{key}_{mode}"] = v.numpy()
        _, kept, M = so.batch_stoi(est, ref, sr)
        out[key + "_kept"], out[key + "_M"] = kept, M
        print(key, out[key + "_std"], out[key + "_ext"], kept, M)
    path = os.path.join(HERE, "reference_golden_quality.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
