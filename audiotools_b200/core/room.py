"""Shoebox-room impulse responses by the image-source method (Allen & Berkley 1979) for a whole batch on the GPU
(csrc/rir.cu, DESIGN.md K20).

``image_source_ir(room, source, mics, sample_rate, length, beta=... | rt60=...)`` returns an ``AudioSignal``
[B, C, length]: channel c of item b is the response from item b's source to its microphone c, ready for
``AudioSignal.apply_ir``.  Lengths are in metres, the sound speed in m/s.  Each image of the source adds a
Hann-windowed fractional delay of 2 floor(0.004 sample_rate + 1/2) samples, centred on its distance, scaled by the
product of the wall reflection coefficients it meets over 4 pi times its distance in metres; ``high_pass`` then
applies Allen & Berkley's 100 Hz high-pass as one second-order section.  ``rt60`` in place of ``beta`` gives all six
walls the reflection coefficient of Sabine's formula (``sabine_beta``).

``diffuse_after`` (seconds, scalar or [B]) with ``seed`` (int or [B] ints) makes a hybrid response: the images
arriving before sample n_d = ceil(diffuse_after sample_rate) only, and from n_d - Tw/2 on a diffuse tail, Gaussian
noise under the energy envelope the same room's images have on average (a raised-cosine crossfade over the Tw samples
centred on n_d).  The image count up to a time t grows with t^3, so a short ``diffuse_after`` makes long responses
cheap.  The tail is frequency-flat like the walls, and the tails of different microphones are independent; it depends
only on the item's geometry, its seed and the microphone, so a batch equals its items one at a time.

``bands=K`` gives every wall, and with ``air_absorption`` the air, its own value in each of K octave bands centred on
f_k = 125 2^k Hz: r_k is the response (images, and the tail with ``diffuse_after``) with band k's reflection
coefficients, every image also scaled by 10^(-a_k d / 20) (d in metres, a_k in dB/m) and the tail's envelope by
10^(-a_k (c n / fs) / 10); the tails of all bands share one noise.  The bands are joined by zero-phase windowed-sinc
low-passes LP_k at the crossovers e_k = 125 2^(k + 1/2) Hz, y = r_{K'-1} + sum_{k < K'-1} LP_k * (r_k - r_{k+1}),
where K' counts the bands whose lower crossover is below sample_rate / 2.  The crossovers are 2 half_0 + 1 taps long,
half_0 = int(8 fs / e_0 / 2), and zero-phase, so a response can start up to half_0 samples before its first arrival
(the window's Tw / 2 comes on top).  Equal bands without air give the ``bands=None`` response bit for bit.

``mic_pattern`` / ``source_pattern`` with ``mic_orientation`` / ``source_orientation`` make the microphones and the
sources directional (DESIGN.md K20 "Directivity"): a first-order pattern p in [0, 1] (a name of ``PATTERNS`` or a
value) with an orientation v has the amplitude gain D(u) = p + (1 - p) u.v for a unit direction u, negative in a rear
lobe and the same at every frequency.  Every image is scaled by the microphone's gain at the direction its sound
arrives from and by the source's gain at the direction the source emitted it in (each wall reflection mirrors one
axis), so swapping a source and a microphone together with their patterns gives the same response.  The diffuse tail
follows the expected energy of those scaled arrivals.  An end whose p is 1 everywhere is omnidirectional whatever its
orientation, and its response is the omnidirectional one bit for bit.

The geometry is checked on host values (``util.host_view`` reads a table's host mirror, so no device sync is needed)
and is a constant: a geometry tensor that requires a gradient raises ``NotImplementedError``.
"""
import math

import numpy as np
import torch

from . import grad as _grad
from . import util

MIN_SAMPLE_RATE = 125.0     # below it the window 2 floor(0.004 fs + 1/2) is empty
MAX_SAMPLE_RATE = 384000.0  # csrc/rir.cu's largest window table
MIN_DISTANCE = 1e-3         # metres between the source and a microphone
MAX_BANDS = 8               # octave bands centred on 125 2^k Hz, k < 8 (up to 16 kHz)
MAX_ROWS = 65535            # items x microphones x bands of one call (csrc/rir.cu's grid)
# first-order patterns D(u) = p + (1 - p) u.v by name: p = 1 / (1 + sqrt 3) = (sqrt 3 - 1) / 2 is the supercardioid
# (the largest front-to-back energy ratio), 1/4 the hypercardioid (the largest directivity factor)
PATTERNS = {"omni": 1.0, "subcardioid": 0.75, "cardioid": 0.5, "supercardioid": (math.sqrt(3.0) - 1.0) / 2.0,
            "hypercardioid": 0.25, "figure8": 0.0}


def _host(name: str, v) -> np.ndarray:
    _grad.refuse_param_grad("image_source_ir", name, v)
    if torch.is_tensor(v):
        v = util.host_view(v).detach().cpu().numpy()  # the host mirror belongs to v itself, not to a detached view
    return np.asarray(v, dtype=np.float64)


def _room_sizes(room: np.ndarray):
    """Volume and surface of rooms [..., 3]."""
    lx, ly, lz = room[..., 0], room[..., 1], room[..., 2]
    return lx * ly * lz, 2.0 * (lx * ly + lx * lz + ly * lz)


def min_rt60(room, sound_speed: float = 343.0) -> np.ndarray:
    """The smallest RT60 Sabine's formula gives a room [..., 3]: every wall fully absorbing (alpha = 1)."""
    vol, surf = _room_sizes(np.asarray(room, dtype=np.float64))
    return 24.0 * math.log(10.0) * vol / (sound_speed * surf)


def sabine_beta(room, rt60, sound_speed: float = 343.0) -> np.ndarray:
    """Wall reflection coefficients [..., 6] for rooms [..., 3] and reverberation times ``rt60`` (seconds, scalar or
    [...]) by Sabine: alpha = 24 ln 10 V / (c S rt60), beta = sqrt(1 - alpha), the same for all six walls; rt60 = 0
    gives beta = 0.  A time below the room's smallest feasible RT60 (alpha > 1) raises ``ValueError``."""
    room = np.asarray(room, dtype=np.float64)
    rt60 = np.asarray(rt60, dtype=np.float64)
    if not (np.all(np.isfinite(rt60)) and np.all(rt60 >= 0)):
        raise ValueError(f"rt60 must be finite and >= 0, got {rt60}")
    vol, surf = _room_sizes(room)
    pos = rt60 > 0
    alpha = np.where(pos, 24.0 * math.log(10.0) * vol / (sound_speed * surf * np.where(pos, rt60, 1.0)), 1.0)
    bad = alpha > 1.0
    if np.any(bad):
        lo = np.broadcast_to(min_rt60(room, sound_speed), alpha.shape)[bad].flat[0]
        t = np.broadcast_to(rt60, alpha.shape)[bad].flat[0]
        raise ValueError(f"rt60 = {t:.6g} s is below the room's smallest feasible RT60, {lo:.6g} s (Sabine, every "
                         "wall fully absorbing)")
    return np.repeat(np.sqrt(1.0 - alpha)[..., None], 6, axis=-1)


def _directivity(end: str, pattern, orientation):
    """(p, unit orientations) on the host for one end (``"mic"`` or ``"source"``); (None, None) when it is
    omnidirectional: no pattern, or p = 1 everywhere without an orientation."""
    if pattern is None:
        if orientation is not None:
            raise ValueError(f"image_source_ir: {end}_orientation without a {end}_pattern")
        return None, None
    if isinstance(pattern, str):
        if pattern not in PATTERNS:
            raise ValueError(f"image_source_ir: {end}_pattern = {pattern!r}; one of {', '.join(PATTERNS)} or a "
                             "value in [0, 1]")
        p = np.float64(PATTERNS[pattern])
    else:
        p = _host(f"{end}_pattern", pattern)
        if not (p.size and np.all(np.isfinite(p)) and np.all(p >= 0) and np.all(p <= 1)):
            raise ValueError(f"image_source_ir: {end}_pattern = {p}; p must be in [0, 1] (1: omni, 0: figure8)")
    if orientation is None:
        if np.any(p != 1):
            raise ValueError(f"image_source_ir: a directional {end}_pattern needs a {end}_orientation")
        return p, None
    v = _host(f"{end}_orientation", orientation)
    if v.ndim == 0 or v.shape[-1] != 3:
        raise ValueError(f"image_source_ir: {end}_orientation has 3 coordinates, got shape {v.shape}")
    big = np.abs(v).max(axis=-1, keepdims=True)
    if not (np.all(np.isfinite(v)) and np.all(big > 0)):
        raise ValueError(f"image_source_ir: every {end}_orientation must be finite and non-zero")
    v = v / big  # scaled first, so that the norm neither overflows nor underflows
    return p, v / np.sqrt((v * v).sum(axis=-1, keepdims=True))


def _dir_table(p: np.ndarray, v, shape: tuple):
    """[*shape, 4] (p, v) of one end, or None when p = 1 everywhere (omnidirectional: no table is passed)."""
    if p is None or np.all(p == 1):
        return None
    v = np.zeros(shape + (3,)) if v is None else v
    return np.concatenate([np.broadcast_to(p, shape)[..., None], np.broadcast_to(v, shape + (3,))], axis=-1)


def _batch(name: str, v: np.ndarray, item_ndim: int, B: int) -> np.ndarray:
    if v.ndim == item_ndim:
        return np.broadcast_to(v, (B,) + v.shape)
    if v.ndim == item_ndim + 1 and v.shape[0] in (1, B):
        return np.broadcast_to(v, (B,) + v.shape[1:])
    raise ValueError(f"image_source_ir: {name} of shape {v.shape} does not fit a batch of {B}")


def image_source_ir(room, source, mics, sample_rate: float, length: int, *, beta=None, rt60=None,
                    max_order: int = -1, sound_speed: float = 343.0, high_pass: bool = True, diffuse_after=None,
                    seed=None, bands=None, air_absorption=None, mic_pattern=None, mic_orientation=None,
                    source_pattern=None, source_orientation=None, device="cuda"):
    """Impulse responses [B, C, length] of shoebox rooms by the image-source method, as an ``AudioSignal`` at
    ``sample_rate``.

    ``room`` [3] or [B, 3] (Lx, Ly, Lz), ``source`` [3] or [B, 3], ``mics`` [C, 3] or [B, C, 3]; exactly one of
    ``beta`` ([6] or [B, 6]: the walls x = 0, x = Lx, y = 0, y = Ly, z = 0, z = Lz, each in [0, 1]) and ``rt60``
    (seconds, scalar or [B]; ``sabine_beta``).  ``max_order`` >= 0 keeps the images of at most that order (the number
    of wall reflections); -1 keeps every image that arrives within ``length`` samples.  One kernel launch, three more
    with ``high_pass``; no host sync.

    ``diffuse_after`` (seconds > 0, scalar or [B]) and ``seed`` (an int or [B] ints in [0, 2^63)) add the diffuse tail
    (module docstring; DESIGN.md K20 "Hybrid"): two kernel launches before the high-pass.  It needs ``max_order =
    -1`` (the tail stands for images of every order).

    ``bands=K`` (1 .. 8) makes the walls, and with ``air_absorption`` the air, frequency-dependent over K octave bands
    centred on 125 2^k Hz (module docstring; DESIGN.md K20 "Bands"): ``beta`` is then [6, K] or [B, 6, K], ``rt60``
    [K] or [B, K] (``sabine_beta`` per band) and ``air_absorption`` (dB/m, finite, >= 0) [K] or [B, K].  Bands whose
    lower crossover is at or above sample_rate / 2 are checked but not computed.  One launch (two with the tail), the
    crossovers' ``fftconv`` and one launch for their sum when more than one band is computed, then the high-pass.
    ``bands=None`` is the frequency-flat room, computed as one band.

    ``mic_pattern`` (a name of ``PATTERNS`` or p in [0, 1]: scalar, [C] or [B, C]) with ``mic_orientation`` ([3],
    [C, 3] or [B, C, 3], normalised here) makes the microphones directional, and ``source_pattern`` (a name or p:
    scalar or [B]) with ``source_orientation`` ([3] or [B, 3]) the sources (module docstring; DESIGN.md K20
    "Directivity").  A pattern other than omni needs its orientation, and an orientation its pattern.  It works with
    every option above and adds no launch."""
    from ..engine import get_engine
    from .audio_signal import AudioSignal

    if (beta is None) == (rt60 is None):
        raise ValueError("image_source_ir: give exactly one of beta and rt60")
    room_h, src_h, mics_h = _host("room", room), _host("source", source), _host("mics", mics)
    wall_h = _host("beta" if rt60 is None else "rt60", beta if rt60 is None else rt60)
    sample_rate, length, max_order, sound_speed = float(sample_rate), int(length), int(max_order), float(sound_speed)
    if not MIN_SAMPLE_RATE <= sample_rate <= MAX_SAMPLE_RATE:
        raise ValueError(f"image_source_ir: sample_rate = {sample_rate:g}; {MIN_SAMPLE_RATE:g} .. "
                         f"{MAX_SAMPLE_RATE:g} Hz are supported (below 125 Hz the window 2 round(0.004 fs) is empty)")
    if length < 1:
        raise ValueError(f"image_source_ir: length = {length} must be >= 1")
    if max_order < -1:
        raise ValueError(f"image_source_ir: max_order = {max_order} must be >= -1 (-1: every image)")
    if not (math.isfinite(sound_speed) and sound_speed > 0):
        raise ValueError(f"image_source_ir: sound_speed = {sound_speed} must be positive")
    n_tail = 1
    if bands is None and air_absorption is not None:
        raise ValueError("image_source_ir: air_absorption is per octave band; give bands too")
    if bands is not None:
        if isinstance(bands, bool) or not isinstance(bands, (int, np.integer)) or not 1 <= bands <= MAX_BANDS:
            raise ValueError(f"image_source_ir: bands = {bands!r}; an int in 1 .. {MAX_BANDS} (octaves from 125 Hz)")
        bands = int(bands)
    air_h = None if air_absorption is None else _host("air_absorption", air_absorption)
    if diffuse_after is None and seed is not None:
        raise ValueError("image_source_ir: seed is for the diffuse tail; give diffuse_after too")
    if diffuse_after is not None:
        td_h = _host("diffuse_after", diffuse_after).reshape(-1)
        if not (td_h.size and np.all(np.isfinite(td_h)) and np.all(td_h > 0)):
            raise ValueError(f"image_source_ir: diffuse_after = {td_h} must be finite and > 0 seconds")
        if max_order != -1:
            raise ValueError(f"image_source_ir: max_order = {max_order} with diffuse_after; the diffuse tail stands "
                             "for images of every order, so it needs max_order = -1")
        if seed is None:
            raise ValueError("image_source_ir: diffuse_after needs a seed (an int or one per item)")
        sd = np.asarray(util.host_view(seed).detach().cpu().numpy() if torch.is_tensor(seed) else seed).reshape(-1)
        if sd.dtype.kind not in "iu" or not (sd.size and np.all(sd >= 0) and np.all(sd < 2 ** 63)):
            raise ValueError(f"image_source_ir: seed = {sd} must be integers in [0, 2^63)")
        sd = sd.astype(np.int64)
        n_tail = max(td_h.size, sd.size)
    if bands is None:
        n_wall = (wall_h.shape[0] if wall_h.ndim == 2 else 1) if rt60 is None else (wall_h.size if wall_h.ndim else 1)
    else:  # the item axis leads a [B, 6, K] beta, a [B, K] rt60 and a [B, K] air absorption
        n_wall = max(wall_h.shape[0] if wall_h.ndim == (3 if rt60 is None else 2) else 1,
                     air_h.shape[0] if air_h is not None and air_h.ndim == 2 else 1)
    mic_p, mic_v = _directivity("mic", mic_pattern, mic_orientation)
    src_p, src_v = _directivity("source", source_pattern, source_orientation)
    n_dir = max(mic_p.shape[0] if mic_p is not None and mic_p.ndim == 2 else 1,
                mic_v.shape[0] if mic_v is not None and mic_v.ndim == 3 else 1,
                src_p.shape[0] if src_p is not None and src_p.ndim == 1 else 1,
                src_v.shape[0] if src_v is not None and src_v.ndim == 2 else 1)
    B = max(room_h.shape[0] if room_h.ndim == 2 else 1, src_h.shape[0] if src_h.ndim == 2 else 1,
            mics_h.shape[0] if mics_h.ndim == 3 else 1, n_wall, n_tail, n_dir)
    room_h = _batch("room", room_h, 1, B)
    src_h = _batch("source", src_h, 1, B)
    mics_h = _batch("mics", mics_h, 2, B)
    if room_h.shape[-1] != 3 or src_h.shape[-1] != 3 or mics_h.shape[-1] != 3:
        raise ValueError("image_source_ir: room, source and microphone positions have 3 coordinates")
    if not (np.all(np.isfinite(room_h)) and np.all(room_h > 0)):
        raise ValueError(f"image_source_ir: room dimensions must be positive, got {room_h.min(axis=0)} at least")
    for name, p in (("source", src_h[:, None]), ("microphone", mics_h)):
        if not (np.all(np.isfinite(p)) and np.all(p > 0) and np.all(p < room_h[:, None])):
            raise ValueError(f"image_source_ir: every {name} must be strictly inside its room")
    gap = np.sqrt(((mics_h - src_h[:, None]) ** 2).sum(-1))
    if np.any(gap < MIN_DISTANCE):
        raise ValueError(f"image_source_ir: a microphone is {gap.min():.3g} m from the source; at least "
                         f"{MIN_DISTANCE:g} m is needed")
    if bands is not None:
        if rt60 is None:
            beta_h = _batch("beta", wall_h, 2, B)
            if beta_h.shape[1:] != (6, bands):
                raise ValueError(f"image_source_ir: beta must be [6, {bands}] or [B, 6, {bands}] with bands = "
                                 f"{bands}, got {wall_h.shape}")
        else:
            rt_h = _batch("rt60", wall_h, 1, B)
            if rt_h.shape[1:] != (bands,):
                raise ValueError(f"image_source_ir: rt60 must be [{bands}] or [B, {bands}] with bands = {bands}, "
                                 f"got {wall_h.shape}")
            beta_h = np.swapaxes(sabine_beta(room_h[:, None], rt_h, sound_speed), 1, 2)  # [B, 6, K]
        if air_h is not None:
            air_h = _batch("air_absorption", air_h, 1, B)
            if air_h.shape[1:] != (bands,):
                raise ValueError(f"image_source_ir: air_absorption must be [{bands}] or [B, {bands}] dB/m with bands "
                                 f"= {bands}, got {air_h.shape}")
            if not (np.all(np.isfinite(air_h)) and np.all(air_h >= 0)):
                raise ValueError("image_source_ir: air_absorption must be finite and >= 0 dB/m")
        if B * mics_h.shape[1] * bands > MAX_ROWS:
            raise ValueError(f"image_source_ir: {B * mics_h.shape[1] * bands} rows (items x microphones x bands); "
                             f"at most {MAX_ROWS}")
    elif rt60 is None:
        beta_h = _batch("beta", wall_h, 1, B)
        if beta_h.shape[-1] != 6:
            raise ValueError(f"image_source_ir: beta must have 6 walls, got {beta_h.shape}")
    else:
        beta_h = sabine_beta(room_h, _batch("rt60", wall_h.reshape(-1) if wall_h.ndim else wall_h, 0, B),
                             sound_speed)
    if not (np.all(beta_h >= 0) and np.all(beta_h <= 1)):
        raise ValueError("image_source_ir: every reflection coefficient beta must be in [0, 1]")
    if bands is None:
        beta_h = beta_h[..., None]  # a frequency-flat room is one band: [B, 6, 1]
    C = mics_h.shape[1]
    mic_dir = src_dir = None
    if mic_p is not None:
        mp = _batch("mic_pattern", np.broadcast_to(mic_p, (C,)) if mic_p.ndim == 0 else mic_p, 1, B)
        mv = None if mic_v is None else _batch("mic_orientation", np.broadcast_to(mic_v, (C, 3)) if mic_v.ndim == 1
                                               else mic_v, 2, B)
        if mp.shape != (B, C) or (mv is not None and mv.shape != (B, C, 3)):
            raise ValueError(f"image_source_ir: mic_pattern / mic_orientation must fit {C} microphones: scalar, [C] or "
                             f"[B, C] / [3], [C, 3] or [B, C, 3], got {mic_p.shape} / "
                             f"{None if mic_v is None else mic_v.shape}")
        mic_dir = _dir_table(mp, mv, (B, C))
    if src_p is not None:
        sp = _batch("source_pattern", src_p, 0, B)
        sv = None if src_v is None else _batch("source_orientation", src_v, 1, B)
        src_dir = _dir_table(sp, sv, (B,))
    dev = torch.device(device)

    def upload(a, dtype=np.float64):
        return None if a is None else torch.from_numpy(np.array(a, dtype=dtype)).to(dev, non_blocking=True)

    tab = [upload(a) for a in (room_h, src_h, mics_h, beta_h)]
    tail = {}
    if diffuse_after is not None:
        tail = dict(diffuse_after=upload(_batch("diffuse_after", td_h, 0, B)),
                    seed=upload(_batch("seed", sd, 0, B), np.int64))
    ir = get_engine().image_source_ir(*tab, length, sample_rate, sound_speed, max_order, high_pass,
                                      air=upload(air_h), mic_dir=upload(mic_dir), src_dir=upload(src_dir), **tail)
    return AudioSignal(ir, sample_rate)
