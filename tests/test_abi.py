"""The C-ABI library loads and exports every symbol include/b2a.h declares (no compute calls:
this runs without a GPU); argument validation returns error codes instead of crashing."""
import ctypes
import os
import re

import numpy as np

import pytest

import __graft_entry__ as graft
from audiotools_b200 import _lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    graft.build()
    return _lib.B2ALibrary(_lib.LIB_PATH)


def declared_symbols():
    src = open(os.path.join(REPO, "include", "b2a.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b2a_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_are_exported_and_bound(lib):
    syms = declared_symbols()
    assert "b2a_spectral_f32" in syms and "b2a_lufs_f32" in syms
    assert sorted(_lib.SIGNATURES) == syms, "audiotools_b200/_lib.py must bind exactly what b2a.h declares"
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for s in syms:
        assert getattr(raw, s) is not None


def test_version_and_pure_host_queries(lib):
    assert lib.b2a_version() == 100
    # frame / block counts are integer host arithmetic (bit-exact requirement of BASELINE.json)
    assert lib.b2a_stft_num_frames(16000, 512, 128, 0, 0, 0) == 126          # cfg1
    assert lib.b2a_stft_num_frames(441000, 2048, 512, 0, 0, 0) == 862        # cfg2
    assert lib.b2a_stft_num_frames(16000, 256, 64, 96, 0, 2) == 250          # match_stride: T/hop
    assert lib.b2a_stft_num_frames(15999, 256, 64, 96, 1, 2) == 250
    assert lib.b2a_lufs_num_blocks(441000, 44100.0, 0.4) == 97               # cfg2
    assert lib.b2a_lufs_num_blocks(8000, 16000.0, 0.4) == 2
    assert lib.b2a_lufs_num_blocks(22050, 11025.0, 0.4) == 18                # K=4410, stride=1102
    assert lib.b2a_lufs_workspace_bytes(64, 2, 441000, 44100.0, 0.4) > 0


def test_bad_arguments_return_codes_not_crashes(lib):
    # null pointers / unsupported sizes are rejected before any CUDA call is made
    rc = lib.b2a_spectral_f32(None, 1, 100, 512, 128, None, None, 0, 0, 0, 0, None, 1, None, None, None, None, 0, 0, 0,
                              0.0, 1.0, None, None, None, 0, None)
    assert rc == -1 and b"null" in lib.b2a_last_error()
    buf = (ctypes.c_float * 1024)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    for n_fft, hop in ((65536, 128), (512, 0)):  # no forward route: a power of two above 32768; hop < 1
        rc = lib.b2a_spectral_f32(p, 1, 1024, n_fft, hop, p, None, 0, 0, 0, 0, None, 1, None, None, None, None, 0, 0, 0,
                                  0.0, 1.0, None, p, None, 0, None)
        assert rc == -2 and f"spectral: n_fft={n_fft} hop={hop}".encode() in lib.b2a_last_error()
    rc = lib.b2a_spectral_f32(p, 1, 100, 512, 128, p, None, 0, 0, 0, 0, None, 1, None, None, None, None, 0, 0, 0, 0.0,
                              1.0, None, p, None, 0, None)
    assert rc == -1 and b"n_fft/2" in lib.b2a_last_error()
    with pytest.raises(_lib.B2AError):
        lib.check(rc)
    # LARGE / DENSE: the checks of the gain + STFT + mel sequence come before its first launch
    for n_fft, hop in ((8192, 2048), (500, 125)):
        rc = lib.b2a_spectral_f32(p, 1, 20000, n_fft, hop, p, p, 0, 0, 0, 0, None, 1, None, None, None, None, 0, 0, 0,
                                  0.0, 1.0, None, None, None, 0, None)
        assert rc == -1 and lib.b2a_last_error() == b"spectral: neither mel_out nor stft_out requested"
        need = lib.b2a_spectral_workspace_bytes(1, 20000, n_fft, hop, 0, 0, 0, 1, 0)
        for ws, ws_bytes in ((None, 0), (p, need - 1)):  # the STFT under a mel-only call needs scratch
            rc = lib.b2a_spectral_f32(p, 1, 20000, n_fft, hop, p, p, 0, 0, 0, 0, None, 1, None, p, p, p, 4, 0, 0, 0.0,
                                      1.0, p, None, ws, ws_bytes, None)
            assert rc == -1 and lib.b2a_last_error() == b"spectral: workspace too small"
        rc = lib.b2a_spectral_f32(p, 3, 20000, n_fft, hop, p, p, 0, 0, 0, 0, p, 2, p, None, None, None, 0, 0, 0, 0.0,
                                  1.0, None, p, None, 0, None)  # the gain pass scales whole items of rows_per_gain rows
        assert rc == -1 and lib.b2a_last_error() == b"spectral: rows_per_gain"
    for n_fft, hop in ((65536, 16384), (512, 513)):  # no inverse route: a power of two above 32768; hop > n_fft
        rc = lib.b2a_istft_f32(p, 1, 4, n_fft, hop, p, None, 0, 0, 1024, p, None, 0, None)
        assert rc == -2 and f"istft: n_fft={n_fft} hop={hop}".encode() in lib.b2a_last_error()


def test_spectral_workspace_bytes(lib):
    # 0 where b2a_spectral_f32 needs no scratch: the FFT route, no route, no frames
    for n_fft, hop, T in ((512, 128, 20000), (4096, 1024, 20000), (65536, 128, 20000), (512, 0, 20000), (500, 125, 0)):
        assert [lib.b2a_spectral_workspace_bytes(3, T, n_fft, hop, 0, 0, 0, s, g) for s in (0, 1) for g in (0, 1)] == \
            [0, 0, 0, 0], (n_fft, hop, T)
    # LARGE / DENSE: the STFT [rows, F, n_frames] complex64 and / or the scaled signal [rows, T] float32, nothing more
    for n_fft, hop in ((8192, 2048), (32768, 8192), (500, 125), (8191, 2047)):
        T, pad, right_pad, drop_edge = 40000, (n_fft - hop) // 2, 37, 2
        N = lib.b2a_stft_num_frames(T, n_fft, hop, pad, right_pad, drop_edge)
        stft, scaled = 3 * (n_fft // 2 + 1) * N * 8, 3 * T * 4
        got = [lib.b2a_spectral_workspace_bytes(3, T, n_fft, hop, pad, right_pad, drop_edge, s, g)
               for s in (0, 1) for g in (0, 1)]
        assert got == [0, scaled, stft, stft + scaled], (n_fft, hop)


def test_spectral_tc_enable_is_a_stub(lib):
    # the tensor-core spectral kernel is gone: switching it off is a no-op, switching it on is unsupported
    assert lib.b2a_spectral_tc_enable(0) == 0
    assert lib.b2a_spectral_tc_enable(1) == -2 and b"tensor-core spectral kernel was removed" in lib.b2a_last_error()
    assert lib.b2a_spectral_tc_enable(0) == 0


# every forward / backward STFT entry point checks torch's stft(center=True) framing of the padded signal with the
# same codes and messages, before any CUDA call
FRAMING_ENTRY_POINTS = {  # prefix of the message, n_fft, hop
    "spectral": (512, 128),
    "stft_large": (8192, 2048),
    "stft_dense": (500, 125),
    "stft_backward": (512, 128),
    "spectral_loss": (512, 128),
}
FRAMING_FAILURES = {  # (T, pad, right_pad, pad_mode, drop_edge) as functions of n_fft -> (code, message)
    "negative_padding": (lambda n: (n, -1, 0, 0, 0), lambda n: (-1, "negative padding")),
    "negative_right_pad": (lambda n: (n, 0, -1, 0, 0), lambda n: (-1, "negative padding")),
    "negative_drop_edge": (lambda n: (n, 0, 0, 0, -1), lambda n: (-1, "negative padding")),
    "pad_mode": (lambda n: (n, 0, 0, 5, 0), lambda n: (-2, "pad mode 5")),
    "pad_mode_3": (lambda n: (n, 0, 0, 3, 0), lambda n: (-2, "pad mode 3")),  # circular: FIR padding only
    "pad_mode_negative": (lambda n: (n, 0, 0, -1, 0), lambda n: (-2, "pad mode -1")),
    "short_signal": (lambda n: (n // 4, 0, 0, 0, 0),
                     lambda n: (-1, f"n_fft/2 ({n // 2}) must be < padded length ({n // 4})")),
    "reflect_padding": (lambda n: (n, n, 0, 0, 0), lambda n: (-1, f"reflect padding ({n}) must be < signal length ({n})")),
    "reflect_right_padding": (lambda n: (n, 0, n, 0, 0),
                              lambda n: (-1, f"reflect padding ({n}) must be < signal length ({n})")),
    "no_frames": (lambda n: (n, 0, 0, 0, 100), lambda n: (-1, "no frames")),
}


def _call_framed(lib, who, T, n_fft, hop, pad, right_pad, pad_mode, drop_edge):
    buf = (ctypes.c_float * 1024)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    if who in ("spectral", "stft_large", "stft_dense"):  # the one forward entry point, on its three routes
        return lib.b2a_spectral_f32(p, 1, T, n_fft, hop, p, p, pad, right_pad, pad_mode, drop_edge, None, 1, None, None,
                                    None, None, 0, 0, 0, 0.0, 1.0, None, p, None, 0, None)
    if who == "stft_backward":
        return lib.b2a_stft_backward_f32(p, 1, T, n_fft, hop, p, None, pad, right_pad, pad_mode, drop_edge, p, p, 4096,
                                         None)
    return lib.b2a_spectral_loss_f32(p, p, 1, T, n_fft, hop, p, pad, right_pad, pad_mode, drop_edge, None, None, None,
                                     None, None, 0, 1e-5, 2.0, 1.0, 1.0, p, None, None, p, 4096, None)


@pytest.mark.parametrize("failure", sorted(FRAMING_FAILURES))
@pytest.mark.parametrize("who", sorted(FRAMING_ENTRY_POINTS))
def test_framing_failures_have_one_code_and_message(lib, who, failure):
    n_fft, hop = FRAMING_ENTRY_POINTS[who]
    shape, expect = FRAMING_FAILURES[failure]
    T, pad, right_pad, pad_mode, drop_edge = shape(n_fft)
    code, msg = expect(n_fft)
    rc = _call_framed(lib, who, T, n_fft, hop, pad, right_pad, pad_mode, drop_edge)
    assert rc == code
    assert lib.b2a_last_error() == f"{who}: {msg}".encode()


def test_missing_library_fails_loudly(tmp_path):
    with pytest.raises(ImportError, match="no CPU fallback"):
        _lib.B2ALibrary(str(tmp_path / "libb2a.so"))


def test_engine_rejects_cpu_tensors(lib):
    import torch

    from audiotools_b200 import AudioSignal
    from audiotools_b200.engine import Engine

    eng = Engine(lib)  # product configuration: require_cuda=True
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        eng.lufs(torch.zeros(1, 1, 16000), 16000)
    sig = AudioSignal(torch.zeros(1, 1, 16000), 16000)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        sig.stft()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        sig.loudness()


def test_host_num_frames_equals_the_abi_function():
    from audiotools_b200.engine import Engine

    lib = _lib.get_lib()
    rng = np.random.RandomState(0)
    for _ in range(300):
        T, n_fft, hop = int(rng.randint(-2, 100000)), int(2 ** rng.randint(0, 13)), int(rng.randint(-1, 5000))
        pad, rp, de = int(rng.randint(-1, 2048)), int(rng.randint(-1, 4096)), int(rng.choice([0, 0, 2]))
        assert Engine.num_frames(T, n_fft, hop, pad, rp, de) == lib.b2a_stft_num_frames(T, n_fft, hop, pad, rp, de)
