"""``b2a_stft_route`` is the one table that picks the kernel family of an STFT (inverse 0) and of an inverse STFT and
both backward passes (inverse 1); ``Engine.route`` memoises it.  The expected values below are the table of
include/b2a.h written out, not derived from the library."""
import torch

import audiotools_b200.engine as engine_mod
from audiotools_b200 import AudioSignal, _lib
from audiotools_b200.engine import Engine
from tests.cusim.sim_engine import sim_engine

CODE = {"N": _lib.ROUTE_NONE, "F": _lib.ROUTE_FFT, "L": _lib.ROUTE_LARGE, "D": _lib.ROUTE_DENSE}

POW2 = [2 ** k for k in range(1, 18)]  # 2 .. 131072
# the route of each length at a supported hop: (forward, inverse)
TABLE = {
    **dict(zip(POW2, zip("DDDDFFFFFFFFLLLNN", "DDDDDFFFFFFLLLLNN"))),
    3: ("D", "D"), 5: ("D", "D"), 401: ("D", "D"), 400: ("D", "D"), 4095: ("D", "D"),
    8191: ("D", "D"), 8193: ("N", "N"), 12288: ("N", "N"),
}


def _expected(n, hop, inverse):
    if hop < 1 or (inverse and hop > n):
        return _lib.ROUTE_NONE
    return CODE[TABLE[n][inverse]]


def _sweep():
    for n in sorted(TABLE):
        for hop in sorted({0, 1, n // 4, n, n + 1}):
            for inverse in (0, 1):
                yield n, hop, inverse


def test_route_table():
    lib = sim_engine().lib
    got = {case: lib.b2a_stft_route(*case) for case in _sweep()}
    assert got == {case: _expected(*case) for case in _sweep()}


def test_engine_route_equals_the_abi():
    lib = sim_engine().lib
    eng = Engine(lib, require_cuda=False)
    for case in _sweep():
        assert eng.route(*case) == lib.b2a_stft_route(*case), case
        assert eng.route(*case) == lib.b2a_stft_route(*case), case  # the memoised answer


def test_repeated_stft_makes_no_route_query(monkeypatch):
    lib = sim_engine().lib
    eng = Engine(lib, require_cuda=False)
    monkeypatch.setattr(engine_mod, "_ENGINE", eng)
    calls = []
    query = lib.b2a_stft_route
    monkeypatch.setattr(lib, "b2a_stft_route", lambda *a: calls.append(a) or query(*a))
    sig = AudioSignal(torch.randn(1, 1, 4000, generator=torch.Generator().manual_seed(0)), 16000)
    sig.stft(window_length=512, hop_length=128)
    assert calls == [(512, 128, 0)]
    sig.stft(window_length=512, hop_length=128)
    assert calls == [(512, 128, 0)]
