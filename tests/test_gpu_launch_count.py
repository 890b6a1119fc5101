"""``Engine.launches`` against the kernels the H100 actually ran (``-m gpu``): each call runs under ``torch.profiler``
with CUDA activities, and the kernel events whose demangled name lies in ``namespace b2a`` (every kernel of libb2a does)
must number exactly what the call added to ``Engine.launches``.  The sizes are those of a training batch, where the
overlap-save engine of csrc/fftconv.cu splits the rows into several chunks of at most 256 MB of spectra.
tests/test_sim_launch_count.py pins the counts of every method on the CPU simulator."""
import pytest
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
SR = 44100


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200.engine import get_engine

    return get_engine()


@pytest.fixture(scope="module")
def batch():
    """64 clips x 2 channels x 10 s at 44.1 kHz."""
    return 0.1 * torch.randn(64, 2, 10 * SR, generator=torch.Generator().manual_seed(0)).to(DEV)


def _profiled(eng, fn):
    """(libb2a kernels the profiler saw during fn(), what fn() added to ``Engine.launches``)."""
    torch.cuda.synchronize()
    n0 = eng.launches
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    added = eng.launches - n0
    gpu = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    if not gpu:
        pytest.skip("the profiler recorded no GPU activity")
    return sum("b2a::" in e.name for e in gpu), added


def _calls(eng, x):
    from audiotools_b200 import AudioSignal, _lib

    win = AudioSignal.get_window("hann", 2048, DEV)
    fb, lo, hi = AudioSignal._mel_tables(SR, 2048, 128, 0.0, None, DEV)
    win8k = AudioSignal.get_window("hann", 8192, DEV)
    fb8k, lo8k, hi8k = AudioSignal._mel_tables(SR, 8192, 128, 0.0, None, DEV)
    gain = torch.full((x.shape[0],), 0.5, device=DEV)
    db = torch.linspace(-6.0, 6.0, 10, device=DEV).expand(x.shape[0], 10)
    ir = torch.randn(1, 1, 1000, generator=torch.Generator().manual_seed(1)).to(DEV)
    short = x[:8]
    return {
        # taps 563 (one partition): fill, filter FFT, 2 chunks x (origins, block FFT, inverse FFT) = 8
        "sinc_filter": (lambda: eng.sinc_filter(x, torch.full((x.shape[0],), 4000.0), SR), 8),
        # taps 1211 (two partitions): fill, filter FFT, 4 chunks x (origins, block FFT, FIR, inverse FFT) = 18
        "equalizer": (lambda: eng.equalizer(x, SR, db), 18),
        "equalizer_backward": (lambda: eng.equalizer_backward(x, SR, db), 20),  # + the replicate-padding fold
        "circular_convolve": (lambda: eng.circular_convolve(x, ir), 9),  # + the IR's peak
        "circular_convolve_backward": (lambda: eng.circular_convolve_backward(x, ir), 10),  # + the tap reversal
        "lufs": (lambda: eng.lufs(x, SR, target_db=torch.tensor([-24.0], device=DEV)), 2),
        "loudness_stats": (lambda: eng.loudness_stats(x, SR), 3),
        "spectral": (lambda: eng.spectral(x, 2048, 512, win, gain=gain, want_scaled=True, mel_fb=fb, mel_lo=lo,
                                          mel_hi=hi, post=_lib.POST_LOG10, post_eps=1e-5, post_power=2.0,
                                          want_stft=False), 1),
        "spectral_large": (lambda: eng.spectral(short, 8192, 2048, win8k, gain=gain[:8], mel_fb=fb8k, mel_lo=lo8k,
                                                mel_hi=hi8k), 3),
        "pitch_shift": (lambda: eng.pitch_shift(short, SR, [2.0, -3.0] * 4), 4),
        "stoi": (lambda: eng.stoi(short, x[8:16], SR), 4),
    }


CASES = ("sinc_filter", "equalizer", "equalizer_backward", "circular_convolve", "circular_convolve_backward", "lufs",
         "loudness_stats", "spectral", "spectral_large", "pitch_shift", "stoi")


@pytest.mark.parametrize("name", CASES)
def test_launches_match_the_profiled_kernels(eng, batch, name):
    fn, expect = _calls(eng, batch)[name]
    fn()  # first call: module loading, cached tables and matrices
    assert _profiled(eng, fn) == (expect, expect)
