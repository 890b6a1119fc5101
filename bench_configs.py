#!/usr/bin/env python
"""bench_configs.py -- auxiliary measurements of the OTHER BASELINE.json configs (the contract bench is
bench.py, which measures configs[1]).  One JSON line per config: device-resident throughput (CUDA events,
>= 3 warm-ups, inputs larger than L2 or rotated), algorithmic bytes, and the CPU oracle on a bounded sample.

    python bench_configs.py [--only cfg1,cfg3,cfg4,cfg5,istft,specaug,dense,largewin,grad,loss,gate,masked,effects_grad,
                                      specaug_grad,stoi,stoi_grad] [--no-cpu]

Multi-GPU (BASELINE configs[3] = 512 items on 4 GPUs, configs[4] = 2048 items on 8 GPUs): one process per GPU,
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 4 --master-addr 127.0.0.1 --master-port 29511 \
        bench_configs.py --gpus 4 --only cfg4
every rank owns its slice of the batch (128 / 256 items, seeded by rank; no data-path collective), the timed region
is bracketed by a barrier + synchronize, the step time is the MAX over ranks and rank 0 prints the whole-job line.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REPO)


WORLD = int(os.environ.get("WORLD_SIZE", "1"))
RANK = int(os.environ.get("RANK", "0"))
LOCAL = int(os.environ.get("LOCAL_RANK", "0"))


def _barrier():
    if WORLD > 1:
        import torch.distributed as dist

        dist.barrier()


def timed(fn, warmup=3, steps=10):
    """ms per step: CUDA events on the launching stream, >= 3 warm-ups unless stated, barrier + synchronize on both
    sides and the MAX over ranks when launched under torchrun."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    _barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    _barrier()
    ms = e0.elapsed_time(e1) / steps
    if WORLD > 1:
        import torch.distributed as dist

        t = torch.tensor([ms], device=f"cuda:{LOCAL}", dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t.item())
    return ms


def emit(line):
    if RANK == 0:
        line["n_gpus"] = WORLD
        print(json.dumps(line), flush=True)


def cpu_time(fn, reps=2):
    fn()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t0) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="cfg1,cfg3,cfg4,cfg5,istft,specaug,dense,gate,masked")
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--gpus", type=int, default=1, help="ranks (informational: the launcher sets WORLD_SIZE)")
    args = ap.parse_args()
    import __graft_entry__ as graft

    graft.build()
    torch.cuda.set_device(LOCAL)
    if WORLD > 1:
        import torch.distributed as dist

        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device(f"cuda:{LOCAL}"))
        args.no_cpu = True
    from audiotools_b200 import AudioSignal
    from audiotools_b200.data import transforms as tfm
    from oracle import signal_path as sp

    dev = f"cuda:{LOCAL}"
    peak = 3350.0  # GB/s: H100 SXM data sheet (HBM3), not measured
    torch.set_num_threads(os.cpu_count() or 1)
    only = set(args.only.split(","))

    if "cfg1" in only:  # batch=4 mono 1s@16kHz stft(512,128): launch-latency bound
        x = torch.randn(4, 1, 16000, generator=torch.Generator().manual_seed(0))
        sig = AudioSignal(x.clone(), 16000).to(dev)
        ms = timed(lambda: sig.stft(window_length=512, hop_length=128), steps=50)
        line = {"config": "cfg1 batch=4 mono 1s@16k stft(512,128)", "ms": ms, "clips_per_s": 4 / ms * 1e3,
                "alg_bytes": 64000 + 1036224}
        if not args.no_cpu:
            line["cpu_ms"] = 1e3 * cpu_time(lambda: sp.stft(x, 16000, 512, 128), reps=20)
        emit(line)

    if "cfg3" in only:  # batch=256 mono 30s@48k -> 16k polyphase resample + low_pass(8k)
        B = 256
        g = torch.Generator().manual_seed(0)
        x = (0.1 * torch.randn(B, 1, 1440000, generator=g)).to(dev)  # 1.47 GB > L2

        def run():
            s = AudioSignal(x, 48000)
            s.resample(16000)
            s.low_pass(8000)
            return s

        ms_rs = timed(lambda: AudioSignal(x, 48000).resample(16000), steps=5)
        ms = timed(run, steps=5)
        alg = B * (5760000 + 1920000) + B * 2 * 1920000
        line = {"config": "cfg3 batch=256 mono 30s@48k resample->16k + low_pass(8k)", "ms": ms, "ms_resample": ms_rs,
                "clips_per_s": B / ms * 1e3, "alg_bytes": alg, "achieved_GBps": alg / ms / 1e6,
                "frac_of_hbm_peak": alg / ms / 1e6 / peak}
        if not args.no_cpu:
            xc = x[:8].cpu()
            t = cpu_time(lambda: sp.low_pass(sp.resample(xc, 48000, 16000), 16000, 8000), reps=1)
            line["cpu_clips_per_s"] = 8 / t
        emit(line)
        del x

    if "cfg4" in only:  # batch=512 Compose[EQ + IR-convolve + pitch_shift +-2], mono 10s@44.1k (one GPU's share: 128)
        B, T, sr = 128, 441000, 44100
        g = torch.Generator().manual_seed(RANK)
        x = 0.1 * torch.randn(B, 1, T, generator=g)
        t = torch.arange(sr) / sr
        irs = []
        for i in range(8):
            h = torch.randn(1, 1, sr, generator=g) * torch.exp(-t / 0.3) * 0.1
            h[..., 40 + i] = 1.0
            irs.append(AudioSignal(h, sr))
        transform = tfm.Compose([tfm.Equalizer(), tfm.RoomImpulseResponse(sources=irs),
                                 tfm.PitchShift(("choice", [-2, 2]))])
        sig = AudioSignal(x, sr)
        kwargs = transform.batch_instantiate(list(range(RANK * B, (RANK + 1) * B)), sig)
        sig = sig.to(dev)
        from audiotools_b200 import util

        kwargs = util.prepare_batch(kwargs, dev)
        ms = timed(lambda: transform(sig.clone(), **kwargs), warmup=3, steps=5)
        per = {}
        for name, fn in [("equalizer", lambda: sig.clone().equalizer(kwargs["Compose"]["0.Equalizer"]["eq"])),
                         ("apply_ir", lambda: sig.clone().apply_ir(kwargs["Compose"]["1.RoomImpulseResponse"]["ir_signal"].clone(),
                                                                   kwargs["Compose"]["1.RoomImpulseResponse"]["drr"],
                                                                   kwargs["Compose"]["1.RoomImpulseResponse"]["eq"])),
                         ("pitch_shift", lambda: sig.clone().pitch_shift(2))]:
            per[name] = timed(fn, warmup=1, steps=3)
        line = {"config": f"cfg4 batch={B * WORLD} ({B} per GPU) mono 10s@44.1k Compose[EQ+RoomIR+PitchShift+-2]", "ms": ms,
                "clips_per_s": B * WORLD / ms * 1e3, "per_gpu_batch": B, "global_batch": B * WORLD, "ms_parts": per,
                "timing": "CUDA events, barrier + synchronize both sides, max over ranks; no data-path collective"}
        emit(line)

    if "cfg5" in only:  # batch=2048 2ch 10s@44.1k full augment + LUFS + log-mel on 8 GPUs: one GPU's share (256 items)
        B, T, sr = 256, 441000, 44100
        g = torch.Generator().manual_seed(100 + RANK)
        x = 0.1 * torch.randn(B, 2, T, generator=g)
        t = torch.arange(sr) / sr
        irs = []
        for i in range(8):
            h = torch.randn(1, 1, sr, generator=g) * torch.exp(-t / 0.3) * 0.1
            h[..., 40 + i] = 1.0
            irs.append(AudioSignal(h, sr))
        transform = tfm.Compose([tfm.Equalizer(), tfm.RoomImpulseResponse(sources=irs),
                                 tfm.PitchShift(("choice", [-2, 2]))])
        sig = AudioSignal(x, sr)
        kwargs = transform.batch_instantiate(list(range(RANK * B, (RANK + 1) * B)), sig)
        sig = sig.to(dev)
        from audiotools_b200 import util

        kwargs = util.prepare_batch(kwargs, dev)

        def full():
            s = transform(sig.clone(), **kwargs)
            s.normalize(-24.0)
            return s.mel_spectrogram(n_mels=128, window_length=2048, hop_length=512, log=True)

        ms = timed(full, warmup=3, steps=5)
        emit({"config": f"cfg5 batch={B * WORLD} ({B} per GPU) 2ch 10s@44.1k Compose[EQ+RoomIR+PitchShift+-2] + "
                        "LUFS normalize + log-mel", "ms": ms, "clips_per_s": B * WORLD / ms * 1e3, "per_gpu_batch": B,
              "global_batch": B * WORLD,
              "timing": "CUDA events, barrier + synchronize both sides, max over ranks; no data-path collective"})
        del x, sig

    if "istft" in only:  # SURVEY 8f.1: inverse STFT at cfg2's shape (64 x 2ch x 10 s @ 44.1 kHz, 2048/512)
        g = torch.Generator().manual_seed(0)
        x = (0.1 * torch.randn(64, 2, 441000, generator=g)).to(dev)
        sig = AudioSignal(x, 44100)
        sig.stft(window_length=2048, hop_length=512)
        X = sig.stft_data  # 905 MB > L2
        ms = timed(lambda: sig.istft(window_length=2048, hop_length=512), steps=10)
        w = torch.hann_window(2048, periodic=True, device=dev)
        Xr = X.reshape(128, 1025, -1)
        ms_torch = timed(lambda: torch.istft(Xr, 2048, 512, window=w, center=True, length=441000), steps=5)
        alg = X.numel() * 8 + x.numel() * 4
        emit({"config": "istft 64x2ch 10s@44.1k n_fft=2048 hop=512", "ms": ms, "ms_torch_istft_cufft": ms_torch,
                          "clips_per_s": 64 / ms * 1e3, "alg_bytes": alg, "achieved_GBps": alg / ms / 1e6,
                          "frac_of_hbm_peak": alg / ms / 1e6 / peak})

    if "dense" in only:  # arbitrary window length (csrc/dft.cu): the 25 ms / 10 ms / 80-mel speech front-end at 16 kHz
        B, T, sr = 64, 160000, 16000
        x = (0.1 * torch.randn(B, 1, T, generator=torch.Generator().manual_seed(0))).to(dev)
        sig = AudioSignal(x, sr)
        ms_stft = timed(lambda: sig.stft(window_length=400, hop_length=160), steps=10)
        ms_mel = timed(lambda: sig.mel_spectrogram(n_mels=80, window_length=400, hop_length=160, log=True), steps=10)
        sig.stft(window_length=400, hop_length=160)
        ms_inv = timed(lambda: sig.istft(window_length=400, hop_length=160), steps=10)
        w = torch.hann_window(400, periodic=True, device=dev)
        ms_torch = timed(lambda: torch.stft(x.reshape(B, T), 400, 160, window=w, center=True, return_complex=True), steps=10)
        nfr = 1 + T // 160
        macs = B * nfr * 400 * 201  # complex-real multiply-accumulates = FFMA2 instructions x 32 lanes
        emit({"config": "dense DFT 64 x 1ch x 10s@16k window 400 hop 160 (+ 80-mel log-mel, inverse)", "ms_stft": ms_stft,
              "ms_logmel": ms_mel, "ms_istft": ms_inv, "ms_torch_stft_cufft": ms_torch, "clips_per_s": B / ms_mel * 1e3,
              "gflops_stft": 4 * macs / ms_stft / 1e6, "fp32_peak_gflops": 67000.0,  # H100 SXM data sheet
              "frac_of_fp32_peak": 4 * macs / ms_stft / 1e6 / 67000.0})

    if "largewin" in only:  # large power-of-two windows (csrc/fft_large.cu): the default 8192 window at 192 kHz
        import subprocess

        from audiotools_b200.engine import get_engine

        B, C, T, sr = 64, 2, 1_920_000, 192000
        g = torch.Generator().manual_seed(0)
        x = torch.empty(B, C, T)
        for i in range(0, B, 8):
            x[i:i + 8] = 0.1 * torch.randn(8, C, T, generator=g)
        x = x.to(dev)  # 983 MB > L2
        sig = AudioSignal(x, sr)
        eng = get_engine()
        ms_stft = timed(lambda: sig.stft(), steps=5)  # default stft_params: 8192 / 2048, hann
        ms_logmel = timed(lambda: sig.mel_spectrogram(n_mels=128, log=True), steps=5)
        sig.stft()
        X = sig.stft_data
        ms_istft = timed(lambda: sig.istft(), steps=5)
        ms_32k = timed(lambda: AudioSignal(x, sr).stft(window_length=32768, hop_length=8192), steps=3)
        xs = x.reshape(B * C, T)
        wt = torch.hann_window(8192, periodic=True, device=dev)
        ms_torch = timed(lambda: torch.stft(xs, 8192, 2048, window=wt, center=True, return_complex=True), steps=5)
        Xr = X.reshape(B * C, 4097, -1)
        ms_torch_inv = timed(lambda: torch.istft(Xr, 8192, 2048, window=wt, center=True, length=T), steps=5)
        alg = x.numel() * 4 + X.numel() * 8  # x read + STFT written
        try:
            plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(LOCAL)],
                                  capture_output=True, text=True, timeout=30).stdout.strip()
        except Exception:  # noqa: BLE001 (informational field)
            plim = "unknown"
        emit({"config": "largewin 64x2ch 10s@192k default window 8192 hop 2048 (stft, log-mel, istft; stft 32768)",
              "kernel": eng.spectral_kernel_name(8192, 2048, want_mel=False, want_stft=True),
              "ms_stft": ms_stft, "ms_logmel": ms_logmel, "ms_istft": ms_istft, "ms_stft_32768": ms_32k,
              "ms_torch_stft_cufft": ms_torch, "ms_torch_istft_cufft": ms_torch_inv,
              "clips_per_s_stft": B / ms_stft * 1e3, "alg_bytes_stft": alg, "achieved_GBps": alg / ms_stft / 1e6,
              "frac_of_hbm_peak": alg / ms_stft / 1e6 / peak, "gpu": torch.cuda.get_device_name(LOCAL),
              "power_limit": plim})
        del X, Xr, sig, x

    if "grad" in only:  # forward + backward through the spectral front end (csrc/grad.cu) next to torch autograd
        import subprocess

        import torch.nn.functional as F

        from audiotools_b200.engine import get_engine

        eng = get_engine()
        sr = 44100

        def l1_log(a, b, pw):
            return F.l1_loss(a.clamp(1e-5).pow(pw).log10(), b.clamp(1e-5).pow(pw).log10())

        # the reference's losses (ref:audiotools/metrics/spectral.py:70-95, 159-192): (kind, n_mels, windows, mag, pow)
        losses = [("mel", [150, 80], [2048, 512], 1.0, 2.0), ("stft", None, [2048, 512], 1.0, 2.0),
                  ("mel", [5, 10, 20, 40, 80, 160, 320], [32, 64, 128, 256, 512, 1024, 2048], 0.0, 1.0)]
        fbs = {}

        def torch_mel(x, nm, wl):  # the reference's arithmetic on the GPU: torch.stft (cuFFT) + abs + matmul (cuBLAS)
            if (nm, wl) not in fbs:
                fbs[nm, wl] = torch.from_numpy(np.asarray(AudioSignal.get_mel_filters(sr, wl, nm), np.float32)).to(dev)
            return (torch_mag(x, wl).transpose(2, -1) @ fbs[nm, wl].T).transpose(-1, 2)

        def torch_mag(x, wl):
            w = AudioSignal.get_window("hann", wl, x.device)
            X = torch.stft(x.reshape(-1, x.shape[-1]), wl, wl // 4, window=w, center=True, return_complex=True)
            return X.reshape(*x.shape[:2], *X.shape[1:]).abs()

        def loss_of(x, y, cfg, ours):
            kind, nms, wls, mag, pw = cfg
            loss = 0.0
            for i, wl in enumerate(wls):
                if kind == "mel":
                    if ours:
                        a = AudioSignal(x, sr).mel_spectrogram(nms[i], window_length=wl, hop_length=wl // 4)
                        b = AudioSignal(y, sr).mel_spectrogram(nms[i], window_length=wl, hop_length=wl // 4)
                    else:
                        a, b = torch_mel(x, nms[i], wl), torch_mel(y, nms[i], wl)
                else:
                    if ours:
                        sa, sb = AudioSignal(x, sr), AudioSignal(y, sr)
                        sa.stft(wl, wl // 4, "hann")
                        sb.stft(wl, wl // 4, "hann")
                        a, b = sa.magnitude, sb.magnitude
                    else:
                        a, b = torch_mag(x, wl), torch_mag(y, wl)
                loss = loss + l1_log(a, b, pw) + mag * F.l1_loss(a, b)
            return loss

        g = torch.Generator().manual_seed(0)
        x = (0.1 * torch.randn(16, 1, sr, generator=g)).to(dev)
        y = (0.1 * torch.randn(16, 1, sr, generator=g)).to(dev)
        res = {}
        for name, cfg in zip(["mel_default", "stft_default", "mel_7scale"], losses):
            for ours in (True, False):
                def step():
                    xg = x.clone().requires_grad_()
                    loss_of(xg, y, cfg, ours).backward()

                res[name + ("_ms" if ours else "_torch_ms")] = timed(step, steps=20)
        # cfg2 size: 64 x 2 ch x 10 s, 2048 / 512, 128 mels -- the backward alone (forward done once, untimed)
        B, C, T = 64, 2, 441000
        xb = (0.1 * torch.randn(B, C, T, generator=g)).to(dev)
        xg = xb.clone().requires_grad_()
        mel = AudioSignal(xg, sr).mel_spectrogram(128, window_length=2048, hop_length=512)
        gm = torch.randn_like(mel)
        ms_bwd = timed(lambda: torch.autograd.grad(mel, xg, gm, retain_graph=True), steps=5)
        xt = xb.clone().requires_grad_()
        melt = torch_mel(xt, 128, 2048)
        ms_bwd_torch = timed(lambda: torch.autograd.grad(melt, xt, gm, retain_graph=True), steps=5)
        F_, N = 1025, mel.shape[-1]
        Lpp = T + 2048
        # mel backward: STFT read twice, dmel read, dX written; STFT adjoint: dX read, padded range written; pad
        # adjoint: padded range read, dx written
        alg = B * C * (3 * 8 * F_ * N + 4 * 128 * N + 8 * F_ * N + 4 * Lpp + 4 * Lpp + 4 * T)
        try:
            plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(LOCAL)],
                                  capture_output=True, text=True, timeout=30).stdout.strip()
        except Exception:  # noqa: BLE001 (informational field)
            plim = "unknown"
        emit({"config": "grad: forward+backward of the reference's 3 spectral losses at 16x1ch x 1s@44.1k; "
                        "mel backward at 64x2ch x 10s@44.1k (2048/512, 128 mels)",
              **res, "ms_mel_backward_cfg2": ms_bwd, "ms_mel_backward_cfg2_torch_autograd": ms_bwd_torch,
              "alg_bytes_mel_backward_cfg2": alg, "achieved_GBps_mel_backward_cfg2": alg / ms_bwd / 1e6,
              "frac_of_hbm_peak": alg / ms_bwd / 1e6 / peak, "launches_total": eng.launches,
              "gpu": torch.cuda.get_device_name(LOCAL), "power_limit": plim})
        del xb, xg, xt, mel, melt, gm

    if "loss" in only:  # audiotools_b200.metrics: fused losses (csrc/loss.cu) vs the reference's code vs torch autograd
        import subprocess

        import torch.nn.functional as F

        from audiotools_b200 import metrics

        sr = 44100
        # the reference's code (ref:audiotools/metrics/spectral.py:70-95, 159-192) over this package's AudioSignal, and
        # the same arithmetic on torch.stft (cuFFT) + abs + matmul (cuBLAS)
        cfgs = {"mel_default": dict(n_mels=[150, 80], window_lengths=[2048, 512]),
                "stft_default": dict(window_lengths=[2048, 512]),
                "mel_7scale": dict(n_mels=[5, 10, 20, 40, 80, 160, 320],
                                   window_lengths=[32, 64, 128, 256, 512, 1024, 2048], mag_weight=0.0, pow=1.0,
                                   mel_fmin=[0.0] * 7, mel_fmax=[None] * 7)}
        fbs = {}

        def t_mag(x, wl):
            w = AudioSignal.get_window("hann", wl, x.device)
            X = torch.stft(x.reshape(-1, x.shape[-1]), wl, wl // 4, window=w, center=True, return_complex=True)
            return X.reshape(*x.shape[:2], *X.shape[1:]).abs()

        def composed(x, y, cfg, on_torch):
            loss, mw, pw = 0.0, cfg.get("mag_weight", 1.0), cfg.get("pow", 2.0)
            for i, wl in enumerate(cfg["window_lengths"]):
                nm = cfg["n_mels"][i] if "n_mels" in cfg else None
                if on_torch:
                    a, b = t_mag(x, wl), t_mag(y, wl)
                    if nm is not None:
                        if (nm, wl) not in fbs:
                            fbs[nm, wl] = torch.from_numpy(
                                np.asarray(AudioSignal.get_mel_filters(sr, wl, nm), np.float32)).to(dev)
                        a = (a.transpose(2, -1) @ fbs[nm, wl].T).transpose(-1, 2)
                        b = (b.transpose(2, -1) @ fbs[nm, wl].T).transpose(-1, 2)
                elif nm is not None:
                    a = AudioSignal(x, sr).mel_spectrogram(nm, window_length=wl, hop_length=wl // 4)
                    b = AudioSignal(y, sr).mel_spectrogram(nm, window_length=wl, hop_length=wl // 4)
                else:
                    sa, sb = AudioSignal(x, sr), AudioSignal(y, sr)
                    sa.stft(wl, wl // 4, "hann")
                    sb.stft(wl, wl // 4, "hann")
                    a, b = sa.magnitude, sb.magnitude
                loss = loss + F.l1_loss(a.clamp(1e-5).pow(pw).log10(), b.clamp(1e-5).pow(pw).log10())
                loss = loss + mw * F.l1_loss(a, b)
            return loss

        def path(name, cfg):
            if name == "fused":
                mod = (metrics.MelSpectrogramLoss if "n_mels" in cfg else metrics.MultiScaleSTFTLoss)(**cfg)
                return lambda x, y: mod(AudioSignal(x, sr), AudioSignal(y, sr))
            return lambda x, y: composed(x, y, cfg, name == "torch")

        try:
            plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(LOCAL)],
                                  capture_output=True, text=True, timeout=30).stdout.strip()
        except Exception:  # noqa: BLE001 (informational field)
            plim = "unknown"
        g = torch.Generator().manual_seed(0)
        for size, (B, C, secs, steps) in {"16x1chx1s": (16, 1, 1, 20), "64x2chx10s": (64, 2, 10, 5)}.items():
            x = (0.1 * torch.randn(B, C, secs * sr, generator=g)).to(dev)
            y = (0.1 * torch.randn(B, C, secs * sr, generator=g)).to(dev)
            res = {}
            for lname, cfg in cfgs.items():
                for pname in ("fused", "composed", "torch"):
                    fn = path(pname, cfg)

                    def fwd_bwd():
                        xg = x.clone().requires_grad_()
                        fn(xg, y).backward()

                    def fwd():
                        with torch.no_grad():
                            fn(x, y)

                    for mode, step in (("fwd_bwd", fwd_bwd), ("fwd_nograd", fwd)):
                        torch.cuda.synchronize()
                        torch.cuda.empty_cache()
                        torch.cuda.reset_peak_memory_stats(dev)
                        base = torch.cuda.memory_allocated(dev)
                        ms = timed(step, steps=steps)
                        res[f"{lname}_{pname}_{mode}_ms"] = ms
                        res[f"{lname}_{pname}_{mode}_peak_MB"] = (torch.cuda.max_memory_allocated(dev) - base) / 2**20
            emit({"config": f"loss: forward+backward / no_grad forward of the reference's spectral losses at {size}@44.1k; "
                            "fused = audiotools_b200.metrics (csrc/loss.cu), composed = the reference's code over "
                            "AudioSignal, torch = the same arithmetic on torch.stft; peak_MB above the inputs",
                  **res, "gpu": torch.cuda.get_device_name(LOCAL), "power_limit": plim})
            del x, y

    if "gate" in only:  # SpectralGate (csrc/specmask.cu) at 64 x 2ch x 10 s: stft x2 + gate + istft
        from audiotools_b200.ml.layers import SpectralGate

        g = torch.Generator().manual_seed(0)
        x = (0.1 * torch.randn(64, 2, 441000, generator=g)).to(dev)
        nz = (0.01 * torch.randn(1, 1, 88200, generator=g)).to(dev)
        gate = SpectralGate().to(dev)
        sig, nzs = AudioSignal(x, 44100), AudioSignal(nz, 44100)
        ms = timed(lambda: gate(sig, nzs, 0.9), warmup=3, steps=5)
        from audiotools_b200.engine import get_engine

        s2 = sig.clone(); s2.stft(2048, 512, "sqrt_hann"); n2 = nzs.clone(); n2.stft(2048, 512, "sqrt_hann")
        ms_k = timed(lambda: get_engine().spec_gate(s2.stft_data, n2.stft_data, 3.0, torch.tensor([0.9]), gate._rf.tolist(),
                                                    gate._rt.tolist()), steps=10)
        alg = 2 * s2.stft_data.numel() * 8
        emit({"config": "SpectralGate 64x2ch 10s@44.1k (2048/512): clone + 2 stft + gate kernels + istft", "ms": ms,
              "ms_gate_kernels": ms_k, "alg_bytes_gate": alg, "gate_GBps": alg / ms_k / 1e6, "gate_frac_of_hbm_peak": alg / ms_k / 1e6 / peak})

    if "masked" in only:  # SURVEY 8f.3: a prob = 0.5 augmentation chain, kernel-side bypass flags vs gather / scatter
        B, T, sr = 128, 441000, 44100
        g = torch.Generator().manual_seed(0)
        x = 0.1 * torch.randn(B, 1, T, generator=g)
        transform = tfm.Compose([tfm.VolumeNorm(prob=0.5), tfm.Equalizer(prob=0.5), tfm.LowPass(prob=0.5),
                                 tfm.HighPass(prob=0.5), tfm.PitchShift(("choice", [-2, 2]), prob=0.5)])
        sig = AudioSignal(x, sr)
        kwargs = transform.batch_instantiate(list(range(B)), sig)
        sig = sig.to(dev)
        from audiotools_b200 import util

        kwargs = util.prepare_batch(kwargs, dev)
        ms_aware = timed(lambda: transform(sig.clone(), **kwargs), warmup=3, steps=5)
        for t in transform.transforms:
            t._mask_aware = False
        ms_gather = timed(lambda: transform(sig.clone(), **kwargs), warmup=3, steps=5)
        emit({"config": f"masked chain batch={B} mono 10s@44.1k Compose[VolumeNorm, Equalizer, LowPass, HighPass, PitchShift] "
                        "each prob 0.5", "ms_bypass_flags": ms_aware, "ms_gather_scatter": ms_gather,
              "clips_per_s": B / ms_aware * 1e3})

    if "effects_grad" in only:  # backward kernels of the time-domain effects at 64 x 2ch x 10 s@44.1k
        import subprocess

        from audiotools_b200.engine import get_engine
        from tests import effects_grad_cases as ec

        try:
            plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(LOCAL)],
                                  capture_output=True, text=True, timeout=30).stdout.strip()
        except Exception:  # noqa: BLE001 (informational field)
            plim = "unknown"
        eng = get_engine()
        B, C, T, sr = 64, 2, 441000, 44100
        g = torch.Generator().manual_seed(0)
        x = (0.1 * torch.randn(B, C, T, generator=g)).to(dev)
        db = ec.db_curve(B, 6, 1).to(dev)
        ir = ec.synthetic_ir(B, sr, 2).to(dev)
        fp32_peak = 67e12  # FLOP/s: H100 SXM data sheet, dense FP32, not measured
        cases = {"resample_44k1_16k": ("resample", dict(new_sr=16000)),
                 "resample_44k1_22k05": ("resample", dict(new_sr=22050)),
                 "equalizer_6band": ("equalizer", dict(db=db)), "apply_ir_1s": ("apply_ir", dict(ir=ir))}
        res = {}
        for name, (method, kw) in cases.items():
            fn = ec.ours(method, sr, **kw)
            y = fn(x)
            gy = torch.randn(y.shape, generator=g).to(dev)

            def fwd_bwd():
                xg = x.clone().requires_grad_()
                (fn(xg) * gy).sum().backward()

            def fwd():
                with torch.no_grad():
                    fn(x)

            res[f"{name}_fwd_bwd_ms"] = timed(fwd_bwd, steps=5)
            res[f"{name}_fwd_ms"] = timed(fwd, steps=5)
            ref = ec.ref(method, sr, **kw)

            def torch_fwd_bwd():
                xg = x.clone().requires_grad_()
                (ref(xg) * gy).sum().backward()

            res[f"{name}_torch_autograd_fp32_ms"] = timed(torch_fwd_bwd, warmup=1, steps=3)
        # each backward entry point alone, next to its forward launch at the same shape
        for new_sr, tag in ((16000, "44k1_16k"), (22050, "44k1_22k05")):
            y = eng.resample(x, sr, new_sr)
            gy = torch.randn(y.shape, generator=g).to(dev)
            res[f"resample_{tag}_forward_ms"] = timed(lambda: eng.resample(x, sr, new_sr), steps=10)
            res[f"resample_{tag}_backward_ms"] = ms_b = timed(lambda: eng.resample_backward(gy, T, sr, new_sr), steps=10)
            kt, width, old, new = eng._resample_kernel(sr, new_sr, dev)
            flop = 2.0 * B * C * y.shape[-1] * kt.shape[0]  # one FMA per (output, tap), both directions
            byts = 4.0 * B * C * (T + y.shape[-1])
            res[f"resample_{tag}_backward_alg_GFLOP"] = flop / 1e9
            res[f"resample_{tag}_backward_frac_of_fp32_peak"] = flop / (ms_b * 1e-3) / fp32_peak
            res[f"resample_{tag}_backward_frac_of_hbm_peak"] = byts / (ms_b * 1e-3) / (peak * 1e9)
        gx = torch.randn(B, C, T, generator=g).to(dev)
        res["equalizer_forward_ms"] = timed(lambda: eng.equalizer(x, sr, db), steps=10)
        res["equalizer_backward_ms"] = timed(lambda: eng.equalizer_backward(gx, sr, db), steps=10)
        res["circconv_forward_ms"] = timed(lambda: eng.circular_convolve(x, ir), steps=10)
        res["circconv_backward_ms"] = timed(lambda: eng.circular_convolve_backward(gx, ir), steps=10)
        res["peak_scale_backward_ms"] = ms_p = timed(lambda: eng.peak_scale_backward(gx, x, x), steps=10)
        res["peak_scale_backward_frac_of_hbm_peak"] = 4.0 * B * C * T * 5 / (ms_p * 1e-3) / (peak * 1e9)
        emit({"config": "effects_grad 64x2ch 10s@44.1k: forward+backward, no-grad forward, each backward entry point "
                        "next to its forward, and torch autograd (fp32, same GPU) over the float64 restatements' code",
              **res, "gpu": torch.cuda.get_device_name(LOCAL), "power_limit": plim})
        del x, gx

    if "specaug_grad" in only:  # backward kernels of the spectral masks and the gate at 64 x 2ch x 10 s@44.1k, 2048/512
        import subprocess

        from audiotools_b200.engine import get_engine
        from audiotools_b200.ml.layers import SpectralGate

        try:
            plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(LOCAL)],
                                  capture_output=True, text=True, timeout=30).stdout.strip()
        except Exception:  # noqa: BLE001 (informational field)
            plim = "unknown"
        eng = get_engine()
        B, C, T, sr = 64, 2, 441000, 44100
        g = torch.Generator().manual_seed(0)
        x = (0.1 * torch.randn(B, C, T, generator=g)).to(dev)
        nz = (0.01 * torch.randn(1, 1, 22050, generator=g)).to(dev)
        fmin = (torch.rand(B, generator=g) * 8000).to(dev)
        fmax = fmin + 2000.0
        tmin = (torch.rand(B, generator=g) * 9.0).to(dev)
        tmax = tmin + 0.25
        gy = torch.randn(B, C, T, generator=g).to(dev)
        gate = SpectralGate().to(dev)
        amount = torch.full((B,), 0.9, device=dev)
        res = {}

        def chain(v):
            s = AudioSignal(v, sr)
            s.stft(window_length=2048, hop_length=512)
            s.mask_frequencies(fmin, fmax).mask_timesteps(tmin, tmax)
            return s.istft(window_length=2048, hop_length=512).audio_data

        def gated(v):
            return gate(AudioSignal(v, sr), AudioSignal(nz, sr), amount).audio_data

        w = torch.hann_window(2048, periodic=True, device=dev)
        sw = w.sqrt()

        def torch_chain(v):  # the reference's tensor ops (torch.stft / polar masks / torch.istft) under torch autograd
            X = torch.stft(v.reshape(-1, T), 2048, 512, window=w, center=True, return_complex=True).reshape(B, C, 1025, -1)
            for vals, lo, hi, shape in ((torch.linspace(0, sr / 2, 1025, device=dev), fmin, fmax, (1, 1, -1, 1)),
                                        (torch.linspace(0, T / sr, X.shape[-1], device=dev), tmin, tmax, (1, 1, 1, -1))):
                m = (lo.reshape(-1, 1, 1, 1) <= vals.reshape(shape)) & (vals.reshape(shape) < hi.reshape(-1, 1, 1, 1))
                X = torch.abs(X).masked_fill(m, 0.0) * torch.exp(1j * torch.angle(X).masked_fill(m, 0.0))
            return torch.istft(X.reshape(-1, 1025, X.shape[-1]), 2048, 512, window=w, center=True, length=T).reshape(B, C, T)

        def torch_gate(v):  # ref:audiotools/ml/layers/spectral_gate.py:97-127's tensor ops under torch autograd
            X = torch.stft(v.reshape(-1, T), 2048, 512, window=sw, center=True, return_complex=True).reshape(B, C, 1025, -1)
            N = torch.stft(nz.reshape(1, -1), 2048, 512, window=sw, center=True, return_complex=True)
            nz_db = 20 * N.abs().clamp(1e-4).log10()
            th = nz_db.mean(-1, keepdim=True) + nz_db.std(-1, keepdim=True) * 3.0
            m = ((20 * X.abs().clamp(1e-4).log10()) < th).float().reshape(B * C, 1, 1025, -1)
            k = gate.smoothing_filter
            m = torch.nn.functional.conv2d(m, k, padding=(k.shape[-2] // 2, k.shape[-1] // 2)).reshape(X.shape)
            X = X * (1 - m * amount.reshape(-1, 1, 1, 1))
            return torch.istft(X.reshape(-1, 1025, X.shape[-1]), 2048, 512, window=sw, center=True, length=T).reshape(B, C, T)

        for name, fn, ref in (("mask_chain", chain, torch_chain), ("spectral_gate", gated, torch_gate)):
            def fwd_bwd(f=fn):
                xg = x.clone().requires_grad_()
                (f(xg) * gy).sum().backward()

            def fwd(f=fn):
                with torch.no_grad():
                    f(x)

            def torch_fwd_bwd(f=ref):
                xg = x.clone().requires_grad_()
                (f(xg) * gy).sum().backward()

            res[f"{name}_fwd_bwd_ms"] = timed(fwd_bwd, steps=5)
            res[f"{name}_no_grad_fwd_ms"] = timed(fwd, steps=5)
            res[f"{name}_torch_autograd_fp32_ms"] = timed(torch_fwd_bwd, warmup=1, steps=3)
        # each backward entry point alone: one read of g and X and one write of gX per cell (24 bytes)
        with torch.no_grad():
            X = eng.spectral(x, 2048, 512, w, want_stft=True)["stft"]
        G = torch.randn(X.shape, dtype=torch.complex64, generator=g).to(dev)
        cells = X.numel()
        bins_f = torch.linspace(0, sr / 2, 1025, device=dev)
        bins_t = torch.linspace(0, T / sr, X.shape[-1], device=dev)
        cut = torch.full((B,), -20.0, device=dev)
        _, ws = eng.spec_mask_low_out(X, cut, 0.5)
        _, thresh = eng.spec_gate(X, eng.spectral(nz, 2048, 512, sw, want_stft=True)["stft"], 3.0, amount,
                                  gate._rf.tolist(), gate._rt.tolist())
        kernels = {
            "band_mask_freq": (lambda: eng.spec_band_mask_out(X, bins_f, fmin, fmax, 0),
                               lambda: eng.spec_band_mask_backward(G, X, bins_f, fmin, fmax, 0)),
            "band_mask_time": (lambda: eng.spec_band_mask_out(X, bins_t, tmin, tmax, 1),
                               lambda: eng.spec_band_mask_backward(G, X, bins_t, tmin, tmax, 1)),
            "mask_low_val05": (lambda: eng.spec_mask_low_out(X, cut, 0.5),
                               lambda: eng.spec_mask_low_backward(G, X, cut, 0.5, ws)),
            "gate_apply": (None, lambda: eng.spec_gate_backward(G, X, thresh, amount, gate._rf.tolist(),
                                                                 gate._rt.tolist())),
        }
        for name, (f_out, f_bwd) in kernels.items():
            if f_out is not None:
                res[f"{name}_out_of_place_forward_ms"] = timed(f_out, steps=20)
            res[f"{name}_backward_ms"] = ms_b = timed(f_bwd, steps=20)
            res[f"{name}_backward_frac_of_hbm_peak"] = 24.0 * cells / (ms_b * 1e-3) / (peak * 1e9)
        emit({"config": "specaug_grad 64x2ch 10s@44.1k 2048/512: forward+backward of stft->mask_frequencies->"
                        "mask_timesteps->istft and of SpectralGate, their no-grad forwards, torch autograd (fp32, same "
                        "GPU) over the reference's tensor ops, and each mask backward alone",
              **res, "stft_cells": cells, "gpu": torch.cuda.get_device_name(LOCAL), "power_limit": plim})
        del x, X, G

    if "stoi" in only:  # metrics.quality.stoi on 64 x 10 s validation batches against the per-item float64 CPU loop
        import subprocess

        from audiotools_b200 import metrics
        from tests import stoi_oracle as so
        from tests.golden.make_golden_quality import speech

        try:
            plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(LOCAL)],
                                  capture_output=True, text=True, timeout=30).stdout.strip()
        except Exception:  # noqa: BLE001 (informational field)
            plim = "unknown"
        B, n_cpu = 64, 0 if args.no_cpu else 4
        for sr, C in ((16000, 1), (44100, 1), (44100, 2)):
            T = 10 * sr
            # 8 distinct speech-like clips tiled over the batch, the estimate at 5 dB SNR of white noise
            clips = np.stack([np.stack([speech(sr, T, 8 * i + c) for c in range(C)]) for i in range(8)])
            ref = torch.from_numpy(np.tile(clips, (B // 8, 1, 1)))
            est = ref + 0.3 * ref.std() * torch.randn(ref.shape, generator=torch.Generator().manual_seed(sr + C))
            e, r = AudioSignal(est, sr).to(dev), AudioSignal(ref, sr).to(dev)
            res = {}
            for mode, ext in (("std", False), ("ext", True)):
                res[f"{mode}_ms"] = timed(lambda: metrics.quality.stoi(e, r, ext), warmup=2, steps=10)
                if n_cpu:
                    est_np, ref_np = est[:n_cpu].numpy(), ref[:n_cpu].numpy()
                    want = so.batch_stoi(est_np, ref_np, sr, ext)[0]
                    res[f"{mode}_max_abs_err_vs_float64"] = float(np.abs(metrics.quality.stoi(e, r, ext)[:n_cpu].numpy()
                                                                         - want).max())
                    res[f"{mode}_cpu_float64_per_item_loop_ms"] = cpu_time(
                        lambda: so.batch_stoi(est_np, ref_np, sr, ext), reps=1) * 1e3 * B / n_cpu
            emit({"config": f"stoi {B}x{C}ch 10s@{sr}: metrics.quality.stoi (standard / extended, incl. the device->host "
                            "copy of the scores) vs the float64 restatement of pystoi looped over the items on the CPU "
                            f"(timed on {n_cpu} items, scaled to {B})", **res,
                  "gpu": torch.cuda.get_device_name(LOCAL), "power_limit": plim})
            del e, r, est, ref

    if "stoi_grad" in only:  # metrics.STOILoss: forward, forward + backward, backward alone, against its floors
        import subprocess

        from audiotools_b200 import metrics
        from audiotools_b200.engine import Engine, get_engine
        from tests import stoi_grad_cases as sg
        from tests.golden.make_golden_quality import speech

        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(LOCAL)],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        eng = get_engine()
        fp64_peak = 34.0e12  # FLOP/s: H100 SXM data sheet, FP64 (non-tensor), not measured
        B, n_t = 64, 8
        for sr, C, sec in ((16000, 1, 4), (44100, 2, 10)):
            T = sec * sr
            clips = np.stack([np.stack([speech(sr, T, 8 * i + c) for c in range(C)]) for i in range(8)])
            ref = torch.from_numpy(np.tile(clips, (B // 8, 1, 1))).to(dev)
            est = (ref + 0.3 * ref.std() * torch.randn(ref.shape, generator=torch.Generator().manual_seed(sr + C))
                   .to(dev)).contiguous()
            r = AudioSignal(ref, sr)
            up, down = Engine.stoi_ratio(sr)
            n_taps = Engine.stoi_taps(sr).size
            n10 = -(-T * up // down)
            n_fr = max(-(-(n10 - 256) // 128), 0)
            # backward floors from shapes: the transposed FIR's FP64 FMAs, and the bytes the four kernels must move
            fma = B * T * -(-n_taps // down) if up * down > 1 else 0
            nbytes = B * (4 * n10 + 2 * 4 * 15 * n_fr + 2 * 1800 * n_fr + 2 * 120 * n_fr + 2 * 1024 * n_fr
                          + 2 * 4 * n10 + 4 * C * T)
            res = {}
            for mode, ext in (("std", False), ("ext", True)):
                x = est.clone().requires_grad_()
                loss_fn = metrics.STOILoss(ext)

                def fwd():
                    with torch.no_grad():
                        return loss_fn(AudioSignal(x, sr), r)

                def fwd_bwd():
                    return torch.autograd.grad(loss_fn(AudioSignal(x, sr), r), x)

                _, _, _, ws = eng.stoi(est, ref, sr, ext, return_workspace=True)
                gs = torch.full((B,), -1.0 / B, dtype=torch.float64, device=dev)
                res[f"{mode}_fwd_ms"] = timed(fwd, warmup=3, steps=10)
                res[f"{mode}_fwd_bwd_ms"] = timed(fwd_bwd, warmup=3, steps=10)
                res[f"{mode}_bwd_ms"] = timed(lambda: eng.stoi_backward(gs, ws, est.shape, sr, ext), warmup=3, steps=10)
                # torch autograd over the float32 restatement (gather resampler, rfft, envelopes; a per-item loop, so
                # timed on the first n_t items), same GPU
                try:
                    xt = est[:n_t].clone().requires_grad_()

                    def torch_fb():
                        return torch.autograd.grad(-sg.batch_stoi(xt, ref[:n_t], sr, ext).mean(), xt)

                    res[f"{mode}_torch_autograd_fp32_{n_t}_items_ms"] = timed(torch_fb, warmup=1, steps=1)
                except torch.cuda.OutOfMemoryError:
                    res[f"{mode}_torch_autograd_fp32_{n_t}_items_ms"] = "does not fit in memory"
                del ws
                torch.cuda.empty_cache()
            emit({"config": f"stoi_grad {B}x{C}ch {sec}s@{sr}: STOILoss (standard / extended) no-grad forward, "
                            "forward + backward, backward alone (Engine.stoi_backward: 4 launches), and torch autograd "
                            f"over the float32 restatement on {n_t} of the items ({n_t}x{C}x{T})", **res,
                  "bwd_fp64_fma": fma, "bwd_fp64_floor_ms": 2 * fma / fp64_peak * 1e3, "bwd_bytes": nbytes,
                  "bwd_hbm_floor_ms": nbytes / (peak * 1e9) * 1e3, "gpu_and_power_limit": q})
            del est, ref, r

    if "specaug" in only:  # SURVEY 8f.1: SpectralTransform chain stft -> FrequencyMask -> TimeMask -> istft at cfg2's shape
        g = torch.Generator().manual_seed(0)
        B = 64
        x = (0.1 * torch.randn(B, 2, 441000, generator=g)).to(dev)
        fmin, fmax = (torch.rand(B, generator=g) * 8000).to(dev), None
        fmax = fmin + 2000.0
        tmin = (torch.rand(B, generator=g) * 9.0).to(dev)
        tmax = tmin + 0.25

        def ours():
            s = AudioSignal(x, 44100)
            s.stft(window_length=2048, hop_length=512)
            s.mask_frequencies(fmin, fmax)
            s.mask_timesteps(tmin, tmax)
            return s.istft(window_length=2048, hop_length=512)

        w = torch.hann_window(2048, periodic=True, device=dev)

        def stock_ops():  # the reference's own tensor ops (torch.stft / polar masks / torch.istft), run on the GPU
            X = torch.stft(x.reshape(-1, 441000), 2048, 512, window=w, center=True, return_complex=True)
            X = X.reshape(B, 2, 1025, -1)
            mag, ph = torch.abs(X), torch.angle(X)
            bins = torch.linspace(0, 22050, 1025, device=dev)[None, None, :, None].repeat(B, 1, 1, X.shape[-1])
            m = (fmin[:, None, None, None] <= bins) & (bins < fmax[:, None, None, None])
            X = mag.masked_fill(m, 0.0) * torch.exp(1j * ph.masked_fill(m, 0.0))
            mag, ph = torch.abs(X), torch.angle(X)
            bt = torch.linspace(0, 10.0, X.shape[-1], device=dev)[None, None, None, :].repeat(B, 1, 1025, 1)
            m = (tmin[:, None, None, None] <= bt) & (bt < tmax[:, None, None, None])
            X = mag.masked_fill(m, 0.0) * torch.exp(1j * ph.masked_fill(m, 0.0))
            return torch.istft(X.reshape(-1, 1025, X.shape[-1]), 2048, 512, window=w, center=True, length=441000)

        ms = timed(ours, warmup=2, steps=5)
        ms_stock = timed(stock_ops, warmup=1, steps=3)
        emit({"config": "specaug 64x2ch 10s@44.1k stft->mask_frequencies->mask_timesteps->istft (2048/512)",
                          "ms": ms, "ms_reference_tensor_ops_on_gpu": ms_stock, "clips_per_s": B / ms * 1e3})


if __name__ == "__main__":
    main()
    if WORLD > 1:
        import torch.distributed as dist

        dist.destroy_process_group()
