"""Accuracy table of the spectral routes against float64 (DESIGN.md "Spectral accuracy") and the split of the 7-scale
MelSpectrogramLoss gradient error by scale and by cause.  Prints JSON lines.

    python tests/probes/spectral_accuracy_probe.py          # on the H100
    python tests/probes/spectral_accuracy_probe.py --sim    # small shapes on the CPU simulator (a rehearsal)
"""
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)

SIM = "--sim" in sys.argv


def emit(**kw):
    print(json.dumps(kw), flush=True)


def main():
    import audiotools_b200.engine as em
    from audiotools_b200 import AudioSignal
    from tests import grad_cases as gc
    from tests import spectral64 as s64

    if SIM:
        from tests.cusim.sim_engine import sim_engine

        em._ENGINE = sim_engine()
        dev = "cpu"
    else:
        import __graft_entry__ as graft

        graft.build()
        dev = "cuda:0"
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True)
        emit(gpu=q.stdout.strip())
    eng = em.get_engine()

    def ours_stft(x, n, hop, w):
        return eng.spectral(x.to(dev), n, hop, w.to(dev))["stft"]

    def cufft_stft(x, n, hop, w):
        return torch.stft(x.reshape(-1, x.shape[-1]).to(dev), n, hop, window=w.to(dev), center=True,
                          pad_mode="reflect", return_complex=True).reshape(*x.shape[:-1], n // 2 + 1, -1)

    lengths = [32, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 2, 3, 400, 1001, 4095, 8191]
    if SIM:
        lengths = [32, 64, 256, 2048, 4096, 8192, 3, 400]
    g = torch.Generator().manual_seed(0)
    for n in lengths:
        rt = s64.route(n)
        hop = max(1, n // 4)
        # the DFT matrix: rectangular window, hop = n, one impulse per interior frame
        offs = np.arange(n) if (n < 8192 and not SIM) else np.sort(np.random.default_rng(n).choice(n, min(n, 64 if SIM else 1024), replace=False))
        x = s64.impulse_signal(n, offs)[None, None]
        ones = torch.ones(n)
        want = s64.impulse_spectrum(n, offs)
        o = ours_stft(x, n, n, ones)[0, 0, :, 1:1 + len(offs)]
        imp = s64.worst(o, want)
        imp_cu = s64.worst(cufft_stft(x, n, n, ones)[0, 0, :, 1:1 + len(offs)], want) if not SIM else (float("nan"),) * 2
        # noise, hann
        T = max(20 * hop + n, 4 * n)
        rows = 2 if n >= 8192 else 4
        xn = torch.randn(rows, 1, T, generator=g)
        w = AudioSignal.get_window("hann", n, "cpu")
        ref = gc.stft64(xn.double().to(dev), n, hop).cpu()
        on = ours_stft(xn, n, hop, w)
        fr, be = s64.frame_errors(on, ref)
        if not SIM:
            frc, bec = s64.frame_errors(cufft_stft(xn, n, hop, w), ref)
            cu = dict(cufft_frame_rel_mean=frc.mean().item(), cufft_frame_rel_max=frc.max().item(),
                      cufft_bin_max=bec.max().item())
        else:
            cu = {}
        u_g = s64.U * s64.growth(n, rt)
        emit(kind="fwd", n_fft=n, route=rt, impulse_bin_max=imp[1], impulse_C=imp[1] / u_g, impulse_cufft_bin_max=imp_cu[1],
             frame_rel_mean=fr.mean().item(), frame_rel_max=fr.max().item(), bin_max=be.max().item(),
             noise_C=be.max().item() / u_g, **cu)
        # inverse: consistent spectrum of the noise
        if n >= 4:
            L = xn.shape[-1]
            y = eng.istft(on, n, hop, w.to(dev), length=L).cpu()
            yd = torch.istft(on.to(torch.complex128).reshape(-1, n // 2 + 1, on.shape[-1]), n, hop,
                             window=w.double().to(on.device), center=True, length=L).cpu().reshape(y.shape)
            keep = slice(0, L - 2 * hop)
            e = s64.istft_errors(y, yd, on, w, hop, keep)
            res = dict(kind="inv", n_fft=n, ours_max=e.max().item(), ours_C=e.max().item() / u_g)
            if not SIM:
                yc = torch.istft(on.reshape(-1, n // 2 + 1, on.shape[-1]), n, hop, window=w.to(dev), center=True,
                                 length=L).cpu().reshape(y.shape)
                ec = s64.istft_errors(yc, yd, on, w, hop, keep)
                res.update(cufft_max=ec.max().item())
            emit(**res)

    # mel, one-bin and empty bands
    for n, nm, sr in [(2048, 320, 44100), (32, 5, 44100), (8192, 128, 44100), (400, 40, 44100), (512, 160, 44100)]:
        hop = n // 4
        T = 30 * hop + n
        xn = torch.randn(2, 1, T, generator=g)
        w = AudioSignal.get_window("hann", n, "cpu")
        fb, lo, hi = AudioSignal._mel_tables(sr, n, nm, 0.0, None, dev)
        m = eng.spectral(xn.to(dev), n, hop, w.to(dev), mel_fb=fb, mel_lo=lo, mel_hi=hi, want_stft=False)["mel"]
        ref = gc.stft64(xn.double().to(dev), n, hop).cpu()
        bound0, mel = s64.mel_bound(fb, ref, s64.budget(n), 0.0)
        err = (m.cpu().double() - mel).abs()
        need = ((err - bound0).clamp_min(0) / mel.clamp_min(1e-300)).max().item()
        widths = (hi - lo).cpu()
        emit(kind="mel", n_fft=n, n_mels=nm, empty_bands=int((widths <= 0).sum()),
             one_bin_bands=int((widths == 1).sum()), max_err_over_fbdelta=(err / bound0.clamp_min(1e-300)).max().item(),
             rtol_needed_u=need / s64.U)

    seven_scale(eng, dev, AudioSignal, gc, s64)


def seven_scale(eng, dev, AudioSignal, gc, s64):
    """dL/dx of the 7-scale loss per scale: ours end to end, torch FP32, and the float64 pipeline evaluated at our /
    cuFFT's complex64 STFT (isolates the forward transform); counts of L1 sign flips and clamp flips."""
    from tests.conftest import rel_err

    B, T, sr = (2, 6000, 16000) if SIM else (16, 44100, 44100)
    gen = torch.Generator().manual_seed(21)
    x = (0.5 * torch.randn(B, 1, T, generator=gen)).to(dev)
    gen = torch.Generator().manual_seed(22)
    y = (0.5 * torch.randn(B, 1, T, generator=gen)).to(dev)
    if not SIM:  # the same inputs as tests/test_gpu_grad.py::test_training_step_reference_losses
        x = (0.5 * torch.randn(16, 1, 44100, generator=torch.Generator().manual_seed(21))).to(dev)
        y = (0.5 * torch.randn(16, 1, 44100, generator=torch.Generator().manual_seed(22))).to(dev)
    P = gc.MEL_LOSS_7SCALE
    xd = x.double().requires_grad_()
    tot = {"ours": 0, "torch32": 0, "f64": 0, "at_ours_stft": 0, "at_cufft_stft": 0}
    per = []
    for nm, wl in zip(P["n_mels"], P["window_lengths"]):
        one = dict(P, n_mels=[nm], window_lengths=[wl])
        xg = x.clone().requires_grad_()
        def sig_mel(t):
            return lambda a, b, c: AudioSignal(t, sr).mel_spectrogram(a, window_length=b, hop_length=c,
                                                                      window_type="hann")

        (g_ours,) = torch.autograd.grad(gc.mel_loss(sig_mel(xg), sig_mel(y), **one), xg)
        (g64,) = torch.autograd.grad(gc.mel_loss(lambda a, b, c: gc.mel64(xd, sr, a, b, c),
                                                 lambda a, b, c: gc.mel64(y.double(), sr, a, b, c), **one), xd)
        xr = x.clone().requires_grad_()
        g32 = None
        if not SIM:
            (g32,) = torch.autograd.grad(gc.mel_loss(lambda a, b, c: gc.mel64(xr, sr, a, b, c),
                                                     lambda a, b, c: gc.mel64(y, sr, a, b, c), **one), xr)
        fb = torch.from_numpy(np.asarray(AudioSignal.get_mel_filters(sr, wl, nm), dtype=np.float64)).to(dev)
        hop = wl // 4
        w = AudioSignal.get_window("hann", wl, dev)

        def at_stft(Sx, Sy):
            """float64 loss gradient with the mel taken from given complex spectra (x's is the leaf)."""
            S = Sx.detach().to(torch.complex128).requires_grad_()
            xm = (S.abs().transpose(2, -1) @ fb.T).transpose(-1, 2)
            ym = (Sy.detach().to(torch.complex128).abs().transpose(2, -1) @ fb.T).transpose(-1, 2)
            loss = torch.nn.functional.l1_loss(xm.clamp(1e-5).log10(), ym.clamp(1e-5).log10())
            (gS,) = torch.autograd.grad(loss, S)
            xe = x.double().requires_grad_()
            (gx,) = torch.autograd.grad(gc.real_inner(gc.stft64(xe, wl, hop), gS), xe)
            return gx, xm.detach()

        S_ours_x = eng.spectral(x, wl, hop, w)["stft"]
        S_ours_y = eng.spectral(y, wl, hop, w)["stft"]
        g_at_ours, xm_ours = at_stft(S_ours_x, S_ours_y)
        X64, Y64 = gc.stft64(x.double(), wl, hop), gc.stft64(y.double(), wl, hop)
        xm64 = (X64.abs().transpose(2, -1) @ fb.T).transpose(-1, 2)
        ym64 = (Y64.abs().transpose(2, -1) @ fb.T).transpose(-1, 2)
        ym_ours = (S_ours_y.to(torch.complex128).abs().transpose(2, -1) @ fb.T).transpose(-1, 2)
        sign_flips = int(((xm_ours.clamp(1e-5).log10() > ym_ours.clamp(1e-5).log10()) !=
                          (xm64.clamp(1e-5).log10() > ym64.clamp(1e-5).log10())).sum())
        clamp_flips = int(((xm_ours > 1e-5) != (xm64 > 1e-5)).sum())
        r = dict(kind="mel7", n_mels=nm, wl=wl, ours=rel_err(g_ours.cpu(), g64.cpu()),
                 at_ours_stft=rel_err(g_at_ours.cpu(), g64.cpu()), sign_flips_ours=sign_flips,
                 clamp_flips_ours=clamp_flips, max_abs_g64=g64.abs().max().item(),
                 min_mel_rel=(xm64 / xm64.amax(dim=-2, keepdim=True).clamp_min(1e-300)).min().item())
        tot["ours"] = tot["ours"] + g_ours.double()
        tot["f64"] = tot["f64"] + g64.detach()
        tot["at_ours_stft"] = tot["at_ours_stft"] + g_at_ours
        if not SIM:
            S_cu_x = torch.stft(x.reshape(B, T), wl, hop, window=w, center=True, return_complex=True)[:, None]
            S_cu_y = torch.stft(y.reshape(B, T), wl, hop, window=w, center=True, return_complex=True)[:, None]
            g_at_cu, xm_cu = at_stft(S_cu_x, S_cu_y)
            ym_cu = (S_cu_y.to(torch.complex128).abs().transpose(2, -1) @ fb.T).transpose(-1, 2)
            r.update(torch32=rel_err(g32.cpu(), g64.cpu()), at_cufft_stft=rel_err(g_at_cu.cpu(), g64.cpu()),
                     sign_flips_cufft=int(((xm_cu.clamp(1e-5).log10() > ym_cu.clamp(1e-5).log10()) !=
                                           (xm64.clamp(1e-5).log10() > ym64.clamp(1e-5).log10())).sum()),
                     clamp_flips_cufft=int(((xm_cu > 1e-5) != (xm64 > 1e-5)).sum()))
            tot["torch32"] = tot["torch32"] + g32.double()
            tot["at_cufft_stft"] = tot["at_cufft_stft"] + g_at_cu
            # the cell that dominates: where is ours' largest deviation, relative to the float64 gradient
        per.append((nm, wl, g_ours.double() - g64))
        emit(**r)
    f64 = tot["f64"].cpu()
    emit(kind="mel7_total", **{k: rel_err(v.cpu(), f64) for k, v in tot.items() if k != "f64" and torch.is_tensor(v)})
    # which scale owns the worst element of the total error
    d = (tot["ours"] - tot["f64"]).abs()
    i = int(d.reshape(-1).argmax())
    emit(kind="mel7_worst_element", index=i, total_err=d.reshape(-1)[i].item() / f64.abs().max().item(),
         by_scale={f"{nm}/{wl}": e.reshape(-1)[i].item() / f64.abs().max().item() for nm, wl, e in per})


if __name__ == "__main__":
    main()
