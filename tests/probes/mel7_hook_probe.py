"""The 5-mel / 32-sample term of the 7-scale loss through AudioSignal with the engine's backward calls recorded, each
compared with float64 given its recorded inputs.  ``--sim`` runs it on the CPU simulator."""
import json, os, sys
import numpy as np
import torch
REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
SIM = "--sim" in sys.argv


def main():
    import audiotools_b200.engine as em
    from audiotools_b200 import AudioSignal
    from tests import grad_cases as gc
    from tests.conftest import rel_err
    if SIM:
        from tests.cusim.sim_engine import sim_engine
        em._ENGINE = sim_engine(); dev = "cpu"
    else:
        import __graft_entry__ as graft
        graft.build(); dev = "cuda:0"
    eng = em.get_engine()
    rec = {}
    for name in ("mel_backward", "stft_backward", "spectral"):
        f = getattr(eng, name)
        def wrap(*a, _f=f, _n=name, **k):
            out = _f(*a, **k)
            rec.setdefault(_n, []).append((a, k, out))
            return out
        setattr(eng, name, wrap)
    sr = 44100
    x = (0.5 * torch.randn(16, 1, 44100, generator=torch.Generator().manual_seed(21))).to(dev)
    y = (0.5 * torch.randn(16, 1, 44100, generator=torch.Generator().manual_seed(22))).to(dev)
    for nm, wl in ((5, 32), (320, 2048)):
        rec.clear()
        one = dict(gc.MEL_LOSS_7SCALE, n_mels=[nm], window_lengths=[wl])
        def sig_mel(t):
            return lambda a, b, c: AudioSignal(t, sr).mel_spectrogram(a, window_length=b, hop_length=c, window_type="hann")
        xg = x.clone().requires_grad_()
        (g,) = torch.autograd.grad(gc.mel_loss(sig_mel(xg), sig_mel(y), **one), xg)
        xd = x.double().requires_grad_()
        (g64,) = torch.autograd.grad(gc.mel_loss(lambda a, b, c: gc.mel64(xd, sr, a, b, c),
                                                 lambda a, b, c: gc.mel64(y.double(), sr, a, b, c), **one), xd)
        print(json.dumps(dict(wl=wl, end_to_end=rel_err(g.cpu(), g64.cpu()), calls={k: len(v) for k, v in rec.items()})))
        (a, k, gS) = rec["mel_backward"][0]
        S, gm, fb, lo, hi = a[:5]
        print(json.dumps(dict(wl=wl, mel_bwd_args=[str(v) for v in a[5:]], kw={kk: str(vv) for kk, vv in k.items()},
                              gm_absmax=gm.abs().max().item(), gm_finite=bool(torch.isfinite(gm).all()))))
        d = (gm.double().transpose(2, -1) @ fb.double()).transpose(-1, 2)
        S64 = S.to(torch.complex128)
        want = d * S64 / S64.abs().clamp_min(1e-300)
        e = (gS.to(torch.complex128) - want).abs()
        i = int(e.reshape(-1).argmax())
        print(json.dumps(dict(wl=wl, mel_bwd_rel=(e.max() / want.abs().max()).item(), at=[int(v) for v in np.unravel_index(i, e.shape)],
                              got=str(gS.reshape(-1)[i].item()), want=str(want.reshape(-1)[i].item()),
                              S=str(S.reshape(-1)[i].item()))))
        (a, k, gx) = rec["stft_backward"][0]
        xe = x.double().requires_grad_()
        (gx64,) = torch.autograd.grad(gc.real_inner(gc.stft64(xe, wl, wl // 4), a[0].to(torch.complex128)), xe)
        print(json.dumps(dict(wl=wl, stft_bwd_rel=rel_err(gx.cpu(), gx64.cpu()), args=[str(v) for v in a[1:3]] + [str(v) for v in a[4:]])))
        # the incoming mel gradient against float64 arithmetic on the same forward mels
        xm = [r for r in rec["spectral"] if r[1].get("want_stft")][0][2]["mel"].double()
        ym = [r for r in rec["spectral"] if not r[1].get("want_stft")][0][2]["mel"].double()
        sg = torch.sign(xm.clamp(1e-5).log10() - ym.clamp(1e-5).log10()) * (xm >= float(np.float32(1e-5)))
        mine = sg / (xm.clamp(1e-5) * np.log(10) * xm.numel())
        dd = (gm.double() - mine).abs()
        bad = dd > 1e-3 * mine.abs().max()
        idx = bad.nonzero()[:8].tolist()
        print(json.dumps(dict(wl=wl, gmel_rel=(dd.max() / mine.abs().max()).item(), n_bad=int(bad.sum()),
                              cells=[dict(at=i, xm=xm[tuple(i)].item(), ym=ym[tuple(i)].item(), torch=gm[tuple(i)].item(),
                                          f64=mine[tuple(i)].item()) for i in idx])))
        # the forward mel the loss used against |S| fb in float64
        (a, k, out) = [r for r in rec["spectral"] if r[1].get("want_stft")][0]
        m64 = (out["stft"].to(torch.complex128).abs().transpose(2, -1) @ fb.double().T).transpose(-1, 2)
        r = (out["mel"].double() - m64).abs() / m64.clamp_min(1e-300)
        print(json.dumps(dict(wl=wl, fwd_mel_rel_max=r.max().item(), min_mel=m64.min().item())))


if __name__ == "__main__":
    main()
