"""Float64 oracles and error models for the effect kernels of csrc/effects.cu (order statistics, ``alter_drr``,
quantisation, the peak-scale backward), the MFCC basis product of csrc/dft.cu and the gather of csrc/collate.cu.
Each oracle restates the reference's definition (ref:audiotools/core/effects.py, audio_signal.py), not the kernel.

Error models (u = 2^-24), each constant set once from the H100 measurement with about 2x headroom (DESIGN.md
"Effect kernel accuracy"):
  order statistics, pack_rows   exact (values; -0 == +0)
  quantile                      bit for bit with torch.quantile at integer ranks; else |err| <= C_Q u (|a| + |b|)
  alter_drr                     per sample |err| <= C_DRR u (2 eps_alpha + 4) |y|, eps_alpha = sqrt(n) kappa (or 4 when
                                alpha sits clearly on the min_alpha floor), kappa = (E_out + P L) / |c| + 1
  peak-scale backward           |err| <= C_PS u (|S g| + [at the arg-max] S sqrt(T) sum|g y| / My)
  mfcc DCT                      |err| / sum_m |v_m d_mj| <= C_DCT u sqrt(n_mels)   (gamma_n is the hard ceiling)
"""
import numpy as np
import torch

U = 2.0 ** -24
F32_1E8 = float(np.float32(1e-8))  # the reference clamps a float32 tensor: its 1e-8 is this float

C_Q = 0.6
C_DRR = 0.35
C_PS = 4.0
C_DCT = 2.5


# --------------------------------------------------------------------------- order statistics and quantile
def order_stats(row, ks):
    """The ks-th smallest values of ``row`` (float32 values, float64 arithmetic): a stable sort with every NaN last,
    as torch.sort; ks clamped to [0, n-1] as the kernel documents."""
    r = np.sort(np.asarray(row, dtype=np.float64), kind="stable")  # numpy sorts NaN of either sign to the end
    k = np.clip(np.asarray(ks, dtype=np.int64), 0, r.size - 1)
    return r[k]


def quantile(row, q):
    """torch.quantile(row, q) for a 1-D float32 row (linear interpolation), by aten's rules: float32 ranks q (n - 1),
    floor and ceil, the two-sided lerp (here in float64), and NaN for every q when the row holds a NaN.
    Returns (values, a, b, integer_rank) so callers can pick the budget."""
    row = np.asarray(row, dtype=np.float32)
    q = np.asarray(q, dtype=np.float32).reshape(-1)
    ranks = q * np.float32(row.size - 1)
    lo, hi = np.floor(ranks), np.ceil(ranks)
    w = (ranks - lo).astype(np.float64)
    a, b = order_stats(row, lo.astype(np.int64)), order_stats(row, hi.astype(np.int64))
    v = np.where(w < 0.5, a + w * (b - a), b - (b - a) * (1 - w))
    if np.isnan(row).any():
        v = np.full_like(v, np.nan)
    return v, a, b, lo == hi


def same_values(got, want):
    """Exact equality of values: NaN matches NaN, -0 matches +0."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    return got.shape == want.shape and bool(np.array_equal(got, want, equal_nan=True))


# --------------------------------------------------------------------------- alter_drr
def alter_drr(ir, sample_rate, drr):
    """ImpulseResponseMixin.alter_drr in float64 for ir [B, C, T] (float32 values) and drr [B]: decompose_ir (window =
    the early region of channel 0: scipy's hann(1) == 1), solve_alpha, the min_alpha floor, ensure_max_of_audio.
    Returns the output and, per row, what the error model needs."""
    x = torch.as_tensor(ir).double()
    B, C, T = x.shape
    d = torch.as_tensor(drr).double().reshape(-1).expand(B).reshape(B, 1)
    td = x.argmax(dim=-1, keepdim=True)  # NaN is the largest, first index on ties
    t0 = int(sample_rate * 0.0025)
    idx = torch.arange(T)[None, None, :]
    early_idx = (idx >= td - t0) & (idx <= td + t0)
    zero = torch.zeros_like(x)
    early, late = torch.where(early_idx, x, zero), torch.where(early_idx, zero, x)
    wd = early_idx[:, :1].double().expand_as(x)
    e_sq = early ** 2
    a = (wd ** 2 * e_sq).sum(-1)
    b = (2 * (1 - wd) * wd * e_sq).sum(-1)
    p = torch.pow(10.0, d / 10)
    e_out = ((1 - wd) ** 2 * e_sq).sum(-1)
    l_sq = (late ** 2).sum(-1)
    c = e_out - p * l_sq
    expr = (b ** 2 - 4 * a * c).sqrt()
    raw = torch.maximum((-b - expr) / (2 * a), (-b + expr) / (2 * a))
    min_alpha = late.abs().max(dim=-1)[0] / early.abs().max(dim=-1)[0]
    alpha = torch.maximum(raw, min_alpha)
    y = alpha[..., None] * wd * early + (1 - wd) * early + late
    peak = y.abs().max(dim=-1, keepdim=True)[0]
    gain = torch.ones_like(peak)
    gain[peak > 1.0] = 1.0 / peak[peak > 1.0]
    y = y * gain
    kappa = (e_out + p * l_sq) / c.abs() + 1
    floored = raw < min_alpha * (1 - 1e-3)
    eps_alpha = torch.where(floored, torch.full_like(kappa, 4.0), np.sqrt(T) * kappa)
    return y, {"alpha": alpha, "raw": raw, "min_alpha": min_alpha, "eps_alpha": eps_alpha, "c": c}


def alter_drr_err(got, ir, sample_rate, drr):
    """(worst |err| / (u (2 eps_alpha + 4) |y|) over finite samples, NaN pattern mismatches)."""
    want, info = alter_drr(ir, sample_rate, drr)
    got = torch.as_tensor(got).double()
    nan_w, nan_g = want.isnan(), got.isnan()
    mism = int((nan_w != nan_g).sum())
    scale = U * (2 * info["eps_alpha"][..., None] + 4) * want.abs()
    diff = (got - want).abs()
    ok = ~nan_w & ~nan_g
    exact = ok & (diff == 0)
    ratio = torch.where(ok & ~exact, diff / scale.clamp_min(1e-300), torch.zeros_like(diff))
    return float(ratio.max()) if ratio.numel() else 0.0, mism


# --------------------------------------------------------------------------- quantisation
def mulaw_ref(x, q):
    """The reference's mulaw_quantization, its own float32 torch expressions (on x's device); q [B] or a number."""
    mu = torch.as_tensor(q, dtype=torch.float32, device=x.device).reshape(-1, 1, 1) - 1.0
    y = torch.sign(x) * torch.log1p(mu * torch.abs(x)) / torch.log1p(mu)
    y = ((y + 1) / 2 * mu + 0.5).to(torch.int64)
    y = (y / mu) * 2 - 1.0
    y = torch.sign(y) * (torch.exp(torch.abs(y) * torch.log1p(mu)) - 1.0) / mu
    return x - (x - y)


def linear_ref(x, q):
    """The reference's quantization, float32 torch expressions."""
    qc = torch.as_tensor(q, dtype=torch.float32, device=x.device).reshape(-1, 1, 1)
    y = (x + 1) / 2
    y = (y * qc).floor() / qc
    y = 2 * y - 1
    return x - (x - y)


def mulaw_level64(x, q):
    """The mu-law level before truncation, in float64: (sign(x) log1p(mu |x|) / log1p(mu) + 1) / 2 mu + 0.5."""
    x = np.asarray(x, dtype=np.float64)
    mu = np.asarray(q, dtype=np.float64).reshape(-1, 1, 1) - 1.0
    with np.errstate(all="ignore"):
        return (np.sign(x) * np.log1p(mu * np.abs(x)) / np.log1p(mu) + 1) / 2 * mu + 0.5


def mulaw_boundaries(q):
    """float32 inputs at every mu-law level boundary of q levels and one and two floats to either side."""
    mu = q - 1.0
    k = np.arange(1, q, dtype=np.float64)  # the level switches from k - 1 to k where the pre-truncation value is k
    v = (k - 0.5) / mu * 2 - 1
    xb = np.sign(v) * np.expm1(np.abs(v) * np.log1p(mu)) / mu
    xb = xb.astype(np.float32)
    pts = [xb]
    for s in (1, 2):
        up, dn = xb.copy(), xb.copy()
        for _ in range(s):
            up, dn = np.nextafter(up, np.float32(np.inf)), np.nextafter(dn, np.float32(-np.inf))
        pts += [up, dn]
    return np.concatenate(pts)


def linear_boundaries(q):
    """float32 inputs at every linear level boundary (x + 1) / 2 q = k, and one float to either side."""
    xb = (2 * np.arange(0, q + 1, dtype=np.float64) / q - 1).astype(np.float32)
    return np.concatenate([xb, np.nextafter(xb, np.float32(np.inf)), np.nextafter(xb, np.float32(-np.inf))])


# --------------------------------------------------------------------------- peak-scale backward
def peak_scale_backward(g, y, x_ref=None, max_abs=1.0, bypass=None):
    """torch.autograd in float64 over the reference's expressions: ensure_max_of_audio (x_ref None) or apply_ir's
    restore y * clamp(max|x_ref|, 1e-8) / clamp(max|y|, 1e-8); max(dim) gives the first index on ties and the
    gradient of |.| is sign(.) (0 at 0).  Returns (gy, gx, S, My, b, sum|g y|) per row."""
    y = torch.as_tensor(y).double().clone().requires_grad_(True)
    g = torch.as_tensor(g).double()
    My, b = y.detach().abs().max(dim=-1, keepdim=True)
    if x_ref is None:
        peak = y.abs().max(dim=-1, keepdim=True)[0]
        gain = torch.ones_like(peak)
        m = peak > max_abs
        gain[m] = max_abs / peak[m]
        (y * gain).backward(g)
        return y.grad, None, gain.detach(), My, b, (g * y.detach()).abs().sum(-1, keepdim=True)
    x = torch.as_tensor(x_ref).double().clone().requires_grad_(True)
    scale = x.abs().max(dim=-1, keepdim=True)[0].clamp(F32_1E8) / y.abs().max(dim=-1, keepdim=True)[0].clamp(F32_1E8)
    if bypass is not None:
        byp = torch.as_tensor(bypass).bool().reshape(-1, *([1] * (y.ndim - 1)))
        scale = torch.where(byp, torch.ones_like(scale), scale)
    (y * scale).backward(g)
    return y.grad, x.grad, scale.detach(), My, b, (g * y.detach()).abs().sum(-1, keepdim=True)


def peak_scale_err(gy, gx, g, y, x_ref=None, max_abs=1.0, bypass=None):
    """(worst ratio |err| / budget of gy and gx, NaN pattern mismatches), budget as in the module docstring."""
    wy, wx, S, My, b, sgy = peak_scale_backward(g, y, x_ref, max_abs, bypass)
    T = wy.shape[-1]
    g64 = torch.as_tensor(g).double()
    at_b = torch.zeros_like(wy, dtype=torch.bool).scatter_(-1, b, True)
    corr = S.abs() * np.sqrt(T) * sgy / My.clamp_min(F32_1E8)
    by = U * ((S * g64).abs() + at_b * corr)
    worst, mism = 0.0, 0
    pairs = [(torch.as_tensor(gy).double(), wy, by)]
    if wx is not None:
        bx = U * np.sqrt(T) * sgy / My.clamp_min(F32_1E8) * torch.ones_like(wx)
        pairs.append((torch.as_tensor(gx).double(), wx, bx))
    for got, want, bud in pairs:
        nan_w, nan_g = want.isnan(), got.isnan()
        mism += int((nan_w != nan_g).sum())
        ok = ~nan_w & ~nan_g
        diff = (got - want).abs()
        r = torch.where(ok & (diff > 0), diff / bud.clamp_min(1e-300), torch.zeros_like(diff))
        worst = max(worst, float(r.max()))
    return worst, mism


# --------------------------------------------------------------------------- mfcc DCT, pack_rows
def mel_dct(logmel, dct):
    """out[..., j, n] = sum_m dct[m, j] logmel[..., m, n] in float64, and the per-element scale sum_m |v_m d_mj|."""
    v = torch.as_tensor(logmel).double()
    d = torch.as_tensor(dct).double()
    return torch.einsum("...mn,mj->...jn", v, d), torch.einsum("...mn,mj->...jn", v.abs(), d.abs())


def mel_dct_err(got, logmel, dct):
    want, scale = mel_dct(logmel, dct)
    n = torch.as_tensor(dct).shape[0]
    diff = (torch.as_tensor(got).double() - want).abs()
    r = torch.where(diff > 0, diff / (U * np.sqrt(n) * scale).clamp_min(1e-300), torch.zeros_like(diff))
    return float(r.max())


def pack_rows(rows, offsets, T_out):
    """rows: per item a float32 [C, len] array; out[i, c, t] = rows[i][c, t + off_i] where that index is in
    [0, len), else 0."""
    C = rows[0].shape[0]
    out = np.zeros((len(rows), C, T_out), dtype=np.float32)
    t = np.arange(T_out)
    for i, (r, off) in enumerate(zip(rows, offsets)):
        u = t + off
        ok = (u >= 0) & (u < r.shape[1])
        out[i][:, ok] = r[:, u[ok]]
    return out
