"""float64 references and derived per-element bounds for the HBM-bound kernels (csrc/elementwise.cuh) and the warp-FFT
audio kernels (csrc/audio_vocos.cu, csrc/fft.cuh).  Pure torch, CPU or GPU; the comparison, tile naming and guard
buffers are kernel_check's `assert_within`, `assert_exact` and `Guarded`.

Every bound is a worst case built from the fp32 operations the kernel performs (each rounds with relative error at most
u = 2^-24; an fma contraction removes a rounding and never loosens a bound), the documented maximum errors of the CUDA
math functions (CUDA C Programming Guide, non-fast-math build: sqrtf and IEEE division 0 ulp, rsqrtf 2 ulp, expf 2 ulp,
logf 1 ulp, log1pf 1 ulp, sinf / cosf / sincosf 2 ulp, sincospif 1 ulp; an ulp is at most 2^-23 of the result, i.e. 2u)
and the output rounding.  A sum whose longest chain of dependent additions is d has error at most gam(d) sum |terms|
(Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., section 4.2), so the depth of each kernel's reduction
tree (per-lane chain + 5 warp-shuffle levels + any cross-warp step) sets its bound.
"""
from __future__ import annotations

import math

import torch

from kernel_check import U32, U_BF16, out_bound

U = U32
ULP2 = 2.0 ** -22        # 2 ulp relative (rsqrtf, expf, sinf ...)


def gam(n: int) -> float:
    """gamma_n = n u / (1 - n u): relative error of a chain of n roundings."""
    return n * U / (1 - n * U)


def rows(what: str = "row"):
    def locate(r: int, c: int) -> str:
        return f"{what} {r} col {c}"
    return locate


def frames_locate(frames: int):
    def locate(r: int, c: int) -> str:
        b, n = divmod(r, frames)
        return f"(batch {b}, frame {n}) col {c}"
    return locate


# ---------------------------------------------------------------- LayerNorm family
def ln_depth(D: int) -> int:
    """Longest addition chain of the kernels' row sums: each lane adds a float4's 4 values (3 additions) into a running
    sum over the D / 128 float4s it owns, then 5 warp-shuffle levels; the squares add one rounding."""
    return D // 128 + 8


def ln_ref_bound(x: torch.Tensor, g: torch.Tensor, h: torch.Tensor, add_one: bool, out_dtype: torch.dtype,
                 eps: float = 1e-6):
    """y = (x - mean) rsqrt(var + eps) (add_one + g) + h per row of x [R, D] (biased variance), and its bound.

    Mean: the row sum has error <= gam(d) sum|x| (d = ln_depth); times fl(1/D) (2u) the mean is off by
    e_m <= (gam(d) + 3u) mean|x|.  This is what a row with a large offset and a small spread pays, and it is why the
    kernel's two-pass variance is needed: the centred values a_i = fl(x_i - mean~) = (c_i - e)(1 + d_i) with c = x - mean
    exactly, and because sum c_i = 0, sum (c_i - e)^2 = sum c^2 + D e^2.  So the variance the kernel forms is
    (V + e^2)(1 + theta) with |theta| <= gam(d + 6) (the squares, the sum, the 1/D scale, the eps add), and its error
    relative to V + eps is zeta = (e_m^2 + (V + e_m^2) gam(d + 6) + u eps) / (V + eps).  A constant row (V = 0) has
    zeta <= e_m^2 / eps + ..., which stays small for the magnitudes tested.  rsqrtf adds 2 ulp:
    rho = zeta / (2 (1 - zeta)^1.5) + 2^-22 + u bounds the relative error of rstd.
    Output: ((a~ rstd~) (add_one + g)) + h: three products / roundings (four with the add_one rounding), so with
    K = (1 + rho)(1 + u)^k - 1 the product is within r |G| (e_m (1 + K) + |c| K) of c r G, the add of h rounds once more
    (u |y|), and the output rounding follows (out_bound; for fp32 output that add is the output rounding)."""
    x64, G = x.double(), g.double() + (1.0 if add_one else 0.0)
    D = x.shape[-1]
    mu = x64.mean(-1, keepdim=True)
    c = x64 - mu
    V = (c * c).mean(-1, keepdim=True)
    r = 1 / torch.sqrt(V + eps)
    ref = c * r * G + h.double()
    d = ln_depth(D)
    em = (gam(d) + 3 * U) * x64.abs().mean(-1, keepdim=True)
    zeta = (em * em + (V + em * em) * gam(d + 6) + U * eps) / (V + eps)
    assert zeta.max().item() < 0.25, "LayerNorm bound: the mean's rounding is not small against the spread"
    rho = zeta / (2 * (1 - zeta) ** 1.5) + ULP2 + U
    K = (1 + rho) * (1 + U) ** (4 if add_one else 3) - 1
    b = r * G.abs() * (em * (1 + K) + c.abs() * K)
    if out_dtype == torch.float32:
        return ref, out_bound(ref, b, torch.float32)
    return ref, out_bound(ref, b + U * (ref.abs() + b), out_dtype)


def ln_propagate(x: torch.Tensor, dx: torch.Tensor, g: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    """First-order effect on the affine LayerNorm output of an input error |dx| per element: dy_i/dx_j =
    G_i r (delta_ij - 1/D - c^_i c^_j / D) with c^ = (x - mean) r and mean(c^^2) <= 1, so
    |dy_i| <= r |G_i| (dx_i + mean dx + |c^_i| sqrt(mean dx^2)).  The second-order terms are below 1 % of that when
    r sqrt(mean dx^2) <= 1e-3, which is asserted; the factor 1.01 covers them and the difference between the LayerNorm
    bound evaluated at the exact and at the perturbed input."""
    x64 = x.double()
    c = x64 - x64.mean(-1, keepdim=True)
    r = 1 / torch.sqrt((c * c).mean(-1, keepdim=True) + eps)
    rms = dx.pow(2).mean(-1, keepdim=True).sqrt()
    assert (r * rms).max().item() <= 1e-3
    return 1.01 * r * g.double().abs() * (dx + dx.mean(-1, keepdim=True) + (c * r).abs() * rms)


def dwconv7_ref_bound(x: torch.Tensor, wt: torch.Tensor, wb: torch.Tensor, lw: torch.Tensor, lb: torch.Tensor):
    """Depthwise conv (k 7, zero padding 3 inside each utterance) + bias, then affine LayerNorm, for x [B, N, C]
    fp32 and tap-major weights wt [7, C].  Returns the bf16-output reference and bound as [B N, C].

    acc = bias + sum over in-range taps of x w, evaluated in tap order: each product rounds once and is followed by
    at most 7 additions, so |acc~ - acc| <= gam(8) (|bias| + sum |x| |w|).  That error passes through the LayerNorm
    (ln_propagate); the LayerNorm's own rounding is ln_ref_bound's."""
    B, N, C = x.shape
    x64, w64 = x.double(), wt.double()
    xp = torch.nn.functional.pad(x64, (0, 0, 3, 3))
    acc = wb.double().expand(B, N, C).clone()
    mag = wb.double().abs().expand(B, N, C).clone()
    for t in range(7):
        acc = acc + xp[:, t:t + N] * w64[t]
        mag = mag + (xp[:, t:t + N] * w64[t]).abs()
    acc, mag = acc.reshape(B * N, C), mag.reshape(B * N, C)
    ref, b = ln_ref_bound(acc, lw.expand(B * N, C), lb.expand(B * N, C), False, torch.bfloat16)
    return ref, b + ln_propagate(acc, gam(8) * mag, lw.expand(B * N, C))


# ---------------------------------------------------------------- GRN
def grn_ref_bound(h: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, valid_len=None):
    """GRN over the frames n < valid_len[b] of h bf16 [B, N, C]: Gx = ||h[b, :nv, c]||, Nx = Gx / (mean_c Gx + 1e-6),
    y = gamma (h Nx) + beta + h on every row (rows beyond nv are still written).  Returns reference and bound [B N, C].

    The squares of bf16 values are exact in fp32; each 32-row partial is a chain of 32 fmas and the finalize kernel adds
    the ceil(N/32) partials in order, so the sum of squares (all terms positive) is within gam(32 + nblk) relatively
    and sqrtf (correctly rounded) gives eps_gx = gam(32 + nblk) / 2 + u.  The sum over channels runs ceil(C/256)
    terms per thread, 5 shuffle levels and 8 warp partials in order: eps_tot = gam(ceil(C/256) + 13) + eps_gx; the
    division by C and the eps add 2u.  Nx = Gx / denom then has relative error eps_N = 2 eps_gx + eps_tot + 3u (first
    order; 1.01 covers the rest).  The apply evaluates gamma (h Nx) + beta + h with two products and two additions."""
    B, N, C = h.shape
    h64 = h.double()
    nv = torch.full((B,), N) if valid_len is None else valid_len.cpu().clamp(max=N)
    keep = (torch.arange(N)[None, :] < nv[:, None]).to(h.device)
    gx = (h64 * h64 * keep[..., None]).sum(1, keepdim=True).sqrt()
    nx = gx / (gx.mean(-1, keepdim=True) + 1e-6)
    g64, b64 = gamma.double(), beta.double()
    p = g64 * (h64 * nx)
    ref = p + b64 + h64
    nblk = -(-N // 32)
    e_gx = gam(32 + nblk) / 2 + U
    e_n = 1.01 * (2 * e_gx + gam(-(-C // 256) + 13) + 3 * U)
    b = 1.01 * (p.abs() * (e_n + 2 * U) + U * (p.abs() + b64.abs())) + U * (ref.abs() + h64.abs())
    return ref.reshape(B * N, C), out_bound(ref, b, torch.bfloat16).reshape(B * N, C)


# ---------------------------------------------------------------- duration head
def duration_ref_bound(x: torch.Tensor, lens: torch.Tensor, norm_w: torch.Tensor, pred_w: torch.Tensor):
    """softplus(mean_{n < L} rmsnorm(x[b, n]) . (norm_w * pred_w)), L = clamp(len, 0, N) (the mean of no frames is
    0), for x [B, N, D] fp32.  Returns reference and bound [B].

    Per frame r = rsqrtf(sum x^2 / D + 1e-5): the sum of squares (positive terms) has relative error
    gam(D/128 + 9), the scale and the eps add 2u more, so r is within rho = gam(D/128 + 11) / (2 (1 - ..)^1.5) + 2^-22.
    The x r products (u) are summed per channel over each warp's ceil(L/8) frames and then over the 8 warps
    (gam(ceil(L/8) + 8)); the products with 1/L, norm_w and pred_w round 4 times and the channel sum has depth
    D/256 + 13.  So |t~ - t| <= sum_c P_c ((1 + rho + u)(1 + gam(ceil(L/8) + 8))(1 + 4u)(1 + gam(D/256 + 14)) - 1),
    with P_c = sum_n |x r| |norm_w pred_w| / L.  Softplus: log1pf(expf(t)) moves by at most bt sigmoid(t + bt)
    (its slope), expf's 2 ulp add 4u sigmoid, log1pf's 1 ulp adds 2u |y|; above 20 the kernel returns t, which is
    within exp(-t) of softplus(t); below about -103 expf underflows to 0, an absolute error under 2^-148.
    Also returns t."""
    B, N, D = x.shape
    x64 = x.double()
    L = lens.cpu().long().clamp(0, N)
    r = 1 / torch.sqrt((x64 * x64).mean(-1, keepdim=True) + 1e-5)
    keep = (torch.arange(N)[None, :] < L[:, None]).to(x.device)[..., None]
    xr = x64 * r * keep
    denom = L.clamp(min=1).double().to(x.device)[:, None]
    v = norm_w.double() * pred_w.double()
    t = (xr.sum(1) / denom * v).sum(-1)
    P = ((xr.abs().sum(1) / denom) * v.abs()).sum(-1)
    rho = gam(D // 128 + 11) / (2 * (1 - gam(D // 128 + 11)) ** 1.5) + ULP2
    chain = torch.tensor([gam(-(-int(l) // 8) + 8) for l in L], dtype=torch.float64, device=x.device)
    bt = P * ((1 + rho + U) * (1 + chain) * (1 + 4 * U) * (1 + gam(D // 256 + 14)) - 1)
    ref = torch.nn.functional.softplus(t)
    sig = torch.sigmoid(t + bt)
    b = bt * sig + 4 * U * sig + 2 * U * ref.abs() + torch.where(t + bt > 20, torch.exp(-(t - bt)), torch.zeros_like(t))
    return ref, b + 2.0 ** -148, t


# ---------------------------------------------------------------- timestep MLP
def time_mlp_ref_bound(t: torch.Tensor, w0, b0, w2, b2):
    """TimestepEmbedding for times t [T]: e_i = 1000 t exp(-i ln(1e4) / 127), h0 = [sin e | cos e],
    h1 = silu(W0 h0 + b0), t_emb = W2 h1 + b2; also silu(t_emb) (the kernel's bf16 output).  Returns
    (t_emb, bound, silu, bound) as [T, D].

    Argument: the constant fl(fl(ln 1e4) / 127) and the product with i round 3 times, so the exponent is within
    3u 9.22 absolutely and expf adds 2 ulp: f is within 32u relatively; e = fl(fl(1000 t) f) within
    eps_e = 35u (1.01 covers the products of errors).  sinf / cosf move by at most |de| and add 2 ulp (2^-22 |value|).
    Layer 1: each lane chains 8 fmas, then 5 shuffle levels (gam(13) sum |w0||h0|), plus |w0| . bound(h0) and the
    bias add (u).  silu_f(z) = z / (1 + expf(-z)): expf 2 ulp, the add and the division make it relatively 6u, and
    |silu'| <= 1.1 carries the input error.  Layer 2: chains of D/32 fmas and 5 levels (gam(D/32 + 5)); the bias add
    is the fp32 output rounding.  The bf16 output is silu of that, rounded."""
    T, D = t.shape[0], w2.shape[0]
    t64 = t.double()[:, None]
    i = torch.arange(128, dtype=torch.float64, device=t.device)
    e = 1000 * t64 * torch.exp(-i * math.log(1e4) / 127)
    h0 = torch.cat([torch.sin(e), torch.cos(e)], -1)
    de = 1.01 * 35 * U * e.abs()
    bh0 = torch.cat([de + ULP2 * torch.sin(e).abs(), de + ULP2 * torch.cos(e).abs()], -1)
    W0, W2 = w0.double(), w2.double()
    z = h0 @ W0.T + b0.double()
    bz = bh0 @ W0.abs().T + gam(13) * (h0.abs() @ W0.abs().T) + U * (z.abs() + b0.double().abs())
    silu = torch.nn.functional.silu
    h1 = silu(z)
    bh1 = 1.1 * bz + 6 * U * h1.abs()
    v = h1 @ W2.T + b2.double()
    bv = bh1 @ W2.abs().T + gam(D // 32 + 5) * (h1.abs() @ W2.abs().T)
    bv = bv + U * (v.abs() + bv)
    s = silu(v)
    bs = 1.1 * bv + 6 * U * s.abs()
    return v, bv, s, out_bound(s, bs, torch.bfloat16)


# ---------------------------------------------------------------- ODE stage update
def ode_k(v: torch.Tensor, rows: int, d: int, null_off: int, cfg: float):
    """k = pred + (pred - null) cfg (float64) and its bound: the difference, the product and the add round once each,
    |dk| <= u (2 |pred - null| |cfg| + |k|)."""
    v64 = v.double()
    pred = v64[:rows, :d]
    if null_off <= 0:
        return pred, torch.zeros_like(pred)
    nu = v64[null_off:null_off + rows, :d]
    k = pred + (pred - nu) * cfg
    return k, U * (2 * (pred - nu).abs() * abs(cfg) + k.abs())


def ode_axpy_bound(base: torch.Tensor, a: float, upd: torch.Tensor, bupd: torch.Tensor) -> torch.Tensor:
    """y = base + a upd with upd known within bupd: |a| bupd, the product's and the add's rounding."""
    y = base.double() + a * upd
    return abs(a) * bupd + U * abs(a) * upd.abs() + U * (y.abs() + abs(a) * bupd)


# ---------------------------------------------------------------- warp FFT, mel, iSTFT
TW_ERR = 2 * math.pi * U + math.sqrt(2) * 2 * U   # twiddle(): sincospif 1 ulp each + the rounded argument (2 pi u)


def fft512_rel() -> float:
    """Relative L2 error of fft512_warp: ||Z~ - Z||_2 <= fft512_rel() ||Z||_2 = fft512_rel() sqrt(512) ||z||_2.

    Each of the 9 butterfly stages (4 in fft16, 5 across lanes) and the twiddle multiply between them is a
    complex operation with error at most eta = mu + gam(4)(sqrt 2 + mu) of its input (Higham, Accuracy and Stability,
    Thm 24.2), mu the twiddle error (fft16's rounded constants: sqrt(2) u; the lane stages' twiddle(): TW_ERR).  Ten
    such stages give (1 + eta)^10 - 1."""
    eta = TW_ERR + gam(4) * (math.sqrt(2) + TW_ERR)
    return (1 + eta) ** 10 - 1


def mel_ref_bound(audio: torch.Tensor, window: torch.Tensor, filt_t: torch.Tensor, hop: int, frames: int):
    """log(max(|rfft(frame * window)| @ filt_t, 1e-5)) per frame f = samples [f hop - 512, f hop + 512) of the
    zero-padded signal, audio [B, T].  Returns reference and bound as [B frames, n_mels].

    The windowed input rounds once (u |z|).  The 512-point FFT of z = x_even + i x_odd is within
    E = ((1 + fft512_rel())(1 + u) - 1) sqrt(512) ||z||_2 in every bin (a bin's error is at most the L2 norm of the
    error vector).  The split step X_k = (Z_k + Z*_{512-k})/2 - i W^k (Z_k - Z*_{512-k})/2 takes two bins' errors,
    so 2E, plus its own rounding (TW_ERR + 6u)(|Z_k| + |Z_{512-k}|); the magnitude sqrtf(re^2 + im^2) adds 3u |X_k|.
    The filterbank dot product is a chain of 513 fmas: sum_k |f_km| bound_k + gam(513) sum_k |X_k| |f_km|.  The log of
    max(v, 1e-5) is (1 / max(v - beta, 1e-5))-Lipschitz on [v - beta, v + beta], and logf adds 1 ulp (2u |log v|)."""
    B, T = audio.shape
    x = audio.double()
    w = window.double()
    idx = torch.arange(frames, device=audio.device)[:, None] * hop - 512 + torch.arange(1024, device=audio.device)
    ok = (idx >= 0) & (idx < T)
    fr = torch.where(ok, x[:, idx.clamp(0, T - 1)], torch.zeros((), dtype=torch.float64, device=audio.device)) * w
    fr = fr.reshape(B * frames, 1024)
    X = torch.fft.rfft(fr, dim=-1)
    Z = torch.fft.fft(torch.complex(fr[:, 0::2], fr[:, 1::2]), dim=-1)
    zn = fr.pow(2).sum(-1, keepdim=True).sqrt()
    E = ((1 + fft512_rel()) * (1 + U) - 1) * math.sqrt(512) * zn
    k = torch.arange(513, device=audio.device)
    za = Z.abs()
    bm = 2 * E + (TW_ERR + 6 * U) * (za[:, k % 512] + za[:, (512 - k) % 512]) + 3 * U * X.abs()
    F = filt_t.double()
    mel = X.abs() @ F
    bmel = bm @ F.abs() + gam(513) * (X.abs() @ F.abs())
    ref = torch.log(mel.clamp(min=1e-5))
    b = bmel / (mel - bmel).clamp(min=1e-5) + 2 * U * ref.abs()
    return ref, b


def istft_frames_ref_bound(h: torch.Tensor, window: torch.Tensor):
    """Per frame: S_k = min(exp(logmag_k), 100) e^{i phase_k}, windowed irfft(S, 1024) (the imaginary parts of S_0
    and S_512 ignored), for h [rows, >= 1026].  Returns (frames, bound) [rows, 1024] before the overlap-add.

    expf (2 ulp), sincosf (2 ulp each) and the two products put S_k within |S_k| (4u + 2 2^-22 + 2u) = 12u |S_k|
    (min(., 100) is 1-Lipschitz).  The inverse split step takes two bins (2 max), rounds with
    (TW_ERR + 6u)(|S_k| + |S_{512-k}|), and the FFT of that input is within sqrt(512) (||dA||_2 + fft512_rel() ||A||_2)
    in L2, so every output sample is within that / 512 before the window; the 1/512 scale is exact and the window
    product rounds once."""
    rows = h.shape[0]
    lm, ph = h[:, :513].double(), h[:, 513:1026].double()
    mag = torch.exp(lm).clamp(max=100)
    S = torch.polar(mag, ph)
    x = torch.fft.irfft(S, 1024, dim=-1) * window.double()
    k = torch.arange(512, device=h.device)
    A_abs = mag[:, k] + mag[:, 512 - k]
    dA = 2 * 12 * U * torch.maximum(mag[:, k], mag[:, 512 - k]) + (TW_ERR + 6 * U) * A_abs
    A_l2 = A_abs.pow(2).sum(-1, keepdim=True).sqrt()
    dA_l2 = dA.pow(2).sum(-1, keepdim=True).sqrt()
    e = math.sqrt(512) * (dA_l2 + fft512_rel() * A_l2) / 512
    b = e * window.double().abs() + U * x.abs()
    return x.reshape(rows, 1024), b.reshape(rows, 1024)


def istft_ola_ref_bound(frames: torch.Tensor, bframes: torch.Tensor, window: torch.Tensor, B: int, n_frames: int,
                        hop: int, norm_sq: bool, trim: int, out_len: int):
    """Overlap-add of the windowed frames [B n_frames, 1024] divided by the window envelope (sum of w or w^2 over the
    frames covering the sample; no division where it is <= 1e-11), dropping `trim` leading samples.  Returns
    (out, bound) [B, out_len].  The at most 4 frame values add in order (3u of their magnitudes), the envelope's
    positive terms round within gam(5) (w^2 adds the square's rounding), and the division rounds once; 1 / env is
    what makes the bound grow at the signal's edges."""
    dev = frames.device
    fr = frames.double().reshape(B, n_frames, 1024)
    bf = bframes.double().reshape(B, n_frames, 1024)
    L = (n_frames - 1) * hop + 1024
    acc = torch.zeros(B, L, dtype=torch.float64, device=dev)
    mag = torch.zeros_like(acc)
    err = torch.zeros_like(acc)
    env = torch.zeros(L, dtype=torch.float64, device=dev)
    w = window.double()
    for f in range(n_frames):
        acc[:, f * hop:f * hop + 1024] += fr[:, f]
        mag[:, f * hop:f * hop + 1024] += fr[:, f].abs()
        err[:, f * hop:f * hop + 1024] += bf[:, f]
        env[f * hop:f * hop + 1024] += w * w if norm_sq else w
    sl = slice(trim, trim + out_len)
    acc, mag, err, env = acc[:, sl], mag[:, sl], err[:, sl], env[sl]
    assert acc.shape[1] == out_len
    div = env > 1e-11
    envd = torch.where(div, env, torch.ones_like(env))
    out = acc / envd
    b = (err + 3 * U * mag) / envd + out.abs() * (gam(5) + U)
    b = b + U * (out.abs() + b)
    return out, b + 1e-30
