"""The attention kernels' online softmax, key tile by key tile, in float64 (pure torch, CPU or GPU).

fp8_attn_emul.attention_fp8 and kernel_check.attention_ref take the FINAL row max, so they cannot follow the rounding of
a kernel that forms P against the running max of the tiles seen so far; checking a kernel against them needs a bound on
the whole softmax error, which at 5625 keys accepts errors of several percent.  This module follows the kernels:

  bf16 kernel (attention_sm90.cuh attn_fwd_kernel): per 128-key tile j, with L = fp32(log2 e),
      m' = max(m, max_j s),  sc = 2^((m - m') L),  e = 2^(s L - m' L),  P = bf16(e),
      l = l sc + sum e (the unrounded e),  o = o sc + P V_j;   O = o / l
  FP8 kernel (attention_fp8_sm90.cuh attn_fp8_kernel): the same in units of the row's q scale sq, with the tile's
  k and v scales sk_j and sv_j and the codes qc, kc_j, vc_j,
      m' = max(m, sk_j max_j (qc kc_j)),  sc = 2^((m - m') L sq),  e = 2^(qc kc_j L sq sk_j - (m' L sq - 8)),
      P~ = e4m3(e) (= e4m3(2^8 p)),  l = l sc + sum e,  o = o sc + sv_j (P~ vc_j);   O = o / l

With logits that are exact in the kernel (integer-valued q and k: see assert_exact_logits), the kernel and this
emulation form the same m and the same sc and e up to fp32 and ex2.approx rounding, and so the same P except where e
lies within that rounding of a P rounding boundary.  `online_softmax` returns O (before the output rounding) and a
per-element tolerance beta on the kernel's fp32 O:

  (a) P.  The kernel's exponent argument is rounded in fp32: m' L sq (one rounding), minus 8 (one more, or none if the
      compiler fuses it), and the fma x fk - mb (one): |d arg| <= u (|m' L sq| + |m' L sq - 8| + |arg|).  ex2.approx
      adds a relative EPS_EX2, and 2^(arg + d) = 2^arg (1 + ln 2 d (1 + 2^-20)).  So e_kernel = e (1 + d),
      |d| <= 0.7 |d arg| + EPS_EX2.  Where round(e (1 - d)) != round(e (1 + d)) the kernel's P may be either; each
      such key adds |round(e (1 + d)) - round(e (1 - d))| |v| (times the later rescales) / l.
  (b) P V.  e4m3 (FP8 kernel): each tile's partial in a fresh accumulator is off by 2^-10 of its sum |P~||codes|, the
      assumption gemm_acc_bound_fp8 states, and the fp32 o sc and fma(sv, partial, o) add 2u |o| per tile.  bf16 (bf16
      kernel): one fp32 accumulator over every key, 2u per product as gemm_acc_bound, plus u per tile for o sc.  Both
      are charged on A = sum sv_j |P||codes| with the rescales, over l.
  (c) sc, l and 1 / l.  sc multiplies o and l alike, so its error (0.7 u (2 |m L sq| + 2 |m' L sq|) + EPS_EX2 per tile,
      d_sc) only reweights earlier tiles: at most 2 sum_j d_sc A / l.  l sums the kernel's e (relative error <= max d)
      in fp32 (at most 8 adds per tile per row, a rescale per tile and two shuffles: (10 T + 4) u), 1 / l and o / l
      add 2u: |O| (max d + (10 T + 8) u).

beta = (a) + (b) + (c).  `check_output` accepts a kernel output code when it lies between the roundings of O - beta and
O + beta (a code is ambiguous when those differ), and a block scale when it lies between the scales of the row-head's
amax taken on |O| - beta and |O| + beta.
"""
from __future__ import annotations

import math

import torch

from fp8_block_emul import block_scale
from kernel_check import EPS_EX2, U32

TILE = 128
LOG2E = float(torch.tensor(math.log2(math.e), dtype=torch.float32))   # the kernels' fp32 kLog2e
F8 = torch.float8_e4m3fn
# every partial sum of S fits in the retained bits: fp32 (bf16 kernel), 13 bits of the e4m3 wgmma (gemm_acc_bound_fp8)
EXACT_BITS = {"bf16": 24, "fp8": 13}


def round_p(x: torch.Tensor, kind: str) -> torch.Tensor:
    """The kernel's rounding of e (fp32) into the P operand: bf16 or e4m3, to nearest even."""
    if kind == "bf16":
        return x.float().bfloat16().double()
    return x.float().clamp(-448.0, 448.0).to(F8).double()


def round_out(x: torch.Tensor, out: str) -> torch.Tensor:
    """The output rounding of an fp32 value: "bf16", or e4m3 ("e4m3", "e4m3_scaled": x already divided by the scale)."""
    return round_p(x, "bf16" if out == "bf16" else "fp8")


def _grain(x: torch.Tensor, dims) -> torch.Tensor:
    """The largest power of two that divides every element of x over `dims` (1 where all are zero)."""
    m, e = torch.frexp(x.double())
    mi = (m.abs() * 2.0 ** 53).long()
    low = torch.where(mi == 0, torch.full_like(mi, 1 << 62), mi & -mi)
    g = low.double() * torch.exp2(e.double() - 53)
    g = torch.where(mi == 0, torch.full_like(g, math.inf), g).amin(dim=dims)
    return torch.where(torch.isinf(g), torch.ones_like(g), g)


def assert_exact_logits(qc: torch.Tensor, kc: torch.Tensor, kind: str) -> None:
    """Every partial sum of qc kc^T is an integer multiple of (row grain x tile grain) below 2^EXACT_BITS of them, so
    the kernel's S accumulation is exact.  qc, kc [B, H, N, 64]; the bound takes each column's largest |k| in the
    tile."""
    B, H, N, _ = kc.shape
    T = (N + TILE - 1) // TILE
    pad = T * TILE - N
    kt = torch.nn.functional.pad(kc.double(), (0, 0, 0, pad)).reshape(B, H, T, TILE, 64)
    gq = _grain(qc, (-1,))                                       # [B, H, N]
    gk = _grain(kt, (-1, -2))                                    # [B, H, T]
    worst = qc.double().abs() @ kt.abs().amax(-2).transpose(-1, -2)      # [B, H, N, T] >= every |partial sum|
    units = (worst / (gq[..., None] * gk[..., None, :])).max().item()
    assert units < 2.0 ** EXACT_BITS[kind], f"logits not exact in the {kind} kernel: {units:.0f} grains"


def online_softmax(qc, sq, kc, sk, vc, sv, kv_len, kind, *, reverse=False, flip=False, final_max=False,
                   l_rounded=False, perturb=None):
    """qc, kc, vc [B, H, N, 64]: the operands the kernel multiplies (bf16 values, or e4m3 codes); sq [B, H, N] the
    rows' q scales; sk, sv [B, H, T] the key tiles' scales (all ones for the bf16 kernel); kv_len [B] valid keys.
    kind "bf16" or "fp8".  Returns (O, beta), float64 [B, H, N, 64]: O before the output rounding, beta its tolerance
    (module docstring).

    The keyword variants exist to show that the check is sharp (test_attn_online_emul.py): `reverse` sums each tile's
    keys in the opposite order, `flip` rounds P the other way wherever it is ambiguous, `final_max` forms P against
    the row's final max (no rescale: fp8_attn_emul's single-pass answer), `l_rounded` sums the rounded P into l.
    `perturb` (a torch.Generator) moves every error source of beta by its full bound, with one random sign per
    element for P (e (1 +- d) before the rounding), per (row, column) for the P V accumulation and per row for sc, l
    and the output: what a kernel at the edge of the stated error model could write."""
    fp8 = kind == "fp8"
    B, H, N, _ = qc.shape
    T = (N + TILE - 1) // TILE
    dev = qc.device
    qc, kc, vc = qc.double(), kc.double(), vc.double()
    sk, sv = sk.double().to(dev), sv.double().to(dev)
    fr = (LOG2E * sq.double().to(dev))[..., None]               # [B, H, N, 1]: exact, sq is a power of two
    bias = 8.0 if fp8 else 0.0
    valid = torch.arange(N, device=dev)[None] < kv_len.to(dev).long()[:, None]
    m = torch.full((B, H, N, 1), -math.inf, dtype=torch.float64, device=dev)
    l = torch.zeros_like(m)
    o = torch.zeros(B, H, N, 64, dtype=torch.float64, device=dev)
    A, amb = torch.zeros_like(o), torch.zeros_like(o)
    d_sc, d_e = torch.zeros_like(m), torch.zeros_like(m)
    tiles = [slice(j * TILE, min(N, (j + 1) * TILE)) for j in range(T)]
    c_tile = 2.0 ** -10 + 2 * U32 if fp8 else 2 * U32 * (TILE + 1)     # (b) per tile, of sum |P||codes|
    if perturb is not None:
        sign = lambda *shape: (torch.randint(0, 2, shape, generator=perturb) * 2 - 1).double().to(dev)
        s_acc, s_row = sign(B, H, N, 64), sign(B, H, N, 1)

    def scores(j):
        s = qc @ kc[:, :, tiles[j]].transpose(-1, -2)
        return s.masked_fill(~valid[:, None, None, tiles[j]], -math.inf)

    if final_max:
        m_fin = torch.stack([scores(j).amax(-1) * sk[:, :, j, None] for j in range(T)], -1).amax(-1, keepdim=True)
    for j in range(T):
        s = scores(j)
        m_new = m_fin if final_max else torch.maximum(m, s.amax(-1, keepdim=True) * sk[:, :, j, None, None])
        mf, mnf = m * fr, m_new * fr
        sc = torch.exp2(torch.where(torch.isinf(m), torch.full_like(m, -math.inf), mf - mnf))
        d_sc += torch.where(torch.isinf(m), torch.zeros_like(m), 0.7 * 2 * U32 * (mf.abs() + mnf.abs()) + EPS_EX2)
        arg = s * (fr * sk[:, :, j, None, None]) - (mnf - bias)
        e = torch.exp2(arg)
        e = torch.where(e < 2.0 ** -126, torch.zeros_like(e), e)     # ex2.approx.ftz
        fin = torch.isfinite(arg)
        darg = U32 * (mnf.abs() + (mnf - bias).abs() + torch.where(fin, arg.abs(), torch.zeros_like(arg)))
        d = torch.where(fin, 0.7 * darg + EPS_EX2, torch.zeros_like(arg))
        d_e = torch.maximum(d_e, d.amax(-1, keepdim=True))
        P, lo, hi = round_p(e, kind), round_p(e * (1 - d), kind), round_p(e * (1 + d), kind)
        if perturb is not None:
            P = round_p(e * (1 + sign(*e.shape) * d), kind)
            sc = sc * (1 + s_row * torch.where(torch.isinf(m), torch.zeros_like(m), 0.7 * 2 * U32 * (mf.abs() + mnf.abs())
                                                + EPS_EX2))
            e = e * (1 + s_row * d)
        if flip:
            P = torch.where(lo != hi, torch.where(P == lo, hi, lo), P)
        v = vc[:, :, tiles[j]]
        svj = sv[:, :, j, None, None]
        pv = P.flip(-1) @ v.flip(-2) if reverse else P @ v
        l = l * sc + (P if l_rounded else e).sum(-1, keepdim=True)
        if perturb is not None:
            pv = pv + s_acc * c_tile * (P.abs() @ v.abs())
        o = o * sc + svj * pv
        A = A * sc + svj * (P.abs() @ v.abs())
        amb = amb * sc + svj * ((hi - lo).abs() @ v.abs())
        m = m_new
    if perturb is not None:
        l = l * (1 + s_row * (10 * T + 4) * U32)
    O = o / l * (1 + s_row * 2 * U32) if perturb is not None else o / l
    c_acc = 2.0 ** -10 + 2 * U32 * (T + 1) if fp8 else 2 * U32 * (TILE * T + T + 1)
    beta = (amb + (c_acc + 2 * d_sc) * A) / l + O.abs() * (d_e + (10 * T + 8) * U32)
    return O, beta


def operands(qkv: torch.Tensor, B: int, N: int, H: int, kind: str, kv_len=None):
    """bf16 qkv [B N, 3 H 64] -> (qc, sq, kc, sk, vc, sv) for online_softmax: the bf16 values with unit scales, or the
    quantise pass's e4m3 codes and scales (the host rule, restated in fp8_attn_emul), with the keys at or beyond
    kv_len [B] (None: N) out of their tiles' scales."""
    import fp8_attn_emul as A
    q, k, v = [t.reshape(B, N, H, 64).permute(0, 2, 1, 3) for t in qkv.double().split(H * 64, dim=1)]
    if kind == "bf16":
        ones = torch.ones(B, H, (N + TILE - 1) // TILE, dtype=torch.float64)
        return q, torch.ones(B, H, N, dtype=torch.float64), k, ones, v, ones
    mask = None if kv_len is None else torch.arange(N)[None] < kv_len.cpu().long()[:, None]
    qc, sq = A.q_heads(q)
    kc, sk = A.q_tiles(k, mask)
    vc, sv = A.q_tiles(v, mask)
    return qc, sq[..., 0], kc, sk[:, :, ::TILE, 0], vc, sv[:, :, ::TILE, 0]


KV_LEN = {300: 201, 937: 650, 5625: 4588, 6000: 4963, 8192: 7155}   # the second utterance ends inside a key tile


def make_qkv(case: str, B: int, N: int, H: int, seed: int = 0) -> torch.Tensor:
    """bf16 qkv [B N, 3 H 64] with integer-valued q (times a power of two) and k, so the logits are exact:
      random   q, k uniform integers in [-4, 4], q / 8: logits within about +-30;
      rising / falling   k rows at round(ramp) in [-15, 15] plus integer jitter in [-1, 1], q = 1 / 16: logits ramp
               over about +-60 (the running max grows every tile, or never after the first);
      tail     q = 1 / 4, one dominant key per (utterance, head) at logit 32, every other key 9 ... 14 below it;
      tail_last  the same with the dominant key last (kv_len - 1): the running max jumps at the last tile.
    V: integers in [-7, 7]; in the upper half of the heads each key also carries a magnitude 2^-9 ... 2^6, so a tile's
    scale is set by its largest keys and the small ones are e4m3 subnormals."""
    g = torch.Generator().manual_seed(seed)
    D, R = H * 64, B * N
    ri = lambda lo, hi, shape: torch.randint(lo, hi + 1, shape, generator=g).double()
    x = torch.zeros(R, 3 * D, dtype=torch.float64)
    if case == "random":
        x[:, :D] = ri(-4, 4, (R, D)) / 8
        x[:, D:2 * D] = ri(-4, 4, (R, D))
    elif case in ("rising", "falling"):
        ramp = torch.linspace(-15, 15, N).round().double()
        ramp = ramp if case == "rising" else ramp.flip(0)
        x[:, :D] = 1 / 16
        x[:, D:2 * D] = ramp.repeat(B)[:, None] + ri(-1, 1, (R, D))
    elif case in ("tail", "tail_last"):
        x[:, :D] = 1 / 4
        twos = ri(8, 28, (R, H))                                  # k = 2 in the first `twos` columns, 1 elsewhere
        k = 1 + (torch.arange(64)[None, None] < twos[..., None]).double()
        for b in range(B):
            kv = N if b == 0 else KV_LEN.get(N, N)
            for h in range(H):
                top = kv - 1 if case == "tail_last" else int(torch.randint(0, kv, (1,), generator=g))
                k[b * N + top, h] = 2.0                           # logit 32
        x[:, D:2 * D] = k.reshape(R, D)
    else:
        raise ValueError(case)
    v = ri(-7, 7, (R, H, 64))
    v[:, H // 2:] *= torch.exp2(ri(-9, 6, (R, H - H // 2, 1)))
    x[:, 2 * D:] = v.reshape(R, D)
    qkv = x.bfloat16()
    assert torch.equal(qkv.double(), x), "inputs not exact in bf16"
    return qkv


def expected_output(O: torch.Tensor, out: str):
    """The output the kernel should write for O [B, H, N, 64]: (values in code units, scale [B, H, N]).  "bf16" and
    "e4m3" have scale 1; "e4m3_scaled" one power-of-two scale per (row, head), the block mode's rule."""
    s = block_scale(O.abs().amax(-1)).double() if out == "e4m3_scaled" else torch.ones(O.shape[:-1], dtype=torch.float64,
                                                                                         device=O.device)
    return round_out(O / s[..., None], out), s


def locate(b: int, h: int, n: int, c: int = None) -> str:
    return f"(utterance {b}, head {h}, q-tile {n // TILE}, row {n}{'' if c is None else f', col {c}'})"


def check_output(got, O, beta, out: str, scale=None, what: str = "") -> float:
    """got [B, H, N, 64]: the kernel's output in code units (bf16 values, or e4m3 codes as numbers); scale [B, H, N]
    its per-(row, head) scales for "e4m3_scaled".  Every scale and code must be one that O within beta rounds to.
    A failure names the first bad (utterance, head, q-tile, row); returns the fraction of ambiguous codes."""
    got, O, beta = got.double().cpu(), O.cpu(), beta.cpu()
    keep = torch.ones(O.shape[:-1], dtype=torch.bool)
    if out == "e4m3_scaled":
        scale = scale.double().cpu()
        s_lo = block_scale((O.abs() - beta).clamp_min(0).amax(-1)).double()
        s_hi = block_scale((O.abs() + beta).amax(-1)).double()
        bad = ~((scale >= s_lo) & (scale <= s_hi))
        if bad.any():
            b, h, n = bad.nonzero()[0].tolist()
            raise AssertionError(f"{what}: {int(bad.sum())} row scales differ; first at {locate(b, h, n)}: got "
                                 f"{scale[b, h, n].item()!r}, O within beta gives [{s_lo[b, h, n].item()!r}, "
                                 f"{s_hi[b, h, n].item()!r}]")
        keep = s_lo != s_hi
    else:
        scale = torch.ones(O.shape[:-1], dtype=torch.float64)
        keep = torch.zeros_like(keep)
    s = scale[..., None]
    lo, hi = round_out((O - beta) / s, out), round_out((O + beta) / s, out)
    bad = ~((got >= lo) & (got <= hi))
    if bad.any():
        b, h, n, c = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} codes outside the emulation's; first at {locate(b, h, n, c)}: "
                             f"got {got[b, h, n, c].item()!r}, O {O[b, h, n, c].item() / scale[b, h, n].item()!r} +- "
                             f"{beta[b, h, n, c].item() / scale[b, h, n].item():.3g} rounds to "
                             f"[{lo[b, h, n, c].item()!r}, {hi[b, h, n, c].item()!r}]")
    frac = (lo != hi).double().mean().item()
    print(f"{what}: {frac:.4%} of codes ambiguous, {keep.double().mean().item():.4%} of scales")
    return frac
