"""Element-wise checkers for the GEMM and attention kernels (pure torch, CPU or GPU).

* `assert_exact`: bitwise comparison; a mismatch names the first bad (tile, row, column).
* `assert_within`: |got - ref| <= bound for every element; returns the worst err/bound ratio and names the tile where
  it occurs.  The bound helpers below derive per-element bounds from the operation (see their docstrings).
* `Guarded`: an output view inside a larger buffer pre-filled with a NaN pattern (rows above and below, columns left and
  right, so ld > n); `check()` asserts that every element of the view was written and every guard element is unchanged.

Tiles are named by a `locate(row, col)` function: `gemm_tiles` for the GEMM's 128 x BN output tiles (flat or batched
rows), `attn_tiles` for the attention's (batch, head, 128-query tile).
"""
from __future__ import annotations

import math

import torch

U32 = 2.0 ** -24          # unit roundoff of fp32 (round to nearest)
U_BF16 = 2.0 ** -8        # unit roundoff of bf16 (8 significant bits)
U_E4M3 = 2.0 ** -4        # unit roundoff of e4m3 (4 significant bits)
E4M3_SUB = 2.0 ** -10     # half the e4m3 subnormal spacing (2^-9): absolute rounding error below 2^-6
# documented maximum errors of the approximate instructions the epilogues use (PTX ISA / CUDA C Programming Guide)
EPS_TANH = 2.0 ** -10.987  # tanh.approx.f32: maximum relative error
EPS_EX2 = 2.0 ** -22       # ex2.approx.ftz.f32: maximum relative error (2 ulp)

_INT = {4: torch.int32, 2: torch.int16, 1: torch.uint8}
PATTERN = {4: 0x7FA5A5A5, 2: 0x7FA5, 1: 0x7F}   # NaN in fp32 / bf16 / e4m3 (e4m3 0x7F is its only positive NaN)


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.view(_INT[t.element_size()])


def e4m3(x: torch.Tensor) -> torch.Tensor:
    """Round to nearest even e4m3, saturating at +-448: the kernels' cvt.rn.satfinite."""
    return x.float().clamp(-448, 448).to(torch.float8_e4m3fn)


def round_to(ref: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """Round-to-nearest of an fp32-exact float64 reference into the output type."""
    r32 = ref.float()
    assert torch.equal(r32.double(), ref.double()), "reference is not exact in fp32"
    if dtype == torch.float32:
        return r32
    if dtype in (torch.uint8, torch.float8_e4m3fn):
        return e4m3(r32).view(dtype)
    return r32.to(dtype)


def instantiation(*, act: int = 0, out_dtype=torch.bfloat16, rope: bool = False, fp8: bool = False,
                  resid: bool = False, tile: int, conv_grouped: bool = False, scaled: bool = False) -> tuple:
    """(ACT, OUT_BF16, ROPE, FP8, RESID, BN) of the gemm_bf16_tn_kernel a launch selects.  dispatch_epi (gemm.cu): FP8
    when any operand or output is e4m3, RESID = false only for the residual-free GELU-tanh bf16 epilogue.
    dispatch_scaled (`scaled`: any block scale is set): always FP8, and its bf16-output forms (the RoPE QKV, FF1) carry
    no residual.  The grouped convolution always runs 64-column tiles.  The SCALED template flag is `scaled` itself:
    a scaled and an unscaled launch may share the other five flags and still run different kernels."""
    out_bf16 = out_dtype != torch.float32
    if scaled:
        return (act, out_bf16, rope, True, not out_bf16, 64 if conv_grouped else tile)
    no_resid = not resid and act == 1 and out_bf16 and not rope
    return (act, out_bf16, rope, fp8, not no_resid, 64 if conv_grouped else tile)


# ---------------------------------------------------------------- launch geometry (gemm.cu f5_gemm_bf16)
STAGES = {64: 6, 128: 4}     # ring depth of the 64- and 128-wide instantiations (dispatch_* <BN, kStages>)


def cdiv(a: int, b: int) -> int:
    return -(-a // b)


def gemm_bn(n: int, m: int, *, tile_n: int = 0, rows_per_batch: int = 0, num_batches: int = 1, batched: bool = False,
            conv_grouped: bool = False, sms: int) -> int:
    """The launcher's tile width: tile_n when given, 64 for the grouped convolution, else 128 unless that leaves most
    of the SMs idle (fewer than 13/16 of them get a tile) or n <= 64."""
    if conv_grouped:
        return 64
    if tile_n:
        return tile_n
    rpb = rows_per_batch or m
    mt = num_batches * cdiv(rpb, 128) if batched else cdiv(m, 128)
    if n <= 64:
        return 64
    return 128 if mt * cdiv(n, 128) >= (sms * 13) // 16 else 64


def gemm_tile_count(n: int, m: int, bn: int, *, rows_per_batch: int = 0, num_batches: int = 1,
                    batched: bool = False) -> int:
    """Output tiles of a launch: 128-row tiles over the flat rows, or over each utterance when tiles never straddle
    utterances (batched / conv mode), times the column tiles.  The persistent grid is min(tiles, SMs) CTAs."""
    rpb = rows_per_batch or m
    return cdiv(n, bn) * (num_batches * cdiv(rpb, 128) if batched else cdiv(m, 128))


def gemm_num_kb(k: int, *, conv_taps: int = 1, ab8: bool = False) -> int:
    """k-blocks per tile (128 bytes of every row: 64 bf16 or 128 e4m3 elements, per tap)."""
    return conv_taps * cdiv(k, 128 if ab8 else 64)


# ---------------------------------------------------------------- tile naming
def gemm_tiles(bn: int, rows_per_batch: int = 0, batched: bool = False):
    """(row, col) -> tile name.  Batched mode: tiles never straddle utterances (tile = (utterance, tile in utterance))."""
    def locate(row: int, col: int) -> str:
        if batched:
            b, r = divmod(row, rows_per_batch)
            return f"tile (utt {b}, m {r // 128}, n {col // bn}) row {row} col {col}"
        return f"tile (m {row // 128}, n {col // bn}) row {row} col {col}"
    return locate


def attn_tiles(frames: int, head_dim: int = 64):
    def locate(row: int, col: int) -> str:
        b, n = divmod(row, frames)
        return f"(batch {b}, head {col // head_dim}, q-tile {n // 128}) row {row} col {col}"
    return locate


def _first(mask: torch.Tensor):
    idx = mask.nonzero()[0].tolist()
    return idx[0], (idx[1] if len(idx) > 1 else 0)


def assert_exact(got: torch.Tensor, want: torch.Tensor, locate, what: str = "") -> None:
    """Bitwise equality.  `want` has got's dtype (use round_to).  +0 and -0 compare equal: the sign of an exact zero
    depends on whether the compiler contracts a c - b s into an fma, which is no error."""
    assert got.shape == want.shape and got.dtype == want.dtype, (got.shape, want.shape, got.dtype, want.dtype)
    g2, w2 = got.reshape(got.shape[0], -1), want.reshape(want.shape[0], -1)
    sign = {4: -(2 ** 31), 2: -(2 ** 15), 1: 0x80}[got.element_size()]
    gb, wb = bits(g2), bits(w2)
    zero = lambda b: (b | sign) == sign
    bad = (gb != wb) & ~(zero(gb) & zero(wb))
    if bad.any():
        r, c = _first(bad)
        gv = g2[r, c].float().item() if g2.dtype != torch.uint8 else g2[r, c].view(torch.float8_e4m3fn).float().item()
        wv = w2[r, c].float().item() if w2.dtype != torch.uint8 else w2[r, c].view(torch.float8_e4m3fn).float().item()
        raise AssertionError(f"{what}: {int(bad.sum())} elements differ; first at {locate(r, c)}: got {gv!r} want {wv!r}")


def assert_within(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, locate, what: str = "") -> float:
    """|got - ref| <= bound element-wise (non-finite got fails).  Returns the worst err/bound ratio."""
    g = got.view(torch.float8_e4m3fn) if got.dtype == torch.uint8 else got
    g = g.double().reshape(got.shape[0], -1)
    ref, bound = ref.double().reshape(g.shape), bound.double().reshape(g.shape)
    assert (bound > 0).all(), f"{what}: bound must be positive"
    ratio = (g - ref).abs() / bound
    ratio = torch.where(torch.isfinite(g), ratio, torch.full_like(ratio, math.inf))
    worst = ratio.max().item()
    r, c = divmod(int(ratio.argmax()), g.shape[1])
    msg = (f"{what}: worst err/bound {worst:.3g} at {locate(r, c)}: got {g[r, c].item()!r} ref {ref[r, c].item()!r} "
           f"bound {bound[r, c].item():.3g}")
    if not worst <= 1.0:
        raise AssertionError(msg)
    print(msg)
    return worst


# ---------------------------------------------------------------- guard regions
class Guarded:
    """`view` = rows x cols of `dtype` inside a buffer with `pad_rows` extra rows above and below and at least 16 bytes
    of extra columns on each side (ld > cols, every row start 16-byte aligned as the TMA stores need).  `lr=False` puts
    no columns beside the view (contiguous rows, as ln_stats must be)."""

    def __init__(self, rows: int, cols: int, dtype: torch.dtype, device, pad_rows: int = 3, lr: bool = True,
                 pad_cols: int = 0):
        esz = torch.empty((), dtype=dtype).element_size()
        vec = 16 // esz
        pad = max(vec, (pad_cols + vec - 1) // vec * vec) if lr else 0
        self.pl = pad
        ld = self.pl + cols + pad
        ld = (ld + vec - 1) // vec * vec if lr else ld
        self.pr, self.rows, self.cols = pad_rows, rows, cols
        self.buf = torch.empty(rows + 2 * pad_rows, ld, dtype=dtype, device=device)
        self.pat = PATTERN[esz]
        bits(self.buf).fill_(self.pat)
        self.view = self.buf[pad_rows:pad_rows + rows, self.pl:self.pl + cols]

    def check(self, what: str = "") -> None:
        b = bits(self.buf).long() & ((1 << (8 * self.buf.element_size())) - 1)
        inside = torch.zeros_like(b, dtype=torch.bool)
        inside[self.pr:self.pr + self.rows, self.pl:self.pl + self.cols] = True
        untouched = b == self.pat
        if (~untouched & ~inside).any():
            r, c = _first(~untouched & ~inside)
            raise AssertionError(f"{what}: guard element overwritten at buffer row {r - self.pr} col {c - self.pl} "
                                 f"(view is rows [0, {self.rows}) cols [0, {self.cols}))")
        if (untouched & inside).any():
            r, c = _first(untouched & inside)
            raise AssertionError(f"{what}: {int((untouched & inside).sum())} elements never written; first at row "
                                 f"{r - self.pr} col {c - self.pl}")


# ---------------------------------------------------------------- references and bounds
def gemm_acc_bound(a: torch.Tensor, w: torch.Tensor, scale: float = 1.0) -> torch.Tensor:
    """Bound on the fp32 accumulation error of acc = A W^T (float64 [M, N]).

    Every product of two bf16 (or e4m3) values is exact in fp32.  However the tensor core orders and rounds the K - 1
    additions, each one adds at most one ulp (truncation instead of round-to-nearest: 2u, u = 2^-24) of a partial sum
    bounded by sum_k |a_k||w_k|.  So |acc - A W^T| <= 2u (K - 1) / (1 - 2u (K - 1)) (|A||W|^T) < 2u (K + 1) (|A||W|^T)
    for K < 2^20; the epilogue's fma with bias and acc_scale adds u |v|, charged by the callers."""
    k = a.shape[-1]
    return 2 * U32 * (k + 1) * (a.float().double().abs() @ w.float().double().abs().T) * abs(scale)


def gemm_acc_bound_fp8(a: torch.Tensor, w: torch.Tensor, scale: float = 1.0) -> torch.Tensor:
    """The FP8 mode adds each 128-product k-block's e4m3 wgmma partial to the fp32 accumulator on the CUDA cores.  The
    partial's accumulator is shorter than fp32 and its width is not documented; public measurements of Hopper give
    about 14 retained bits.  With 13 bits (ulp 2^-12 relative) and one truncating add per 32-product k-step, a block's
    partial is off by at most 4 * 2^-12 = 2^-10 of the block's sum |products|.  The fp32 promotion of the blocks adds
    2u per block as in gemm_acc_bound."""
    kb = a.shape[-1] // 128
    aa, ww = a.float().double().abs(), w.float().double().abs()
    full = aa @ ww.T
    return (2.0 ** -10 + 2 * U32 * (kb + 1)) * full * abs(scale)


def rope_ref(x: torch.Tensor, tab: torch.Tensor, pos: torch.Tensor, rope_cols: int) -> torch.Tensor:
    """Rotate adjacent column pairs (2j, 2j+1) of the first rope_cols columns by the table entry (cos, sin) of the
    row's position and pair j % 32 of the 64-column head.  x float64 [rows, n]; tab [P, 32, 2]; pos [rows]."""
    y = x.clone()
    if rope_cols == 0:
        return y
    r = x[:, :rope_cols].reshape(x.shape[0], rope_cols // 64, 32, 2)
    cs = tab.double()[pos.long()]                      # rows, 32, 2
    c, s = cs[:, None, :, 0], cs[:, None, :, 1]
    rot = torch.stack([r[..., 0] * c - r[..., 1] * s, r[..., 1] * c + r[..., 0] * s], -1)
    y[:, :rope_cols] = rot.reshape(x.shape[0], rope_cols)
    return y


def rope_bound(x: torch.Tensor, bx: torch.Tensor, tab: torch.Tensor, pos: torch.Tensor, rope_cols: int) -> torch.Tensor:
    """Bound after the rotation of rope_ref, given a bound bx on x: a c - b s moves by |c| bx_a + |s| bx_b, and its fp32
    evaluation (two products, one subtraction) adds at most 2u (|a c| + |b s|) + u |a c - b s|."""
    y = bx.clone()
    if rope_cols == 0:
        return y
    n = x.shape[0]
    xa = x[:, :rope_cols].reshape(n, rope_cols // 64, 32, 2).abs()
    ba = bx[:, :rope_cols].reshape(n, rope_cols // 64, 32, 2)
    cs = tab.double()[pos.long()].abs()
    c, s = cs[:, None, :, 0], cs[:, None, :, 1]
    e0 = c * ba[..., 0] + s * ba[..., 1] + 3 * U32 * (xa[..., 0] * c + xa[..., 1] * s)
    e1 = c * ba[..., 1] + s * ba[..., 0] + 3 * U32 * (xa[..., 1] * c + xa[..., 0] * s)
    y[:, :rope_cols] = torch.stack([e0, e1], -1).reshape(n, rope_cols)
    return y


def _gelu_tanh(v):
    return 0.5 * v * (1 + torch.tanh(math.sqrt(2 / math.pi) * (v + 0.044715 * v ** 3)))


def act_ref(v: torch.Tensor, act: int) -> torch.Tensor:
    """float64 activations: 0 none, 1 GELU-tanh, 2 GELU-erf, 3 Mish."""
    v = v.double()
    if act == 1:
        return _gelu_tanh(v)
    if act == 2:
        return 0.5 * v * (1 + torch.erf(v / math.sqrt(2)))
    if act == 3:
        return v * torch.tanh(torch.nn.functional.softplus(v))
    return v


def act_bound(v: torch.Tensor, bv: torch.Tensor, act: int) -> torch.Tensor:
    """Bound on act(v~) - act(v) for a kernel input v~ with |v~ - v| <= bv, evaluated as the epilogue does.

    Input propagation: |act'| <= 1.13 for GELU (both forms) and <= 1.1 for Mish, everywhere.
    GELU-tanh = 0.5 x (1 + tanh.approx(u)): tanh.approx's relative error EPS_TANH moves the result by at most
    0.5 |x| EPS_TANH; the five fp32 operations that form u and the result add at most 6u |x| (|u| <= 0.8 |x| (1 + |x|^2 / 20),
    whose rounding passes through 0.5 |x| |tanh'| <= 0.5 |x| and is covered by 6u |x| (1 + x^2 / 20)).
    GELU-erf = 0.5 x (1 + erff(x / sqrt 2)): erff is within 2 ulp; with the three fp32 operations <= 5u |x|.
    Mish = x tanh.approx(sp), sp = __logf(1 + __expf(x)) (sp = x beyond 15): __expf has relative error
    (2 + floor(1.173 |x|)) 2^-23 (<= 20 2^-23 for |x| <= 15); 1 + e rounds (u); __logf is within 2^-21.41 absolute for
    arguments in [0.5, 2] and 3 ulp elsewhere; a relative error d of the argument moves the log by d.  So
    |sp~ - sp| <= (20 2^-23 + u) + 2^-21.41 + 3 2^-23 sp, and tanh' <= 1 carries that to tanh.  The result is
    |x| (|sp~ - sp| + EPS_TANH + u)."""
    x, ax = v.double(), v.double().abs()
    if act == 0:
        return bv.clone()
    if act in (1, 2):
        prop = 1.13 * bv
        if act == 1:
            return prop + ax * (0.5 * EPS_TANH + 6 * U32 * (1 + x * x / 20))
        return prop + 5 * U32 * ax
    sp = torch.nn.functional.softplus(x)
    dsp = 21 * 2.0 ** -23 + 2.0 ** -21.41 + 3 * 2.0 ** -23 * sp
    dsp = torch.where(x > 15, U32 * ax, dsp)
    return 1.1 * bv + ax * (dsp + EPS_TANH + U32)


def out_bound(ref: torch.Tensor, b: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """Add the output rounding: the kernel rounds its fp32 value (within b of ref) once, relative error u_out."""
    mag = ref.double().abs() + b
    if dtype == torch.bfloat16:
        return b + U_BF16 * mag
    if dtype in (torch.uint8, torch.float8_e4m3fn):
        return b + U_E4M3 * mag + E4M3_SUB
    return b + U32 * mag


def attention_ref(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, kv_len=None):
    """float64 softmax(q k^T) v per (batch, head) for [B, H, N, 64] inputs; also returns p |v| (the softmax-weighted
    mean of |v|) for attention_bound.  Keys at or beyond kv_len[b] are masked."""
    q, k, v = q.double(), k.double(), v.double()
    s = q @ k.transpose(-1, -2)
    if kv_len is not None:
        n = k.shape[2]
        m = torch.arange(n, device=k.device)[None] < kv_len.to(k.device)[:, None].long()
        s = s.masked_fill(~m[:, None, None, :], float("-inf"))
    p = torch.softmax(s, -1)
    return p @ v, p @ v.abs(), (q.abs() @ k.abs().transpose(-1, -2)).masked_fill(p == 0, 0).amax(-1, keepdim=True)


def attention_bound(o: torch.Tensor, pv: torch.Tensor, qk_abs: torch.Tensor, logit_max: float, tiles: int,
                    out_dtype=torch.bfloat16) -> torch.Tensor:
    """Bound on the flash-attention output, per element.

    The kernel forms p_i = ex2.approx(s_i log2 e - m log2 e), sums the fp32 p_i into l, multiplies bf16(p_i) by v_i
    and scales the result by 1 / l.  O = sum w_i v_i with weights w_i = p_i / l; perturbing each p_i by a relative
    error d_i moves O by at most 2 max|d| sum w_i |v_i| (numerator and denominator), i.e. 2 d p|v|.  Sources of d:
    bf16 rounding of p in the P V product (U_BF16); the S = Q K^T accumulation (2u 65 sum |q||k|, logits' error times
    ln-scale 1); the fp32 argument s log2e - m log2e (3u |s| log2e, then ln 2 per unit of log2) plus ex2.approx
    (EPS_EX2); the running-max rescale of o and l (one ex2.approx and one product per 128-key tile, applied to both o
    and l but rounded separately: 2 (EPS_EX2 + u) per tile).  The P V accumulation adds 2u (N + 1) p|v| as in
    gemm_acc_bound, 1 / l and the product 3u |O|, and the output rounding u_out |O|."""
    d = U_BF16 + 2 * U32 * 65 * qk_abs + 3 * U32 * abs(logit_max) * 1.4427 * 0.6932 + EPS_EX2 \
        + 2 * tiles * (EPS_EX2 + U32)
    b = 2 * d * pv + 2 * U32 * (tiles * 128 + 1) * pv + 3 * U32 * o.abs()
    return out_bound(o, b, out_dtype)


# ---------------------------------------------------------------- fused AdaLN (LayerNorm finished in the GEMM epilogue)
EPS_LN = float(torch.tensor(1e-6, dtype=torch.float32))   # the kernels' 1e-6f
U_HILO = 2.0 ** -16       # |a - hi - lo| <= 2^-8 |a - hi| <= 2^-16 |a| for hi = bf16(a), lo = bf16(a - hi)


def fused_ln_stats_bound(x: torch.Tensor):
    """(mean, var, rstd, dr, dmean) per row [M, 1] of the producer's float64 rows x [M, K], with the bound dr on the
    relative error of the rstd and dmean on the error of the mean that the fused-LN consumer forms.

    The producer adds each 64-column unit in four chains of 8 per 32 columns, the second 32 continuing chain 0 and
    two combining levels after each half: at most 20 roundings per element, the squares by fma (one rounding each
    step).  The consumer adds the K / 64 unit values in unit order.  So |dS1| <= gam(20 + n) sum |x| and
    |dS2| <= gam(20 + n) sum x^2 (n = K / 64); 1 / K is a power of two.  var = E[x^2] - mean^2 then loses the mean's
    error twice, and the square, the subtraction and the eps add round once each:
        dvar <= dE2 + (2 |mean| + dmean) dmean + 3u (E[x^2] + dE2 + eps).
    With zeta = dvar / (var + eps) < 1 the rsqrt of the perturbed argument is within zeta / (2 (1 - zeta)^1.5) of
    rstd relatively, and rsqrtf adds 2 ulp.  zeta grows like n u r^2 with r = |mean| / std: this is the cancellation of
    E[x^2] - mean^2.  At zeta >= 1 the bound is infinite (the variance may cancel to zero and be clamped)."""
    M, K = x.shape
    n = K // 64
    g = (20 + n) * U32 / (1 - (20 + n) * U32)
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    rstd = 1 / torch.sqrt(var + EPS_LN)
    ex2 = (x * x).mean(-1, keepdim=True)
    dmean = g * x.abs().mean(-1, keepdim=True)
    dex2 = g * ex2
    dvar = dex2 + (2 * mean.abs() + dmean) * dmean + 3 * U32 * (ex2 + dex2 + EPS_LN)
    zeta = dvar / (var + EPS_LN)
    dr = torch.where(zeta < 1, zeta / (2 * (1 - zeta.clamp(max=0.999)) ** 1.5), torch.full_like(zeta, math.inf))
    return mean, var, rstd, dr + 2.0 ** -22 + U32, dmean


def fused_ln_ref_bound(x: torch.Tensor, bx: torch.Tensor, s: torch.Tensor, b: torch.Tensor, w: torch.Tensor,
                       bias: torch.Tensor, acc_err: torch.Tensor, *, op_err: torch.Tensor | None = None,
                       operand: torch.Tensor | None = None, w_eff: torch.Tensor | None = None):
    """float64 v = Linear(LayerNorm(x) (1 + s) + b) + bias before the consumer's activation / RoPE, for the
    producer's float64 rows x [M, K] (within bx [M, K] of the kernel's fp32 x), and the bound on the fused-LN
    consumer's fp32 value of it:  rstd (x~ W~^T - mean c1) + c2 with c1 = (1 + s) w^T, c2 = b w^T + bias from the
    hi / lo table of the bf16 weight w [N, K], x~ the producer's operand (bf16 / e4m3 / block-scaled e4m3 of
    x (1 + s)) and W~ the weight the GEMM multiplies (w, or its dequantised e4m3 copy w_eff).

    The bound is the sum of
    * operand: rstd sum_k op_err_k |W~_nk|, op_err >= |x~ - x (1 + s)| (u_op |x (1 + s)|: the rounding is relative to
      |x|, not to the spread, so this term grows like 1 + r with r = |mean| / std);
    * weight (FP8 modes): rstd sum_k (|x (1 + s)| + op_err) |W~ - w|_nk, the e4m3 weight against the bf16 one the
      tables use;
    * accumulation: rstd acc_err (gemm_acc_bound / gemm_acc_bound_fp8 of the operands, times the weight scale);
    * statistics: |rstd (x - mean)(1 + s) W~^T| dr + rstd dmean |c1| (fused_ln_stats_bound: E[x^2] - mean^2 from
      the fp32 unit sums);
    * tables: c1 = hi + lo rows, each an fp32 product of the split (1 + s) with w: the split leaves U_HILO |1 + s|
      and the fp32 products 2u (K + 1) of |1 + s| |w|; the epilogue's add hi + lo rounds once (the same for c2, whose
      c2 + bias adds round twice); that error is multiplied by rstd |mean|;
    * epilogue: rstd * acc_scale, mean * rstd, the inner fma -mu_r c1 + c2 and the outer fma round once each;
    * input: the kernel's x is within bx of x; ln_propagate carries that through the LayerNorm.
    Products of two of these terms are below 1 % of their sum, which the factor 1.01 covers.

    With `operand` (the float64 value of the operand x~ the kernel multiplied) the reference is the consumer's
    arithmetic on that operand with exact statistics and tables, rstd (x~ W~^T - mean c1) + c2, and the operand and
    weight terms drop out: a bound at the fp32 level that a wrong table row or wrong statistics exceed."""
    from hbm_check import ln_propagate
    x = x.double()
    K = x.shape[1]
    a = 1 + s.double()
    wd = w.float().double()
    we = wd if w_eff is None else w_eff.double()
    wa = we.abs()
    mean, var, rstd, dr, dmean = fused_ln_stats_bound(x)
    xs = x * a
    c1 = a @ wd.T
    c2 = b.double() @ wd.T + bias.double()
    if operand is None:
        centred = rstd * ((x - mean) * a) @ we.T
        v = centred + (b.double() @ wd.T) + bias.double()
        if w_eff is not None:
            v = rstd * ((x - mean) * a) @ wd.T + c2
        xa = xs.abs() + (0 if op_err is None else op_err)
        bd = rstd * (op_err @ wa.T) if op_err is not None else torch.zeros_like(v)
        if w_eff is not None:
            bd = bd + rstd * (xa @ (we - wd).abs().T)
    else:
        xt = operand.double()
        centred = rstd * (xt @ we.T - mean * c1)
        v = centred + c2
        xa = xt.abs()
        bd = torch.zeros_like(v)
    bd = bd + rstd * acc_err
    bd = bd + centred.abs() * dr + rstd * dmean * c1.abs()
    aa, ba = a.abs(), b.double().abs()
    dc1 = (U_HILO * aa + 4 * U32 * (K + 1) * aa) @ wd.abs().T + U32 * c1.abs()
    dc2 = (U_HILO * ba + 4 * U32 * (K + 1) * ba) @ wd.abs().T + 2 * U32 * c2.abs()
    bd = bd + rstd * mean.abs() * dc1 + dc2
    inner = -rstd * mean * c1 + c2
    bd = bd + U32 * (rstd * (xa @ wa.T) + 2 * rstd * mean.abs() * c1.abs() + inner.abs() + v.abs())
    bd = bd + ln_propagate(x, bx, a.expand_as(x)) @ wd.abs().T
    return v, 1.01 * bd
