"""-m gpu: known-answer tests of the wgmma GEMM and the flash attention.

The GEMM operands are small integers (bf16) or e4m3 values from {0, +-1, +-2}; bias and residual are integers, gates
and 1 + ln_scale powers of two, q_scale = 0.125 and the RoPE table holds quarter turns only.  Every partial sum is
then an integer (or a dyadic fraction with few bits) below 2^20, so the fp32 result is exact in ANY summation order:
fp32 outputs must equal the float64 reference bitwise, bf16 / e4m3 outputs its round-to-nearest, ln_stats exactly.
Any indexing, masking, tail or ring-phase mistake is a nonzero difference, reported with its tile, row and column.
Every output is written into a NaN-filled buffer with guard rows and columns (ld > n), which must stay untouched.
Block-scaled operands carry power-of-two scales, so they stay exact too; block-scaled e4m3 outputs must equal the scale
rule of the float64 result bitwise.  After an activation (tanh.approx, __expf / __logf, erff) no exact answer exists:
the output is checked against a float64 bound and bitwise against the same GEMM run in one-wave slices.

INSTANTIATIONS lists the kernel instantiation (gemm.cu dispatch_epi) each GEMM case below launches; a CPU test checks it
against gemm.cu so that no instantiation and tile width goes untested.
"""
import pytest
import torch
import torch.nn.functional as F

from kernel_check import (E4M3_SUB, U32, U_E4M3, Guarded, act_bound, act_ref, assert_exact, assert_within, attn_tiles,
                          bits, cdiv, gemm_tile_count, gemm_tiles, instantiation, out_bound, round_to, rope_ref)

pytestmark = pytest.mark.gpu
DEV = "cuda"
F8 = torch.float8_e4m3fn
STAGES = {64: 6, 128: 4}
EXACT_LIMIT = 2.0 ** 20


def ints(shape, amax, seed, density=1.0, dtype=torch.bfloat16):
    """Uniform integers in [-amax, amax], each zero with probability 1 - density."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    v = torch.randint(-amax, amax + 1, shape, generator=g, device=DEV)
    if density < 1.0:
        v = v * (torch.rand(shape, generator=g, device=DEV) < density)
    return v.to(dtype) if dtype != F8 else v.float().to(F8)


def pow2(shape, seed):
    """Gates: +-{0.5, 1, 2}."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    e = torch.randint(-1, 2, shape, generator=g, device=DEV).float()
    s = torch.randint(0, 2, shape, generator=g, device=DEV).float() * 2 - 1
    return s * torch.exp2(e)


def quarter_turns(rows, seed):
    """RoPE table [rows, 32, 2] of (cos, sin) in {(1, 0), (0, 1), (-1, 0), (0, -1)}: rotation is exact."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = torch.randint(0, 4, (rows, 32), generator=g, device=DEV)
    cs = torch.tensor([[1.0, 0.0], [0.0, 1.0], [-1.0, 0.0], [0.0, -1.0]], device=DEV)
    return cs[q].contiguous()


def row_lens(nb, rpb):
    """0, mid-tile and the full utterance, cycling over the utterances."""
    return torch.tensor([(0, rpb // 2 + 1 if rpb > 1 else 1, rpb)[b % 3] for b in range(nb)], dtype=torch.int32, device=DEV)


def pow2_scales(shape, seed, lo, hi):
    """Block scales 2^e, e uniform in [lo, hi] (test_gpu_fp8_block._pow2 on the device)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.exp2(torch.randint(lo, hi + 1, shape, generator=g, device=DEV).float())


def rms_row_stats(M, units, seed, zero_rows=()):
    """RMSNorm consumer input: per row (sum, sum of squares) of every 64-column unit with the unit's sum of squares
    64 4^e, e in {0, 1, 2, 3} per row, so the kernel's rsqrt(sum x^2 / (64 units)) = 2^-e exactly (rsqrtf is exact at
    powers of two, as the fused-LN consumer cases rely on; 1 / (64 units) is exact for units a power of two).  The sums
    are arbitrary integers (the RMS consumer must not read them).  zero_rows get all-zero statistics (their A rows are
    zero too): the kernel clamps the sum to 1e-24, and 0 times its finite rstd is 0, so the output is the bias."""
    assert units & (units - 1) == 0, "the RMS consumer is exact only for K / 64 a power of two"
    g = torch.Generator(device=DEV).manual_seed(seed)
    e = torch.randint(0, 4, (M,), generator=g, device=DEV)
    stats = torch.empty(M, units, 2, device=DEV)
    stats[..., 0] = torch.randint(-50, 51, (M, units), generator=g, device=DEV).float()
    stats[..., 1] = (64.0 * torch.exp2(2.0 * e.float()))[:, None]
    rstd = torch.exp2(-e.double())
    zr = torch.as_tensor(list(zero_rows), dtype=torch.long, device=DEV)
    stats[zr] = 0.0
    return stats, rstd


def ln_row_stats(M, units, seed):
    """Fused-LN consumer input: per row (sum, sum of squares) of every 64-column unit such that mean and rstd are powers
    of two (mean 2, variance 2^20: rstd 2^-10; mean -4, variance 2^16: rstd 2^-8; the LayerNorm's 1e-6 is below half an
    ulp of the variance).  The kernel divides the sums by 64 * units, exactly only when units is a power of two."""
    assert units & (units - 1) == 0, "the fused-LN consumer is exact only for K / 64 a power of two"
    g = torch.Generator(device=DEV).manual_seed(seed)
    kind = torch.rand(M, generator=g, device=DEV) < 0.5
    mean = torch.where(kind, 2.0, -4.0).double()
    var = torch.where(kind, 2.0 ** 20, 2.0 ** 16).double()
    stats = torch.empty(M, units, 2, device=DEV)
    stats[..., 0] = (mean * 64)[:, None].float()
    stats[..., 1] = ((var + mean * mean) * 64)[:, None].float()
    return stats, mean, var.rsqrt()


def granularity(x):
    """The largest power of two 2^-e <= 1 (e <= 30) of which every element of x is a multiple."""
    for e in range(31):
        y = x * 2.0 ** e
        if torch.equal(y, y.round()):
            return 2.0 ** -e
    raise AssertionError("reference is not a dyadic fraction with few bits")


def assert_fp32_exact(x, what):
    assert torch.equal(x.float().double(), x), f"{what}: the float64 reference is not exact in fp32 (operands too large)"


def conv_ref(A, W, *, M, N, K, rpb, nb, taps, pad, grouped, dilation=1):
    """float64 Conv1d of the implicit-GEMM operands: A [nb rpb, channels] (channels = N grouped, else K), W [N, taps K]
    with W[n, t K + c] the weight of input channel c (of the column's 64-channel group when grouped) at tap t; tap t of
    frame m reads frame m + t dilation - pad."""
    if not grouped:   # frames gathered per tap, one float64 matmul (cuBLAS) over [M, taps K]
        src = torch.arange(rpb, device=A.device)[:, None] + torch.arange(taps, device=A.device)[None] * dilation - pad
        ok = (src >= 0) & (src < rpb)
        x = A.reshape(nb, rpb, K)[:, src.clamp(0, rpb - 1)] * ok[None, :, :, None]      # nb, rpb, taps, K
        return x.reshape(M, taps * K) @ W.reshape(N, taps * K).T
    x = A.reshape(nb, rpb, N).transpose(1, 2)
    wt = W.reshape(N, taps, K).permute(0, 2, 1)
    y = F.conv1d(x, wt, padding=pad, dilation=dilation, groups=N // 64)
    return y.transpose(1, 2).reshape(M, N)


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def run_exact(*, M, N, K, tile, w_static, out="bf16", seed=0, amax=4, density=1.0, rpb=0, nb=1, batched=False,
              row_len=False, gate=None, resid=None, out2=None, ln_scale=False, rope=False, ab8=False, pad_cols=0,
              act=0, scaled=False, out_blocks=False, scale_exp=(-3, 3), a_scale_ld=0, ln_in=False, conv_taps=1,
              conv_pad=0, conv_grouped=False, conv_dilation=1, ln_rms=False, ln_stats=False, a_slot=False,
              out2_slot=None, bias=True, rope_cols=0, rope_col2=0, q_cols=0):
    """One GEMM launch against its float64 reference.  out: 'bf16' | 'f32' | 'e4m3'; gate: None | 'shared' (one [N]
    vector for every utterance); resid: None | 'alias' (resid is out itself) | 'sep'; out2: None | 'bf16' | 'e4m3'.

    scaled: block-scaled FP8 (dispatch_scaled) — A and W e4m3 codes from {0, +-1, +-2}, a_scale one power of two per
    (row, 64-column unit) in a [K/64][a_scale_ld] buffer (default ld M + 8, the columns beyond M NaN), w_scale one per
    channel, exponents in scale_exp; e4m3 outputs are then block-scaled (out_scale / out2_scale), and their codes and
    scales must equal weights.quantize_e4m3_blocks of the float64 result bitwise.  out_blocks: block-scaled e4m3
    outputs of bf16 operands (the Mish producer of the block-scaled mode).
    ln_in: fused-LN consumer with power-of-two row statistics (ln_row_stats) and an integer c1 / c2 table.
    conv_taps / conv_pad / conv_grouped / conv_dilation: implicit Conv1d over batched utterances (conv_ref); K is the
    k per tap.  W is [N, taps k_pad] with k_pad = K rounded up to 64 (BigVGAN's C = 96, 48, 24); its padding columns
    hold nonzero integers that the reference ignores, so a k-block that reads past channel K of its row (the next
    frame's channels instead of the TMA's zero fill) changes the result.
    ln_rms: the RMSNorm consumer (UNetT) with power-of-two row scales (rms_row_stats) and all-zero rows 5 and M - 1.
    ln_stats without ln_scale: the UNetT producer, out2 a plain bf16 copy of the fp32 out, ln_stats of it.
    a_slot: A is the right half of a [M, 2K] buffer whose left half holds other integers (lda = 2K, a UNetT skip slot);
    out2_slot 'left' | 'right': out2 is that half of a [M, 2N] buffer (ldo2 = 2N); the other half must stay untouched.
    rope_cols / rope_col2 / q_cols (with rope): the rotated column ranges and the q_scale range; default 2N/3 and N/3.
    act (1 GELU-tanh, 2 GELU-erf, 3 Mish): the pre-activation is exact; the output must be (a) within act_bound of the
    float64 activation and (b) bitwise equal to the same GEMM launched in slices of at most SMs tiles, in which every tile
    is the first and only tile of its CTA."""
    from f5_tts_mlx_b200 import ops
    from f5_tts_mlx_b200.weights import quantize_e4m3_blocks
    odt = {"bf16": torch.bfloat16, "f32": torch.float32, "e4m3": torch.uint8}[out]
    rpb_e = rpb or M
    ab8 = ab8 or scaled
    conv = conv_taps > 1 or conv_grouped
    assert not (conv and ab8) and (not conv or (rpb and batched)), "conv mode: bf16 operands, batched utterances"
    kin = N if conv_grouped else K
    kp = -(-K // 64) * 64 if conv and not conv_grouped else K
    if ab8:
        A, W = ints((M, K), 2, seed, density, F8), ints((N, K), 2, seed + 1, density, F8)
        acc_scale = 1.0 if scaled else 0.5
    else:
        A, W = ints((M, kin), amax, seed, density), ints((N, conv_taps * kp), amax, seed + 1, density)
        acc_scale = 1.0
    if kp != K:       # the padding columns of every tap: nonzero, ignored by the reference
        W.view(N, conv_taps, kp)[:, :, K:] = ints((N, conv_taps, kp - K), amax, seed + 11).abs() + 1
    if a_slot:
        slot = ints((M, 2 * K), amax, seed + 12)
        slot[:, K:] = A
        A = slot[:, K:]
    zero_rows = (5, M - 1) if ln_rms else ()
    if zero_rows:
        A[list(zero_rows)] = 0
    bias = ints((N,), 8, seed + 2, dtype=torch.float32) if bias else None
    rows = torch.arange(M, device=DEV)
    bidx, pos = rows // rpb_e, rows % rpb_e
    A64 = A.float().double()
    W64 = W.float().double().view(N, conv_taps, kp)[:, :, :K].reshape(N, conv_taps * K) if kp != K else W.float().double()
    bias64 = bias.double() if bias is not None else torch.zeros(N, dtype=torch.float64, device=DEV)
    kw = dict(bias=bias, tile_n=tile, w_static=bool(w_static), ab_fp8=ab8, acc_scale=acc_scale)
    colscale = torch.full((N,), acc_scale, dtype=torch.float64, device=DEV)
    sa_buf = None
    if scaled:
        units = K // 64
        sa_buf = torch.full((units, a_scale_ld or M + 8), float("nan"), device=DEV)
        assert sa_buf.shape[1] >= M
        sa = pow2_scales((units, M), seed + 7, *scale_exp)
        sa_buf[:, :M] = sa
        sw = pow2_scales((N,), seed + 8, *scale_exp)
        A64 = (A64.view(M, units, 64) * sa.T.double()[..., None]).view(M, K)
        colscale = sw.double()
        kw.update(a_scale=sa_buf, w_scale=sw)
    if conv:
        cw = dict(M=M, N=N, K=K, rpb=rpb, nb=nb, taps=conv_taps, pad=conv_pad, grouped=conv_grouped,
                  dilation=conv_dilation)
        acc, accb = conv_ref(A64, W64, **cw), conv_ref(A64.abs(), W64.abs(), **cw)
        kw.update(n=N, k=K, conv_taps=conv_taps, conv_pad=conv_pad, conv_grouped=conv_grouped,
                  conv_dilation=conv_dilation)
    else:
        acc, accb = A64 @ W64.T, A64.abs() @ W64.abs().T
    assert (accb < EXACT_LIMIT).all(), "operands too large for an exact test"     # bounds every partial sum
    stats = None
    if ln_rms:
        stats, rstd = rms_row_stats(M, K // 64, seed + 9, zero_rows)
        v = rstd[:, None] * acc + bias64[None]
        vb = rstd[:, None] * accb + bias64.abs()[None]
        kw.update(ln_rms=True, ln_in_stats=stats)
    elif ln_in:
        stats, mean, rstd = ln_row_stats(M, K // 64, seed + 9)
        tab = ints((4, N + 8), 8, seed + 10, dtype=torch.float32)            # ld > N
        c1 = (tab[0] + tab[1])[:N].double()
        c2 = (tab[2] + tab[3])[:N].double() + bias64
        mu_r = (mean * rstd)[:, None]
        v = rstd[:, None] * colscale[None] * acc - mu_r * c1[None] + c2[None]
        vb = rstd[:, None] * colscale[None] * accb + (mu_r * c1[None]).abs() + c2.abs()[None]
        kw.update(ln_in_stats=stats, ln_tab=tab)
    else:
        v = acc * colscale[None] + bias64
        vb = accb * colscale[None] + bias64.abs()
    assert_fp32_exact(v, "pre-activation")
    bnd = None                                     # None: v is exact; else |kernel - v| <= bnd before the output rounding
    if act:
        assert not rope
        pre = v
        v = act_ref(pre, act)
        bnd = act_bound(pre, torch.zeros_like(pre), act)
        kw.update(act=act)
    if rpb:
        kw.update(rows_per_batch=rpb, num_batches=nb, batched_tiles=batched)
    if rope:
        tab_r = quarter_turns(rpb_e, seed + 3)
        rc, qc = rope_cols or 2 * N // 3, q_cols or N // 3
        v = rope_ref(v, tab_r, pos, rc)
        if rope_col2:
            v[:, rope_col2:] = rope_ref(v[:, rope_col2:], tab_r, pos, rc)
        v[:, :qc] *= 0.125
        kw.update(rope=tab_r, rope_cols=rc, rope_col2=rope_col2, q_scale=0.125, q_cols=qc)
    valid = torch.ones(M, dtype=torch.bool, device=DEV)
    lens = None
    if row_len:
        lens = row_lens(nb, rpb_e)
        valid = pos < lens.long()[bidx]
        v = torch.where(valid[:, None], v, torch.zeros_like(v))
        if bnd is not None:
            bnd = torch.where(valid[:, None], bnd, torch.zeros_like(bnd))
        kw.update(row_len=lens)
    g_out = Guarded(M, N, odt, DEV, pad_cols=pad_cols)
    if gate is not None:
        assert gate == "shared"
        gt = pow2((N,), seed + 4)
        gm = gt.double()[None]
        v, vb = v * gm, vb * gm.abs()
        bnd = bnd * gm.abs() if bnd is not None else None
        kw.update(gate=gt)
    r = None
    if resid is not None:
        r = ints((M, N), 16, seed + 5, dtype=torch.float32)
        v, vb = v + r.double(), vb + r.double().abs()
        if resid == "alias":
            assert odt == torch.float32
            g_out.view.copy_(r)
            kw.update(resid=g_out.view)
        else:
            kw.update(resid=r)
    if bnd is not None and (gate is not None or resid is not None):
        bnd = bnd + U32 * v.abs()                  # v * gate + resid: one fma
    if bnd is None:
        assert (vb < EXACT_LIMIT).all(), "operands too large for an exact test"
        assert_fp32_exact(v, "out")
    blk_out, blk_out2 = (scaled or out_blocks) and out == "e4m3", (scaled or out_blocks) and out2 == "e4m3"
    so = s2 = g2 = st = s = None
    if blk_out:
        so = Guarded(N // 64, M, torch.float32, DEV, lr=False)
        kw.update(out_scale=so.view)
    if out2 is not None:
        g2 = Guarded(M, 2 * N if out2_slot else N, torch.uint8 if out2 == "e4m3" else torch.bfloat16, DEV)
        o2 = {None: slice(0, N), "left": slice(0, N), "right": slice(N, 2 * N)}[out2_slot]
        other = slice(N, 2 * N) if out2_slot == "left" else slice(0, N)
        kw.update(out2=g2.view[:, o2], out2_fp8=out2 == "e4m3")
        if blk_out2:
            s2 = Guarded(N // 64, M, torch.float32, DEV, lr=False)
            kw.update(out2_scale=s2.view)
        if ln_scale or ln_stats:
            st = Guarded(M, N // 64 * 2, torch.float32, DEV, lr=False)
            kw.update(ln_stats=st.view.view(M, N // 64, 2))
            if bnd is None:   # every partial unit sum (of squares) is a multiple of gq (gq^2) below 2^24 of them
                gq = granularity(v)
                u = v.view(M, N // 64, 64) / gq
                assert (u.abs().sum(-1) < 2 ** 24).all() and ((u * u).sum(-1) < 2 ** 24).all(), "ln_stats would not be exact"
        if ln_scale:
            s = pow2((N,), seed + 6).abs() - 1          # 1 + s in {0.5, 1, 2}
            kw.update(ln_scale=s)
            want2 = v * (1 + s.double())
        else:
            want2 = v
        if out2 == "e4m3" and not blk_out2:
            assert (want2.abs() + (bnd if bnd is not None else 0) * 2 < 448).all(), "per-tensor e4m3 out2 would saturate"
    ops.gemm(A, W, g_out.view, out_fp8=out == "e4m3", **kw)
    torch.cuda.synchronize()
    loc = gemm_tiles(64 if conv_grouped else tile, rpb_e, batched)
    what = f"M={M} N={N} K={K} tile={tile} w_static={w_static}"
    unit = lambda r_, c_: f"row {r_} unit {c_ // 2}"
    if blk_out:
        _check_blocks(g_out, so, v, bnd, loc, what + " out")
    elif bnd is None:
        assert_exact(g_out.view, round_to(v, odt), loc, what + " out")
    else:
        assert_within(g_out.view, v, out_bound(v, bnd, odt) + 1e-300, loc, what + " out")   # exact zeros: bound 0
    g_out.check(what + " out guard")
    if g2 is not None:
        sc = (1 + s.double()) if s is not None else torch.ones(N, dtype=torch.float64, device=DEV)
        v2 = g2.view[:, o2]
        if blk_out2:
            # the scale rule of the float64 result (exact), or of the kernel's own fp32 out when that is not exact
            _check_blocks(g2, s2, want2 if bnd is None else g_out.view.double() * sc, None, loc, what + " out2")
        elif bnd is None:
            assert_exact(v2, round_to(want2, v2.dtype), loc, what + " out2")
        else:
            assert_within(v2, want2, out_bound(want2, sc.abs() * bnd + U32 * want2.abs(), v2.dtype) + 1e-300,
                          loc, what + " out2")
        if out2_slot:   # the slot's other half is not touched; then it counts as written for the guard check
            half = g2.view[:, other]
            assert (bits(half).long() & 0xFFFF == g2.pat).all(), f"{what} out2: the other half of the slot was written"
            half.zero_()
        g2.check(what + " out2 guard")
    if st is not None:
        u = v.view(M, N // 64, 64)
        want = torch.stack([u.sum(-1), (u * u).sum(-1)], -1).reshape(M, N // 64 * 2)
        if bnd is None:
            assert_exact(st.view, round_to(want, torch.float32), unit, what + " ln_stats")
        else:   # four fp32 chains of 16 per unit, combined (test_gpu_kernels._producer_check)
            ub = bnd.view(M, N // 64, 64)
            b1 = ub.sum(-1) + 64 * U32 * u.abs().sum(-1)
            b2 = (2 * u.abs() * ub + ub * ub).sum(-1) + 66 * U32 * (u * u).sum(-1)
            assert_within(st.view, want, torch.stack([b1, b2], -1).reshape(M, N // 64 * 2) + 1e-300, unit,
                          what + " ln_stats")
        st.check(what + " ln_stats guard")
    if act:
        _check_slices(ops, A, W, kw, g_out, g2.view[:, o2] if g2 is not None else None, st, so, s2,
                      r if resid == "alias" else None,
                      dict(M=M, N=N, tile=64 if conv_grouped else tile, rpb=rpb, nb=nb, batched=batched, lens=lens,
                           stats=stats, sa_buf=sa_buf, resid_sep=r if resid == "sep" else None), loc, what)


def _check_blocks(g, gs, want, bnd, loc, what):
    """Block-scaled e4m3 output: codes g [M, N] and scales gs [N/64][M].  bnd None: codes and scales equal the scale
    rule of `want` bitwise (masked rows without a residual are zero with scale 1); else (`want` inexact) the dequantised
    output is within half an e4m3 ulp of the scale plus bnd, and every nonzero unit's largest code is in [224, 448]."""
    from f5_tts_mlx_b200.weights import quantize_e4m3_blocks
    M, N = g.view.shape
    if bnd is None:
        q, sc = quantize_e4m3_blocks(want, 64)
        assert_exact(gs.view.T.contiguous(), sc, lambda r, c: f"row {r} unit {c}", what + " scales")
        assert_exact(g.view, q, loc, what + " codes")
    else:
        codes = g.view.view(F8).double().view(M, N // 64, 64)
        sc = gs.view.T.double()
        deq = (codes * sc[..., None]).view(M, N)
        b = bnd + U_E4M3 * (want.abs() + bnd) + E4M3_SUB * sc.repeat_interleave(64, 1)
        assert_within(deq, want, b, loc, what + " dequantised")
        amax = codes.abs().amax(-1)
        nz = want.abs().view(M, N // 64, 64).amax(-1) > 0
        assert ((amax >= 224) & (amax <= 448))[nz].all(), what + ": a unit's largest code is outside [224, 448]"
    gs.check(what + " scale guard")


def _check_slices(ops, A, W, kw, g_out, g2, st, so, s2, r_alias, geo, loc, what):
    """(b) of run_exact's activation check: the same GEMM as sub-launches of at most SMs tiles each.  Flat rows are cut at
    128-row boundaries; utterances (batched or conv mode, or a row mask) are kept whole.  Every sub-launch gets views
    with row offsets into A, out, out2, resid, ln_stats, ln_in_stats, a_scale (its ld kept) and row_len, and its own
    [N/64][rows] scale buffers, concatenated for the comparison."""
    M, N, tile, rpb, nb = geo["M"], geo["N"], geo["tile"], geo["rpb"], geo["nb"]
    sms = _sm_count()
    if rpb:      # whole utterances, as many per slice as fit in one wave
        cuts, b = [], 0
        while b < nb:
            e = b + 1
            while e < nb and gemm_tile_count(N, (e + 1 - b) * rpb, tile, rows_per_batch=rpb, num_batches=e + 1 - b,
                                             batched=geo["batched"]) <= sms:
                e += 1
            cuts.append((b * rpb, e * rpb, b, e))
            b = e
    else:
        step = (sms // cdiv(N, tile)) * 128
        assert step > 0
        cuts = [(r0, min(r0 + step, M), 0, 1) for r0 in range(0, M, step)]
    out_s = torch.empty(g_out.view.shape, dtype=g_out.view.dtype, device=DEV)
    if r_alias is not None:
        out_s.copy_(r_alias)
    out2_s = torch.empty(g2.shape, dtype=g2.dtype, device=DEV) if g2 is not None else None
    st_s = torch.empty(st.view.shape, dtype=torch.float32, device=DEV) if st is not None else None
    so_s, s2_s = [], []
    for r0, r1, b0, b1 in cuts:
        m = r1 - r0
        t = gemm_tile_count(N, m, tile, rows_per_batch=rpb if rpb else 0, num_batches=b1 - b0 if rpb else 1,
                            batched=geo["batched"])
        assert t <= sms, f"slice rows [{r0}, {r1}) has {t} tiles > {sms} SMs"
        k = dict(kw)
        if rpb:
            k["num_batches"] = b1 - b0
        if geo["lens"] is not None:
            k["row_len"] = geo["lens"][b0:b1]
        if "resid" in k:
            k["resid"] = out_s[r0:r1] if r_alias is not None else geo["resid_sep"][r0:r1]
        if geo["stats"] is not None:
            k["ln_in_stats"] = geo["stats"][r0:r1]
        if geo["sa_buf"] is not None:
            k["a_scale"] = geo["sa_buf"][:, r0:]
        if out2_s is not None:
            k["out2"] = out2_s[r0:r1]
        if st_s is not None:
            k["ln_stats"] = st_s[r0:r1].view(m, N // 64, 2)
        if so is not None:
            so_s.append(torch.empty(N // 64, m, device=DEV))
            k["out_scale"] = so_s[-1]
        if s2 is not None:
            s2_s.append(torch.empty(N // 64, m, device=DEV))
            k["out2_scale"] = s2_s[-1]
        ops.gemm(A[r0:r1], W, out_s[r0:r1], out_fp8=g_out.view.dtype == torch.uint8, **k)
    torch.cuda.synchronize()
    sl = what + f" vs {len(cuts)} one-wave slices"
    assert_exact(g_out.view, out_s, loc, sl + " out")
    if out2_s is not None:
        assert_exact(g2, out2_s, loc, sl + " out2")
    if st_s is not None:
        assert_exact(st.view, st_s, lambda r_, c_: f"row {r_} unit {c_ // 2}", sl + " ln_stats")
    if so is not None:
        assert_exact(so.view, torch.cat(so_s, 1), lambda u_, r_: f"unit {u_} row {r_}", sl + " out scales")
    if s2 is not None:
        assert_exact(s2.view, torch.cat(s2_s, 1), lambda u_, r_: f"unit {u_} row {r_}", sl + " out2 scales")


def inst_of(c: dict) -> tuple:
    """The instantiation (kernel_check.instantiation) a run_exact case launches."""
    scaled = c.get("scaled", False) or c.get("out_blocks", False)
    fp8 = c.get("ab8", False) or scaled or c.get("out") == "e4m3" or c.get("out2") == "e4m3"
    return instantiation(act=c.get("act", 0),
                         out_dtype={"bf16": torch.bfloat16, "f32": torch.float32, "e4m3": torch.uint8}[c.get("out", "bf16")],
                         rope=c.get("rope", False), fp8=fp8, resid=c.get("resid") is not None, tile=c["tile"],
                         conv_grouped=c.get("conv_grouped", False), scaled=scaled)


# ---------------------------------------------------------------- shape grid (flat, bias only)
def _grid():
    cases = []
    for tile in (64, 128):
        for ws in (0, 1):
            st = STAGES[tile]
            for K in sorted({64, 72, 128, 200, st * 64, st * 64 + 64, 4096}):
                cases.append(dict(M=129, N=136, K=K, tile=tile, w_static=ws))
            for M in (1, 127, 128, 129, 300):
                cases.append(dict(M=M, N=72, K=128, tile=tile, w_static=ws))
            for N in (8, 64, 72, 136, 200):
                cases.append(dict(M=300, N=N, K=200, tile=tile, w_static=ws))
            for N in (4, 100, 132, 200):
                cases.append(dict(M=300, N=N, K=200, tile=tile, w_static=ws, out="f32"))
    return cases


GRID = _grid()


def _cid(c):
    return "-".join(f"{k}{v}" for k, v in c.items())


@pytest.mark.parametrize("c", GRID, ids=_cid)
def test_gemm_exact_shapes(c):
    run_exact(**c)


# ---------------------------------------------------------------- utterances, row mask, gates, residual
def _epi():
    cases = []
    for tile in (64, 128):
        for batched in (False, True):
            for rpb in (1, 127, 129, 937):
                nb = 300 if rpb == 1 else 3
                for gate in ("shared", None):
                    if gate == "shared":   # the block's out-projection / FF2: fp32 stream updated in place
                        cases.append(dict(M=rpb * nb, N=100, K=200, tile=tile, w_static=1, rpb=rpb, nb=nb, batched=batched,
                                          row_len=True, gate=gate, resid="alias", out="f32"))
                    else:                  # a separate residual without a gate, bf16 output
                        cases.append(dict(M=rpb * nb, N=136, K=200, tile=tile, w_static=0, rpb=rpb, nb=nb, batched=batched,
                                          row_len=True, gate=gate, resid="sep", out="bf16"))
    return cases


EPI = _epi()


@pytest.mark.parametrize("c", EPI, ids=_cid)
def test_gemm_exact_epilogue(c):
    run_exact(**c)


# ---------------------------------------------------------------- production-shaped launches
PROD = {
    # InputEmbedding: x W^T + hoist (fp32), plain bf16 copy for the conv position embedding, bucket rows masked
    "input_proj": dict(M=1874, N=1024, K=128, w_static=1, rpb=937, nb=2, row_len=True, resid="sep", out="f32", out2="bf16"),
    # out-projection / FF2 with the fused-LN producer: fp32 stream in place, shared gate, bf16 operand + statistics
    "ln_producer": dict(M=1874, N=1024, K=1024, w_static=1, rpb=937, nb=2, row_len=True, gate="shared", resid="alias",
                        out="f32", out2="bf16", ln_scale=True, amax=1, density=0.125),
    # FP8 out-projection: e4m3 A (the attention's e4m3 output), e4m3 W, producer with an e4m3 operand
    "fp8_out_proj": dict(M=1874, N=1024, K=1024, w_static=1, rpb=937, nb=2, row_len=True, gate="shared", resid="alias",
                         out="f32", out2="e4m3", ln_scale=True, ab8=True, density=0.125),
    # QKV without the fused LN: RoPE on q and k, q_scale on q (quarter-turn table: exact)
    "qkv_rope": dict(M=1874, N=3072, K=1024, w_static=1, rpb=937, nb=2, rope=True, amax=2),
    "fp8_qkv_rope": dict(M=1874, N=3072, K=1024, w_static=1, rpb=937, nb=2, rope=True, ab8=True, density=0.5),
    # FP8 bf16-output and e4m3-output GEMMs without activation
    "fp8_bf16_out": dict(M=300, N=200, K=256, w_static=1, ab8=True),
    "fp8_e4m3_out": dict(M=300, N=208, K=256, w_static=0, ab8=True, out="e4m3", density=0.25),
    # ln_tab GEMMs: 4 x times rows into a column slice of the wide table (n = 100: proj_out's mel columns)
    "ln_tab_mel": dict(M=32, N=100, K=1024, w_static=1, out="f32", pad_cols=1000),
    "ln_tab_qkv": dict(M=32, N=3072, K=1024, w_static=1, out="f32", pad_cols=4096),
}


@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("name", list(PROD))
def test_gemm_exact_production(name, tile):
    run_exact(tile=tile, **PROD[name])


# ---------------------------------------------------------------- UNetT (E2TTS_Base) launches, unett.cu
# D 1024, F 4096, BU = 2 utterances of N1 = 938 rows (937 frames and the time row); the UNetT's row-wise GEMMs run
# flat tiles, rows_per_batch only where RoPE positions or the row mask need it.  The skip slot of a layer is [R1, 2D]:
# the pushed x (right half, also the QKV operand) beside the skip_proj operand (left half).
_D, _FF, _N1 = 1024, 4096, 938
UNETT = {
    # QKV of RMSNorm(x): A the right half of a slot (lda 2D), RoPE on the leading head of q and of k, q scaled
    "unett_qkv": dict(M=2 * _N1, N=3 * _D, K=_D, w_static=1, rpb=_N1, nb=2, a_slot=True, ln_rms=True, rope=True,
                      rope_cols=64, rope_col2=_D, q_cols=_D, amax=2),
    # QKV of a second-half layer: A is skip_proj's bf16 output (lda = D)
    "unett_qkv_after_skip": dict(M=2 * _N1, N=3 * _D, K=_D, w_static=1, rpb=_N1, nb=2, ln_rms=True, rope=True,
                                 rope_cols=64, rope_col2=_D, q_cols=_D, amax=2, seed=1),
    # out-projection: x updated in place, rows beyond seq_len1 masked, bf16 copy + statistics without ln_scale
    "unett_out_proj": dict(M=2 * _N1, N=_D, K=_D, w_static=1, rpb=_N1, nb=2, row_len=True, resid="alias", out="f32",
                           out2="bf16", ln_stats=True, amax=1, density=0.125),
    # the same without seq_len1 (one utterance, or a batch without padding): no row mask
    "unett_out_proj_unmasked": dict(M=2 * _N1, N=_D, K=_D, w_static=1, rpb=_N1, nb=2, resid="alias", out="f32",
                                    out2="bf16", ln_stats=True, amax=1, density=0.125, seed=3),
    # FF1 of RMSNorm(x) with GELU-tanh
    "unett_ff1": dict(M=2 * _N1, N=_FF, K=_D, w_static=1, ln_rms=True, act=1, amax=2),
    # FF2 of a first-half layer: x in place, its bf16 copy pushed into the right half of the next slot with statistics
    "unett_ff2_push": dict(M=2 * _N1, N=_D, K=_FF, w_static=1, resid="alias", out="f32", out2="bf16", out2_slot="right",
                           ln_stats=True, amax=1, density=0.125),
    # FF2 of a second-half layer: the bf16 copy beside its skip (left half), no statistics (skip_proj comes first)
    "unett_ff2_skip": dict(M=2 * _N1, N=_D, K=_FF, w_static=1, resid="alias", out="f32", out2="bf16", out2_slot="left",
                           amax=1, density=0.125),
    # FF2 of the last layer: the bf16 copy and statistics for norm_out (ldo2 = D)
    "unett_ff2_last": dict(M=2 * _N1, N=_D, K=_FF, w_static=1, resid="alias", out="f32", out2="bf16", ln_stats=True,
                           amax=1, density=0.125, seed=2),
    # skip_proj([x | skip]): k = 2D over the whole slot, no bias, fp32 x + bf16 copy + statistics
    "unett_skip_proj": dict(M=2 * _N1, N=_D, K=2 * _D, w_static=1, bias=False, out="f32", out2="bf16", ln_stats=True,
                            amax=1, density=0.125),
    # proj_out(RMSNorm(x)): the 100 mel columns in fp32
    "unett_proj_out": dict(M=2 * _N1, N=100, K=_D, w_static=1, ln_rms=True, out="f32"),
}


@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("name", list(UNETT))
def test_gemm_exact_unett(name, tile):
    run_exact(tile=tile, **UNETT[name])


# ---------------------------------------------------------------- BigVGAN launches, bigvgan.cu f5_bigvgan_decode
# The released config (bigvgan_v2_24khz_100band_256x): C0 = 1536, upsampling (kernel, rate) (8, 4) twice then (4, 2)
# four times, resblock kernels 3 / 7 / 11 with dilations 1 / 3 / 5.  Every convolution is an implicit conv over B = 3
# batched utterances; T in BIGVGAN_T crosses the 128-row tile edges and sits below the taps' reach (k = 11, d = 5 reads
# 25 frames each side; decode at 6 mel frames runs stage 0 at T = 24).
BIGVGAN_T = (1, 2, 24, 127, 128, 129, 300)
BIGVGAN_C = (768, 384, 192, 96, 48, 24)


def _bigvgan_cases():
    from f5_tts_mlx_b200.bigvgan import polyphase_taps
    cases = {"conv_pre": dict(N=1536, K=128, conv_taps=7, conv_pad=3)}          # over the mel padded to 128, bf16 out
    for cin, k, u in ((1536, 8, 4), (768, 8, 4), (384, 4, 2), (192, 4, 2), (96, 4, 2), (48, 4, 2)):
        taps, pad = polyphase_taps(k, u)
        cases[f"ups_c{cin}_k{k}_u{u}"] = dict(N=u * (cin // 2), K=cin, conv_taps=taps, conv_pad=pad, out="f32")
    for c in BIGVGAN_C:
        for k in (3, 7, 11):
            for d in (1, 3, 5):
                cases[f"conv1_c{c}_k{k}_d{d}"] = dict(N=c, K=c, conv_taps=k, conv_pad=(k * d - d) // 2, conv_dilation=d,
                                                      out="f32")
            for r in ("sep", "alias"):   # conv2: the stage input as residual (m = 0), then the stream in place
                cases[f"conv2_c{c}_k{k}_{r}"] = dict(N=c, K=c, conv_taps=k, conv_pad=(k - 1) // 2, out="f32", resid=r)
    return cases


BIGVGAN = _bigvgan_cases()


@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("name", list(BIGVGAN))
def test_gemm_exact_bigvgan(name, tile):
    for T in BIGVGAN_T:
        run_exact(M=3 * T, tile=tile, w_static=1, rpb=T, nb=3, batched=True, seed=T, **BIGVGAN[name])


@pytest.mark.parametrize("tile", [64, 128])
def test_gemm_exact_bigvgan_last_stage_waves(tile):
    """The last stage's dilated conv (C = 24, k = 11, d = 5) over two utterances of 25 600 frames: 400 row tiles, so
    every CTA of a 132-SM H100 walks at least three of them."""
    run_exact(M=2 * 25600, tile=tile, w_static=1, rpb=25600, nb=2, batched=True, **BIGVGAN["conv1_c24_k11_d5"])


def test_gemm_exact_modulation_table():
    """All AdaLN linears of every solver time as one GEMM: M = number of times, N = depth * 6 D + 2 D, 128 tiles."""
    run_exact(M=33, N=22 * 6 * 1024 + 2 * 1024, K=1024, tile=128, w_static=1, out="f32", amax=2)


@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("ws", [0, 1])
def test_conv7_vocos_embed_exact(tile, ws):
    """Vocos embed: Conv1d(100 -> D, k=7, pad 3) as an implicit GEMM over 128-channel rows, channels 100..127 zero."""
    from f5_tts_mlx_b200 import ops
    B, NF, D = 2, 300, 512
    x = ints((B * NF, 128), 4, 11)
    x[:, 100:] = 0
    wt = ints((D, 100, 7), 4, 12)
    wp = torch.zeros(D, 7, 128, device=DEV, dtype=torch.bfloat16)
    wp[:, :, :100] = wt.permute(0, 2, 1)
    wp = wp.reshape(D, 7 * 128)
    bias = ints((D,), 8, 13, dtype=torch.float32)
    g = Guarded(B * NF, D, torch.float32, DEV)
    ops.gemm(x, wp, g.view, n=D, k=128, bias=bias, rows_per_batch=NF, num_batches=B, batched_tiles=True,
             conv_taps=7, conv_pad=3, tile_n=tile, w_static=bool(ws))
    ref = F.conv1d(x.double().view(B, NF, 128)[..., :100].transpose(1, 2), wt.double(), bias.double(), padding=3)
    assert_exact(g.view, round_to(ref.transpose(1, 2).reshape(B * NF, D), torch.float32), gemm_tiles(tile, NF, True), "conv7")
    g.check("conv7 guard")


@pytest.mark.parametrize("ws", [0, 1])
@pytest.mark.parametrize("B,NF", [(2, 200), (3, 129), (1, 1)])
def test_grouped_conv31_exact(B, NF, ws):
    """The conv position embedding's grouped Conv1d(k=31, pad 15, 64 channels per group), no activation."""
    from f5_tts_mlx_b200 import ops
    Cc = 256
    x = ints((B * NF, Cc), 4, 21)
    wt = ints((Cc, 64, 31), 2, 22)
    wp = wt.permute(0, 2, 1).reshape(Cc, 31 * 64).contiguous()
    bias = ints((Cc,), 8, 23, dtype=torch.float32)
    g = Guarded(B * NF, Cc, torch.bfloat16, DEV)
    ops.gemm(x, wp, g.view, n=Cc, k=64, bias=bias, rows_per_batch=NF, num_batches=B, batched_tiles=True,
             conv_taps=31, conv_pad=15, conv_grouped=True, w_static=bool(ws))
    ref = F.conv1d(x.double().view(B, NF, Cc).transpose(1, 2), wt.double(), bias.double(), padding=15, groups=Cc // 64)
    assert_exact(g.view, round_to(ref.transpose(1, 2).reshape(B * NF, Cc), torch.bfloat16), gemm_tiles(64, NF, True), "conv31")
    g.check("conv31 guard")


def test_fp8_block_promotion_exact():
    """FP8 mode adds every 128-product k-block's e4m3 wgmma partial to an fp32 accumulator on the CUDA cores.

    K = 4096: blocks 0..15 contribute exactly +1024 each (sum |products| = 2^10, exact even in a short accumulator),
    so the running total reaches 2^14; blocks 16..31 each contribute one product of +-1.  The exact result
    2^14 + (sum of sixteen +-1) needs 15 significant bits.  The kernel must be bitwise exact.  The same product through
    cuBLAS with fast accumulation (one accumulator for the whole K) is printed to show that the input discriminates a
    kernel without the promotion: on an H100 80GB HBM3 (700 W limit) it was off by up to 6."""
    from f5_tts_mlx_b200 import ops
    M, N, K = 256, 256, 4096
    A = torch.zeros(M, K, device=DEV)
    W = torch.zeros(N, K, device=DEV)
    A[:, : 16 * 128] = 8.0
    W[:, : 16 * 128] = 1.0
    m = torch.arange(M, device=DEV)
    n = torch.arange(N, device=DEV)
    for b in range(16, 32):
        j = 128 * b + (m + b) % 128
        A[m, j] = 1.0
        W[:, 128 * b:128 * b + 128] = torch.where(((n[:, None] * 7 + torch.arange(128, device=DEV)[None] + b) % 3) == 0, 1.0, -1.0)
    A8, W8 = A.to(F8), W.to(F8)
    ref = A8.float().double() @ W8.float().double().T
    assert ((ref - 16384).abs() <= 16).all() and (ref % 2 == 0).all()
    g = Guarded(M, N, torch.float32, DEV)
    ops.gemm(A8, W8, g.view, ab_fp8=True, acc_scale=1.0, tile_n=128, w_static=True)
    assert_exact(g.view, round_to(ref, torch.float32), gemm_tiles(128), "fp8 promotion")
    g.check("fp8 promotion guard")
    one = torch.ones((), device=DEV)
    try:
        fast = torch._scaled_mm(A8, W8.T, scale_a=one, scale_b=one, out_dtype=torch.float32, use_fast_accum=True)
    except RuntimeError as e:   # the reference library's FP8 entry point is not part of what is tested here
        print(f"cuBLAS FP8 fast accumulation unavailable: {e}")
        return
    err = (fast.double() - ref).abs().max().item()
    print(f"cuBLAS FP8 fast accumulation on the promotion input: max |err| = {err} (exact: {err == 0})")


def _declared():
    table = [inst_of(c) for c in GRID + EPI]
    for c in list(PROD.values()) + list(UNETT.values()) + list(BIGVGAN.values()):
        table += [inst_of(dict(c, tile=t)) for t in (64, 128)]
    table += [inst_of(dict(out="f32", tile=128))]                              # modulation table
    table += [inst_of(dict(out="f32", tile=t)) for t in (64, 128)]             # conv7
    table += [instantiation(tile=64, conv_grouped=True)]                       # conv31
    table += [inst_of(dict(out="f32", ab8=True, tile=128))]                    # fp8 promotion
    return sorted(set(table))


INSTANTIATIONS = _declared()


# ---------------------------------------------------------------- attention
def _attn_call(qkv, out, B, N, H, kv_len, fp8=False, scale_out=None):
    """f5_attention_fwd, f5_attention_fwd_e4m3 (fp8), or f5_attention_fwd_e4m3_scaled (scale_out [H, B N] given)."""
    from f5_tts_mlx_b200 import _lib
    lib = _lib.load()
    args = (qkv.data_ptr(), qkv.stride(0), out.data_ptr(), out.stride(0), B, N, H, 64,
            kv_len.data_ptr() if kv_len is not None else None)
    stream = torch.cuda.current_stream().cuda_stream
    if scale_out is not None:
        _lib.check(lib.f5_attention_fwd_e4m3_scaled(*args, scale_out.data_ptr(), stream))
    else:
        _lib.check((lib.f5_attention_fwd_e4m3 if fp8 else lib.f5_attention_fwd)(*args, stream))
    torch.cuda.synchronize()


def _qkv_buffer(B, N, H):
    """[B N, 3 D] view of a wider buffer (ld_qkv = 3 D + 64)."""
    D = H * 64
    return torch.zeros(B * N, 3 * D + 64, device=DEV, dtype=torch.bfloat16)[:, :3 * D]


def assert_ulps(got, want, mant_bits, locate, what, n=1):
    """|got - want| <= n units in the last place of max(|got|, |want|) (mant_bits stored mantissa bits)."""
    g, w = got.double().reshape(got.shape[0], -1), want.double().reshape(got.shape[0], -1)
    mag = torch.maximum(g.abs(), w.abs())
    ulp = torch.where(mag > 0, torch.exp2(torch.floor(torch.log2(mag.clamp_min(1e-300))) - mant_bits), torch.zeros_like(mag))
    bad = ~((g - w).abs() <= n * ulp)
    if bad.any():
        r, c = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} elements off by more than {n} ulp; first at {locate(r, c)}: "
                             f"got {g[r, c].item()} want {w[r, c].item()}")


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("N", [129, 300, 937])
def test_attention_uniform_mean(N, fp8):
    """Q = 0: every output row is the mean of V over the valid keys.  Keys and values at and beyond kv_len are +-2^14
    (finite: 0 * NaN would be NaN even with a correct mask).  bf16: within 1 ulp of the float64 mean (the kernel
    multiplies by 1 / l); e4m3: V is constant per column over the valid keys, so the mean is exact."""
    kvs = [1, 2, 127, 128, 129, 255, 256, N]
    B, H = len(kvs), 2
    D = H * 64
    kv = torch.tensor(kvs, dtype=torch.int32, device=DEV)
    kv_eff = kv.clamp(max=N).long()
    qkv = _qkv_buffer(B, N, H)
    pos = torch.arange(N, device=DEV).repeat(B)
    valid = (pos < kv_eff.repeat_interleave(N))[:, None]
    big = (2.0 ** 14) * (1 - 2 * ((torch.arange(B * N, device=DEV)[:, None] + torch.arange(D, device=DEV)[None]) % 2)).float()
    if fp8:
        vals = torch.tensor([0.5, -1.0, 1.5, -2.0, 0.25, 3.0], device=DEV)
        v_valid = vals[torch.arange(D, device=DEV) % 6][None].expand(B * N, D)
    else:
        v_valid = ints((B * N, D), 16, 31, dtype=torch.float32) / 4
    qkv[:, D:2 * D] = torch.where(valid, ints((B * N, D), 3, 32, dtype=torch.float32), big).bfloat16()
    qkv[:, 2 * D:] = torch.where(valid, v_valid, big).bfloat16()
    g = Guarded(B * N, D, torch.uint8 if fp8 else torch.bfloat16, DEV)
    _attn_call(qkv, g.view, B, N, H, kv, fp8)
    v = qkv[:, 2 * D:].double().view(B, N, D)
    msk = valid.view(B, N, 1).double()
    mean = (v * msk).sum(1) / kv_eff[:, None].double()                       # B, D
    want = mean[:, None, :].expand(B, N, D).reshape(B * N, D)
    loc = attn_tiles(N)
    if fp8:
        assert_exact(g.view, round_to(want, torch.uint8), loc, "uniform attention e4m3")
    else:
        assert_ulps(g.view, want, 7, loc, "uniform attention")
    g.check("uniform attention guard")


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("hot", ["first", "127", "128", "last", "later_mid"])
def test_attention_one_hot_key(hot, fp8):
    """One key per (batch, head) has logit 64, every other valid key 0, so every query's output is V[hot] (the other
    weights are below e^-64).  Keys beyond kv_len have logit 128: a leak would dominate.  Exact in bf16 and e4m3."""
    B, N, H = 2, 937, 3
    D = H * 64
    kv = torch.tensor([937, 700], dtype=torch.int32, device=DEV)
    qkv = _qkv_buffer(B, N, H)
    qkv[:, :D] = 1.0
    vals = torch.tensor([1.0, -1.0, 1.5, -1.5, 2.0, -2.0, 3.0, -3.0], device=DEV)
    g0 = torch.Generator(device=DEV).manual_seed(41)
    qkv[:, 2 * D:] = vals[torch.randint(0, 8, (B * N, D), generator=g0, device=DEV)].bfloat16()
    kk = qkv[:, D:2 * D].view(B, N, H, 64)
    want = torch.empty(B, N, H, 64, device=DEV, dtype=torch.float64)
    vv = qkv[:, 2 * D:].view(B, N, H, 64)
    for b in range(B):
        L = int(kv[b])
        kk[b, L:] = 2.0
        for h in range(H):
            idx = {"first": 0, "127": 127, "128": 128, "last": L - 1, "later_mid": 128 * (2 + h) + 64}[hot]
            kk[b, idx, h] = 1.0
            want[b, :, h] = vv[b, idx, h].double()
    g = Guarded(B * N, D, torch.uint8 if fp8 else torch.bfloat16, DEV)
    _attn_call(qkv, g.view, B, N, H, kv, fp8)
    want = want.reshape(B * N, D)
    assert_exact(g.view, round_to(want, torch.uint8 if fp8 else torch.bfloat16), attn_tiles(N), f"one-hot {hot}")
    g.check("one-hot guard")
