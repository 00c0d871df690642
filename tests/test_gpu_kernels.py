"""-m gpu: per-kernel parity of the C-ABI entry points against a float64 torch restatement of the same op on the same
(bf16 / e4m3) operands.  The GEMM and attention checks are element-wise against bounds derived in kernel_check.py
(fp32 accumulation, the approximate instructions of the epilogue, the output rounding) and name the tile of the worst
element; outputs land in NaN-filled guard buffers.  The LayerNorm / GRN kernels keep relative-norm checks
(4e-3 = 2^-8: bf16 output rounding)."""
import math

import pytest
import torch
import torch.nn.functional as F

from kernel_check import (U32, Guarded, act_bound, act_ref, assert_within, attention_bound, attention_ref, attn_tiles,
                          e4m3, gemm_acc_bound, gemm_acc_bound_fp8, gemm_tiles, instantiation, out_bound, rope_bound,
                          rope_ref)

pytestmark = pytest.mark.gpu
dev = "cuda"
TILES = [64, 128]
INSTANTIATIONS = []      # (ACT, OUT_BF16, ROPE, FP8, RESID, BN) of every GEMM case below


def _declare(tiles=TILES, **kw):
    INSTANTIATIONS.extend(instantiation(tile=t, **kw) for t in tiles)


@pytest.fixture(autouse=True)
def _strict():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dev)


def rel(a, b):
    return ((a.float() - b).norm() / (b.norm() + 1e-30)).item()


def lin(a, w, bias=None, scale=1.0, fp8=False):
    """float64 a w^T * scale + bias and its bound (accumulation + the epilogue's fma)."""
    v = (a.float().double() @ w.float().double().T) * scale
    if bias is not None:
        v = v + bias.double()
    b = (gemm_acc_bound_fp8 if fp8 else gemm_acc_bound)(a, w, scale) + U32 * v.abs()
    return v, b


_declare(out_dtype=torch.float32)


@pytest.mark.parametrize("M,N,K,tile", [(300, 256, 128, 0), (128, 128, 64, 128), (130, 72, 200, 64), (1, 128, 64, 0),
                                        (1874, 1024, 1024, 0), (257, 100, 1024, 0)])
def test_gemm_plain_fp32(M, N, K, tile):
    from f5_tts_mlx_b200 import ops
    a = rnd(M, K).bfloat16(); w = rnd(N, K, scale=K ** -0.5).bfloat16(); bias = rnd(N)
    g = Guarded(M, N, torch.float32, dev)
    ops.gemm(a, w, g.view, bias=bias, tile_n=tile)
    v, b = lin(a, w, bias)
    assert_within(g.view, v, out_bound(v, b, torch.float32), gemm_tiles(tile or 64), f"plain fp32 tile {tile}")
    g.check("plain fp32 guard")


_declare(rope=True)


def test_gemm_qkv_rope_epilogue():
    from f5_tts_mlx_b200 import ops
    from f5_tts_mlx_b200.dit import rope_table
    B, NF, D = 2, 937, 1024
    M = B * NF
    a = rnd(M, D).bfloat16(); w = rnd(3 * D, D, scale=D ** -0.5).bfloat16(); bias = rnd(3 * D)
    rope = rope_table(NF).to(dev)
    v, b = lin(a, w, bias)
    pos = torch.arange(M, device=dev) % NF
    ref, b = rope_ref(v, rope, pos, 2 * D), rope_bound(v, b, rope, pos, 2 * D)
    ref[:, :D] *= 0.125; b[:, :D] *= 0.125
    for tile in TILES:
        g = Guarded(M, 3 * D, torch.bfloat16, dev)
        ops.gemm(a, w, g.view, bias=bias, rope=rope, rope_cols=2 * D, q_scale=0.125, q_cols=D, rows_per_batch=NF,
                 num_batches=B, tile_n=tile, w_static=True)
        assert_within(g.view, ref, out_bound(ref, b, torch.bfloat16), gemm_tiles(tile), f"qkv rope tile {tile}")
        g.check("qkv rope guard")


_declare(out_dtype=torch.float32, resid=True)


def test_gemm_shared_gate_mask_residual_inplace():
    """The out-projection / FF2 form: x = resid + gate * (a W^T + bias) in place, with one [D] gate for every utterance
    and the rows past each utterance's length masked."""
    for tile in TILES:
        _shared_gate_mask_residual_inplace(tile)


def _shared_gate_mask_residual_inplace(tile):
    from f5_tts_mlx_b200 import ops
    B, NF, D = 2, 937, 1024
    M = B * NF
    a = rnd(M, 2048).bfloat16(); w = rnd(D, 2048, scale=2048 ** -0.5).bfloat16(); bias = rnd(D)
    gate = rnd(6 * D); x0 = rnd(M, D)
    g = Guarded(M, D, torch.float32, dev)
    g.view.copy_(x0)
    lens = torch.tensor([937, 700], dtype=torch.int32, device=dev)
    ops.gemm(a, w, g.view, bias=bias, resid=g.view, gate=gate[2 * D:3 * D], row_len=lens, rows_per_batch=NF,
             num_batches=B, tile_n=tile)
    v, b = lin(a, w, bias)
    valid = (torch.arange(M, device=dev) % NF < lens.repeat_interleave(NF))[:, None].double()
    gm = gate[2 * D:3 * D].double()             # one gate vector shared by all utterances, as in the DiT
    ref = x0.double() + gm * v * valid
    b = gm.abs() * b * valid + 2 * U32 * ref.abs()           # gate product and residual add (one FMA)
    assert_within(g.view, ref, out_bound(ref, b, torch.float32), gemm_tiles(tile), f"gate/mask/resid tile {tile}")
    g.check("gate/mask/resid guard")


for _act in (1, 2, 3):
    _declare(act=_act)


@pytest.mark.parametrize("act,fn", [(1, lambda v: F.gelu(v, approximate="tanh")), (2, F.gelu), (3, F.mish)])
def test_gemm_activations(act, fn):
    from f5_tts_mlx_b200 import ops
    a = rnd(500, 512).bfloat16(); w = rnd(1024, 512, scale=512 ** -0.5).bfloat16(); bias = rnd(1024)
    v, b = lin(a, w, bias)
    ref = fn(v)
    bd = out_bound(ref, act_bound(v, b, act), torch.bfloat16)
    for tile in TILES:
        g = Guarded(500, 1024, torch.bfloat16, dev)
        ops.gemm(a, w, g.view, bias=bias, act=act, tile_n=tile)
        assert_within(g.view, ref, bd, gemm_tiles(tile), f"act {act} tile {tile}")
        g.check("activation guard")


for _fp8 in (False, True):
    _declare(act=1, resid=True, fp8=_fp8)


@pytest.mark.parametrize("tile", TILES)
@pytest.mark.parametrize("fp8", [False, True])
def test_gemm_gelu_with_residual(fp8, tile):
    """GELU-tanh followed by a residual add (the residual-carrying GELU instantiation), bf16 or e4m3 operands."""
    from f5_tts_mlx_b200 import ops
    M, N, K = 300, 256, 256
    if fp8:
        a = e4m3(rnd(M, K) * 1.5); wf = rnd(N, K, scale=K ** -0.5); sc = float(wf.abs().max()) / 448.0; w = e4m3(wf / sc)
    else:
        a = rnd(M, K).bfloat16(); w = rnd(N, K, scale=K ** -0.5).bfloat16(); sc = 1.0
    bias = rnd(N); r = rnd(M, N)
    g = Guarded(M, N, torch.bfloat16, dev)
    ops.gemm(a, w, g.view, bias=bias, act=1, resid=r, ab_fp8=fp8, acc_scale=sc, tile_n=tile)
    v, b = lin(a, w, bias, sc, fp8)
    ref = act_ref(v, 1) + r.double()
    b = act_bound(v, b, 1) + U32 * ref.abs()
    assert_within(g.view, ref, out_bound(ref, b, torch.bfloat16), gemm_tiles(tile), f"gelu+resid fp8={fp8} tile {tile}")
    g.check("gelu+resid guard")


def _conv31_ref(x, wt, bias, B, N, C):
    xs = x.double().view(B, N, C).transpose(1, 2)
    v = F.conv1d(xs, wt.double(), bias.double(), padding=15, groups=C // 64).transpose(1, 2).reshape(B * N, C)
    babs = F.conv1d(xs.abs(), wt.double().abs(), None, padding=15, groups=C // 64).transpose(1, 2).reshape(B * N, C)
    return v, 2 * U32 * (31 * 64 + 1) * babs + U32 * v.abs()


_declare(tiles=[64], act=3, conv_grouped=True)


@pytest.mark.parametrize("B,N,C", [(2, 937, 1024), (1, 200, 128), (3, 31, 512), (1, 1, 64)])
def test_grouped_conv31_implicit_gemm(B, N, C):
    from f5_tts_mlx_b200 import ops
    x = rnd(B * N, C).bfloat16()
    wt = rnd(C, 64, 31, scale=(64 * 31) ** -0.5).bfloat16(); bias = rnd(C)
    wp = wt.permute(0, 2, 1).reshape(C, 31 * 64).contiguous()
    g = Guarded(B * N, C, torch.bfloat16, dev)
    ops.gemm(x, wp, g.view, n=C, k=64, bias=bias, act=3, rows_per_batch=N, num_batches=B, batched_tiles=True,
             conv_taps=31, conv_pad=15, conv_grouped=True, w_static=True)
    v, b = _conv31_ref(x, wt, bias, B, N, C)
    ref = act_ref(v, 3)
    assert_within(g.view, ref, out_bound(ref, act_bound(v, b, 3), torch.bfloat16), gemm_tiles(64, N, True), "conv31 mish")
    g.check("conv31 guard")


def _producer_check(g, g2, st, x, bx, s, out2_dtype, loc, what):
    """fp32 stream x (bound bx), its second output bf16/e4m3(x (1 + s)) and the per-64-column (sum, sum of squares).
    The statistics add 64 fp32 values in four chains of 16 and combine them: at most 64u of the sum of magnitudes."""
    M, D = x.shape
    assert_within(g.view, x, out_bound(x, bx, torch.float32), loc, what + " x")
    g.check(what + " x guard")
    sc = (1 + s.double())
    t = x * sc
    assert_within(g2.view, t, out_bound(t, sc.abs() * bx + U32 * t.abs(), out2_dtype), loc, what + " out2")
    g2.check(what + " out2 guard")
    u, ub = x.view(M, D // 64, 64), bx.view(M, D // 64, 64)
    s1, s2 = u.sum(-1), (u * u).sum(-1)
    b1 = ub.sum(-1) + 64 * U32 * u.abs().sum(-1)
    b2 = (2 * u.abs() * ub + ub * ub).sum(-1) + 66 * U32 * s2
    stv = st.view.view(M, D // 64, 2)
    unit = lambda r, c: f"row {r} unit {c}"
    assert_within(stv[..., 0], s1, b1, unit, what + " unit sums")
    assert_within(stv[..., 1], s2, b2, unit, what + " unit sums of squares")
    st.check(what + " ln_stats guard")


_declare(out_dtype=torch.float32, resid=True)


@pytest.mark.parametrize("M,D,K,tile", [(1874, 1024, 1024, 0), (1874, 1024, 2048, 0), (300, 512, 512, 64),
                                        (700, 1024, 1024, 128), (40000, 1024, 2048, 0)])
def test_gemm_fused_ln_producer(M, D, K, tile):
    """out-proj / FF2 shape: x = resid + gate * (a W^T + bias) in fp32, plus the bf16 operand x * (1 + s) and the
    per-row unit statistics (sum, sum of squares per 64 columns) of x."""
    from f5_tts_mlx_b200 import ops
    a = rnd(M, K).bfloat16(); w = rnd(D, K, scale=K ** -0.5).bfloat16(); bias = rnd(D)
    gate = rnd(1, D); x0 = rnd(M, D) * 2 + 0.3; s = rnd(D, seed=5) * 0.3
    g = Guarded(M, D, torch.float32, dev); g.view.copy_(x0)
    g2 = Guarded(M, D, torch.bfloat16, dev)
    st = Guarded(M, D // 64 * 2, torch.float32, dev, lr=False)
    ops.gemm(a, w, g.view, bias=bias, resid=g.view, gate=gate[0], out2=g2.view, ln_scale=s,
             ln_stats=st.view.view(M, D // 64, 2), tile_n=tile, w_static=True)
    v, b = lin(a, w, bias)
    x = x0.double() + gate.double() * v
    bx = gate.double().abs() * b + U32 * x.abs()
    _producer_check(g, g2, st, x, bx, s, torch.bfloat16, gemm_tiles(tile or 64), f"ln producer tile {tile}")


def _ln_tab(scale, shift, w):
    """What f5_dit_precompute's table GEMM produces for one time: rows c1_hi, c1_lo, c2_hi, c2_lo from the bf16
    hi/lo split of (1 + scale) and shift against the bf16 weight."""
    a = 1 + scale
    ah = a.bfloat16().float(); al = (a - ah).bfloat16().float()
    bh = shift.bfloat16().float(); bl = (shift - bh).bfloat16().float()
    return torch.stack([ah @ w.float().T, al @ w.float().T, bh @ w.float().T, bl @ w.float().T]).contiguous()


def ln_consumer_ref(xt, w, stats, tab, bias, scale=1.0, fp8=False):
    """float64 restatement of the fused-LN consumer on its actual inputs: rstd (xt W^T) scale - mean rstd c1 + c2 + bias,
    mean and rstd from the unit statistics (eps = fp32 1e-6), c1 / c2 = the hi + lo table rows.  Returns (v, bound).

    Bound: the statistics are summed in fp32 over n = K / 64 units (n u of the magnitudes) and divided by K (a power of
    two); var = E[x^2] - mean^2 adds the mean's error twice and two roundings; rsqrtf is within 2 ulp, so rstd is off
    by 0.5 dvar / (var + eps) + 2^-22 relative.  mu_r = mean rstd, c1 = hi + lo and c2 + bias each round once (u).  The
    epilogue's two fmas round once each; the accumulator's own bound is scaled by rstd."""
    K = xt.shape[1]
    n = K // 64
    st = stats.double()
    s1, s2 = st[..., 0].sum(-1, keepdim=True), st[..., 1].sum(-1, keepdim=True)
    mean, ex2 = s1 / K, s2 / K
    eps = torch.tensor(1e-6, dtype=torch.float32).item()
    var = (ex2 - mean * mean).clamp_min(0)
    rstd = 1 / torch.sqrt(var + eps)
    dmean = (n + 1) * U32 * st[..., 0].abs().sum(-1, keepdim=True) / K
    dex2 = (n + 1) * U32 * st[..., 1].sum(-1, keepdim=True) / K
    dvar = dex2 + 2 * mean.abs() * dmean + 3 * U32 * (ex2 + mean * mean)
    dr = 0.5 * dvar / (var + eps) + 2.0 ** -22 + U32
    t = tab.double()
    c1 = (t[0] + t[1])[None]
    c2 = (t[2] + t[3])[None] + bias.double()[None]
    acc = (xt.float().double() @ w.float().double().T) * scale
    accb = (gemm_acc_bound_fp8 if fp8 else gemm_acc_bound)(xt, w, scale)
    mu_r = mean * rstd
    v = rstd * acc - mu_r * c1 + c2
    dmu = (dmean * rstd + mean.abs() * rstd * dr + U32 * mu_r.abs())
    inner = (-mu_r * c1 + c2)
    b = (rstd * accb + rstd * acc.abs() * (dr + U32) + dmu * c1.abs() + mu_r.abs() * U32 * c1.abs()
         + U32 * c2.abs() * 2 + U32 * inner.abs() + U32 * v.abs())
    return v, b


for _t in TILES:
    INSTANTIATIONS.extend([instantiation(rope=True, tile=_t), instantiation(act=1, tile=_t),
                           instantiation(out_dtype=torch.float32, tile=_t), instantiation(rope=True, fp8=True, tile=_t)])


@pytest.mark.parametrize("M,D,N,act,rope", [(1874, 1024, 3072, 0, True), (1874, 1024, 2048, 1, False), (937, 1024, 100, 0, False),
                                            (300, 512, 1536, 0, True), (40000, 1024, 2048, 1, False)])
def test_gemm_fused_ln_consumer(M, D, N, act, rope):
    """QKV / FF1 / proj_out shape: Linear(LayerNorm(x) * (1 + s) + b) from the producer's operand x~ = bf16(x (1+s)),
    its unit statistics and the c1/c2 table, against the float64 restatement on those inputs."""
    for tile in TILES:
        _ln_consumer_case(M, D, N, act, rope, False, tile)


def test_gemm_fused_ln_consumer_fp8_qkv():
    """The FP8 QKV: e4m3 operand x~ = e4m3(x (1+s)), e4m3 weights, fused-LN consumer, RoPE and q_scale."""
    for tile in TILES:
        _ln_consumer_case(1874, 1024, 3072, 0, True, True, tile)


def _ln_consumer_case(M, D, N, act, rope, fp8, tile):
    from f5_tts_mlx_b200 import ops
    from f5_tts_mlx_b200.dit import rope_table
    x = rnd(M, D) * 1.7 + 0.4
    s = rnd(D, seed=7) * 0.3; b = rnd(D, seed=8) * 0.5
    wf = rnd(N, D, scale=D ** -0.5); bias = rnd(N)
    w = wf.bfloat16()
    tab = _ln_tab(s, b, w)
    if fp8:
        xt = e4m3(x * (1 + s)); sc = float(wf.abs().max()) / 448.0; wk = e4m3(wf / sc)
    else:
        xt = (x * (1 + s)).bfloat16(); sc = 1.0; wk = w
    units = x.view(M, D // 64, 64)
    stats = torch.stack([units.sum(-1), (units ** 2).sum(-1)], dim=-1).contiguous()
    odt = torch.float32 if N == 100 else torch.bfloat16
    g = Guarded(M, N, odt, dev)
    kw = {}
    if rope:
        kw = dict(rope=rope_table(M).to(dev), rope_cols=2 * N // 3, q_scale=0.125, q_cols=N // 3, rows_per_batch=M, num_batches=1)
    ops.gemm(xt, wk, g.view, bias=bias, act=act, ln_in_stats=stats, ln_tab=tab, ab_fp8=fp8, acc_scale=sc, tile_n=tile,
             w_static=True, **kw)
    v, bd = ln_consumer_ref(xt, wk, stats, tab, bias, sc, fp8)
    ref, bd = act_ref(v, act), act_bound(v, bd, act)
    if rope:
        pos = torch.arange(M, device=dev)
        ref, bd = rope_ref(ref, kw["rope"], pos, 2 * N // 3), rope_bound(ref, bd, kw["rope"], pos, 2 * N // 3)
        ref[:, : N // 3] *= 0.125; bd[:, : N // 3] *= 0.125
    assert_within(g.view, ref, out_bound(ref, bd, odt), gemm_tiles(tile), f"ln consumer N={N} fp8={fp8} tile {tile}")
    g.check("ln consumer guard")


# ---------------------------------------------------------------- Mish with fp32 output (conv position embedding)
for _fp8 in (False, True):
    INSTANTIATIONS.append(instantiation(act=3, out_dtype=torch.float32, resid=True, fp8=_fp8, tile=64, conv_grouped=True))
    INSTANTIATIONS.append(instantiation(act=3, out_dtype=torch.float32, resid=True, fp8=_fp8, tile=128))


@pytest.mark.parametrize("out2_fp8", [False, True])
@pytest.mark.parametrize("conv", [True, False])
def test_mish_fp32_producer(conv, out2_fp8):
    """The conv position embedding's second conv: grouped conv31 + Mish, fp32 out = h + Mish(conv), the fused-LN
    producer's operand (bf16 or e4m3) and statistics.  conv=False runs the same epilogue after a plain GEMM at 128-wide
    tiles (the grouped convolution always runs 64-wide tiles)."""
    from f5_tts_mlx_b200 import ops
    B, NF, C = 2, 300, 512
    M = B * NF
    x = rnd(M, C, seed=3).bfloat16(); bias = rnd(C); h = rnd(M, C, seed=4); s = rnd(C, seed=5) * 0.3
    g = Guarded(M, C, torch.float32, dev)
    g2 = Guarded(M, C, torch.uint8 if out2_fp8 else torch.bfloat16, dev)
    st = Guarded(M, C // 64 * 2, torch.float32, dev, lr=False)
    kw = dict(bias=bias, act=3, resid=h, out2=g2.view, out2_fp8=out2_fp8, ln_scale=s, ln_stats=st.view.view(M, C // 64, 2),
              w_static=True)
    if conv:
        wt = rnd(C, 64, 31, scale=(64 * 31) ** -0.5).bfloat16()
        wp = wt.permute(0, 2, 1).reshape(C, 31 * 64).contiguous()
        ops.gemm(x, wp, g.view, n=C, k=64, rows_per_batch=NF, num_batches=B, batched_tiles=True, conv_taps=31,
                 conv_pad=15, conv_grouped=True, **kw)
        v, b = _conv31_ref(x, wt, bias, B, NF, C)
        tile = 64
    else:
        w = rnd(C, C, scale=C ** -0.5).bfloat16()
        ops.gemm(x, w, g.view, tile_n=128, **kw)
        v, b = lin(x, w, bias)
        tile = 128
    xr = act_ref(v, 3) + h.double()
    bx = act_bound(v, b, 3) + U32 * xr.abs()
    _producer_check(g, g2, st, xr, bx, s, torch.uint8 if out2_fp8 else torch.bfloat16, gemm_tiles(tile, NF, conv),
                    f"mish fp32 conv={conv} fp8={out2_fp8}")


# ---------------------------------------------------------------- attention
def _attn(B, N, H, kv_len=None, scale_in=1.0, seed=0, fp8=False, qkv=None):
    from f5_tts_mlx_b200 import _lib
    D = H * 64
    if qkv is None:
        qkv = rnd(B * N, 3 * D, scale=scale_in, seed=seed).bfloat16()
    g = Guarded(B * N, D, torch.uint8 if fp8 else torch.bfloat16, dev)
    kl = torch.tensor(kv_len, dtype=torch.int32, device=dev) if kv_len is not None else None
    fn = _lib.load().f5_attention_fwd_e4m3 if fp8 else _lib.load().f5_attention_fwd
    _lib.check(fn(qkv.data_ptr(), qkv.stride(0), g.view.data_ptr(), g.view.stride(0), B, N, H, 64,
                  kl.data_ptr() if kl is not None else None, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    g.check("attention guard")
    return g.view, qkv


def check_attention(out, qkv, B, N, H, kv_len=None, fp8=False, what="", heads_per_chunk=16):
    """Element-wise against the float64 softmax, one chunk of heads at a time (N = 5625 needs 250 MB per head)."""
    D = H * 64
    q, k, v = [t.view(B, N, H, 64).permute(0, 2, 1, 3) for t in qkv.split(D, dim=1)]
    kl = torch.tensor(kv_len, device=dev) if kv_len is not None else None
    worst = 0.0
    tiles = math.ceil(N / 128)
    for h0 in range(0, H, heads_per_chunk):
        hs = slice(h0, min(H, h0 + heads_per_chunk))
        o, pv, qk = attention_ref(q[:, hs], k[:, hs], v[:, hs], kl)
        s_max = qk.max().item()
        bd = attention_bound(o, pv, qk, s_max, tiles, torch.uint8 if fp8 else torch.bfloat16)
        cols = slice(h0 * 64, hs.stop * 64)
        ref = o.permute(0, 2, 1, 3).reshape(B * N, -1)
        bd = bd.permute(0, 2, 1, 3).reshape(B * N, -1)
        loc = lambda r, c, h0=h0: attn_tiles(N)(r, c + h0 * 64)
        worst = max(worst, assert_within(out[:, cols], ref, bd, loc, f"{what} heads {hs.start}..{hs.stop - 1}"))
    return worst


@pytest.mark.parametrize("B,N,H,kv,sc", [(1, 128, 1, None, 1.0), (1, 100, 1, None, 1.0), (2, 937, 16, None, 0.35),
                                         (2, 937, 16, [937, 500], 0.35), (3, 300, 8, [300, 129, 1], 1.0),
                                         (1, 1500, 4, None, 0.5), (1, 1, 2, None, 1.0)])
def test_attention(B, N, H, kv, sc):
    out, qkv = _attn(B, N, H, kv, sc)
    check_attention(out, qkv, B, N, H, kv, what=f"attention B={B} N={N} H={H}")


@pytest.mark.parametrize("direction", ["rising", "falling"])
def test_attention_online_softmax_rescale(direction):
    """Logits that rise from key tile to key tile (the running max grows every tile, so o and l are rescaled every
    tile) or fall (never rescaled after the first), reaching about +-60."""
    B, N, H = 2, 937, 4
    D = H * 64
    qkv = torch.zeros(B * N, 3 * D, device=dev, dtype=torch.bfloat16)
    ramp = torch.linspace(-60, 60, N, device=dev) if direction == "rising" else torch.linspace(60, -60, N, device=dev)
    jitter = rnd(B * N, D, scale=0.05, seed=9)
    qkv[:, :D] = (1 / 8 + jitter).bfloat16()                              # q ~ 1/8: logit ~ 8 k
    qkv[:, D:2 * D] = (ramp.repeat(B)[:, None] / 8 + jitter).bfloat16()   # k row ~ ramp / 8 => logit ~ ramp
    qkv[:, 2 * D:] = rnd(B * N, D, seed=10).bfloat16()
    out, qkv = _attn(B, N, H, [937, 650], qkv=qkv)
    check_attention(out, qkv, B, N, H, [937, 650], what=f"rescale {direction}")


def test_attention_long_sequence_properties():
    """N = 5625 (60 s): rows of softmax sum to one -> attention of constant V returns that constant."""
    B, N, H = 1, 5625, 16
    D = H * 64
    qkv = rnd(B * N, 3 * D, scale=0.3).bfloat16()
    qkv[:, 2 * D:] = 0.5
    out, qkv = _attn(B, N, H, None, qkv=qkv)
    check_attention(out, qkv, B, N, H, what="N=5625 constant V", heads_per_chunk=2)


def test_attention_long_sequence_parity():
    """N = 5625 (60 s), B = 1, H = 16: every (head, query tile) against the float64 softmax."""
    B, N, H = 1, 5625, 16
    out, qkv = _attn(B, N, H, None, 0.3)
    check_attention(out, qkv, B, N, H, what="N=5625", heads_per_chunk=2)


@pytest.mark.parametrize("D", [512, 1024])
def test_ln_modulate(D):
    from f5_tts_mlx_b200 import _lib
    rows = 777
    x = rnd(rows, D) * 3 + 1; mod = rnd(6 * D)
    y = torch.empty(rows, D, device=dev, dtype=torch.bfloat16)
    _lib.check(_lib.load().f5_ln_modulate(x.data_ptr(), y.data_ptr(), rows, D, 0, mod[D:].data_ptr(), mod.data_ptr(), 0, 1,
                                          torch.cuda.current_stream().cuda_stream))
    ref = F.layer_norm(x, (D,), eps=1e-6) * (1 + mod[D:2 * D]) + mod[:D]
    assert rel(y, ref) < 4e-3


def test_dwconv7_ln_and_grn():
    from f5_tts_mlx_b200 import _lib
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    B, N, Cc = 2, 333, 512
    x = rnd(B, N, Cc); w = rnd(Cc, 7, scale=0.4); wb = rnd(Cc); lw = 1 + 0.1 * rnd(Cc); lb = 0.1 * rnd(Cc)
    y = torch.empty(B * N, Cc, device=dev, dtype=torch.bfloat16)
    wt = w.t().contiguous()
    _lib.check(lib.f5_dwconv7_ln(x.data_ptr(), y.data_ptr(), B, N, Cc, wt.data_ptr(), wb.data_ptr(), lw.data_ptr(),
                                 lb.data_ptr(), st))
    ref = F.conv1d(x.transpose(1, 2), w[:, None, :], wb, padding=3, groups=Cc).transpose(1, 2)
    ref = F.layer_norm(ref, (Cc,), lw, lb, eps=1e-6)
    assert rel(y, ref.reshape(B * N, Cc)) < 4e-3
    Ci = 1024
    h = rnd(B, N, Ci).bfloat16(); gamma = rnd(Ci) * 0.5; beta = rnd(Ci) * 0.5
    out = torch.empty_like(h); nx = torch.empty(B, 1 + (N + 31) // 32, Ci, device=dev)
    _lib.check(lib.f5_grn(h.data_ptr(), out.data_ptr(), nx.data_ptr(), gamma.data_ptr(), beta.data_ptr(), B, N, Ci, st))
    hf = h.float()
    Gx = hf.pow(2).sum(1, keepdim=True).sqrt()
    ref = gamma * (hf * (Gx / (Gx.mean(-1, keepdim=True) + 1e-6))) + beta + hf
    assert rel(out, ref) < 4e-3


# ---------------------------------------------------------------- FP8 mode (e4m3 operands, e4m3 wgmma)
_declare(fp8=True)


@pytest.mark.parametrize("M,N,K,tile,act", [(1874, 3072, 1024, 0, 0), (1874, 2048, 1024, 0, 1), (300, 256, 128, 0, 0),
                                             (257, 512, 256, 64, 0), (700, 1024, 1024, 128, 0), (40000, 2048, 1024, 0, 1)])
def test_gemm_fp8_operands(M, N, K, tile, act):
    """f5_gemm_args.ab_fp8: A and W as e4m3 bytes, accumulator x acc_scale + bias (+ GELU), bf16 out — against the
    float64 product of the SAME e4m3 values.  The explicit tile widths of FP8 GELU run in the chain tests below."""
    from f5_tts_mlx_b200 import ops
    a8 = e4m3(rnd(M, K) * 1.5); wf = rnd(N, K, scale=K ** -0.5); bias = rnd(N)
    sc = float(wf.abs().max()) / 448.0
    w8 = e4m3(wf / sc)
    g = Guarded(M, N, torch.bfloat16, dev)
    ops.gemm(a8, w8, g.view, bias=bias, act=act, ab_fp8=True, acc_scale=sc, tile_n=tile)
    v, b = lin(a8, w8, bias, sc, fp8=True)
    ref = act_ref(v, act)
    assert_within(g.view, ref, out_bound(ref, act_bound(v, b, act), torch.bfloat16), gemm_tiles(tile or 64),
                  f"fp8 act {act} tile {tile}")
    g.check("fp8 guard")


_declare(out_dtype=torch.float32, resid=True, fp8=True)
_declare(act=1, fp8=True)


def test_gemm_fp8_second_output_and_consumer_chain():
    for tile in TILES:
        _fp8_chain(tile)


def _fp8_chain(tile):
    """Producer writes the fused-LN operand as e4m3 (out2_fp8), an FP8-mode consumer multiplies it: the chain the
    DiT block runs in FP8 mode.  The consumer is checked on the operand and statistics the producer wrote."""
    from f5_tts_mlx_b200 import ops
    M, D, K, N = 1874, 1024, 1024, 2048
    a = rnd(M, K).bfloat16(); w = rnd(D, K, scale=K ** -0.5).bfloat16(); bias = rnd(D)
    gate = rnd(1, D); x0 = rnd(M, D) * 2 + 0.3; s = rnd(D, seed=5) * 0.3
    g = Guarded(M, D, torch.float32, dev); g.view.copy_(x0)
    g2 = Guarded(M, D, torch.uint8, dev)
    st = Guarded(M, D // 64 * 2, torch.float32, dev, lr=False)
    ops.gemm(a, w, g.view, bias=bias, resid=g.view, gate=gate[0], out2=g2.view, ln_scale=s,
             ln_stats=st.view.view(M, D // 64, 2), out2_fp8=True, tile_n=tile)
    v, b = lin(a, w, bias)
    x = x0.double() + gate.double() * v
    bx = gate.double().abs() * b + U32 * x.abs()
    _producer_check(g, g2, st, x, bx, s, torch.uint8, gemm_tiles(tile), f"fp8 producer tile {tile}")
    # consumer in FP8 mode on that operand
    b2 = rnd(D, seed=8) * 0.5
    w2f = rnd(N, D, scale=D ** -0.5); bias2 = rnd(N); sc = float(w2f.abs().max()) / 448.0
    w28 = e4m3(w2f / sc)
    tab = _ln_tab(s, b2, w2f.bfloat16())
    xt8 = g2.view.view(torch.float8_e4m3fn)
    stats = st.view.view(M, D // 64, 2)
    go = Guarded(M, N, torch.bfloat16, dev)
    ops.gemm(xt8, w28, go.view, bias=bias2, act=1, ln_in_stats=stats, ln_tab=tab, ab_fp8=True, acc_scale=sc, tile_n=tile)
    vv, bb = ln_consumer_ref(xt8, w28, stats, tab, bias2, sc, fp8=True)
    ref = act_ref(vv, 1)
    assert_within(go.view, ref, out_bound(ref, act_bound(vv, bb, 1), torch.bfloat16), gemm_tiles(tile), "fp8 consumer")
    go.check("fp8 consumer guard")


def test_gemm_fp8_primary_output_and_attention_e4m3_output():
    """FF1 in FP8 mode writes its GELU output as e4m3 (the A operand of FF2); the attention kernel writes e4m3 for the
    out-projection: both element-wise, e4m3 output rounding included in the bound."""
    from f5_tts_mlx_b200 import ops
    M, K, N = 1874, 1024, 2048
    a8 = e4m3(rnd(M, K) * 1.5); wf = rnd(N, K, scale=K ** -0.5); bias = rnd(N)
    sc = float(wf.abs().max()) / 448.0
    w8 = e4m3(wf / sc)
    v, b = lin(a8, w8, bias, sc, fp8=True)
    ref = act_ref(v, 1)
    for tile in TILES:
        g = Guarded(M, N, torch.uint8, dev)
        ops.gemm(a8, w8, g.view, bias=bias, act=1, ab_fp8=True, acc_scale=sc, out_fp8=True, tile_n=tile)
        assert_within(g.view, ref, out_bound(ref, act_bound(v, b, 1), torch.uint8), gemm_tiles(tile), f"fp8 e4m3 out tile {tile}")
        g.check("fp8 e4m3 out guard")
    B, NF, H = 2, 937, 16
    qkv = (rnd(B * NF, 3 * H * 64) * 0.5).bfloat16()
    out8, qkv = _attn(B, NF, H, [937, 600], qkv=qkv, fp8=True)
    check_attention(out8, qkv, B, NF, H, [937, 600], fp8=True, what="attention e4m3")
