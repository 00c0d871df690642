"""-m gpu: per-kernel parity of the C-ABI entry points against a plain fp32 torch reference of the
same op on the same bf16-rounded operands (tolerances: fp32-output GEMMs 1e-5 rel; anything that
rounds its output to bf16 4e-3 rel = 2^-8)."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
dev = "cuda"


@pytest.fixture(autouse=True)
def _strict():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dev)


def rel(a, b):
    return ((a.float() - b).norm() / (b.norm() + 1e-30)).item()


@pytest.mark.parametrize("M,N,K,tile", [(300, 256, 128, 0), (128, 128, 64, 128), (130, 72, 200, 64), (1, 128, 64, 0),
                                        (1874, 1024, 1024, 0), (257, 100, 1024, 0)])
def test_gemm_plain_fp32(M, N, K, tile):
    from f5_tts_mlx_b200 import ops
    a = rnd(M, K).bfloat16(); w = rnd(N, K, scale=K ** -0.5).bfloat16(); bias = rnd(N)
    out = torch.full((M, N), float("nan"), device=dev)
    ops.gemm(a, w, out, bias=bias, tile_n=tile)
    assert rel(out, a.float() @ w.float().T + bias) < 1e-5


def test_gemm_qkv_rope_epilogue():
    from f5_tts_mlx_b200 import ops
    from f5_tts_mlx_b200.dit import rope_table
    B, NF, D = 2, 937, 1024
    M = B * NF
    a = rnd(M, D).bfloat16(); w = rnd(3 * D, D, scale=D ** -0.5).bfloat16(); bias = rnd(3 * D)
    rope = rope_table(NF).to(dev)
    out = torch.empty(M, 3 * D, device=dev, dtype=torch.bfloat16)
    ops.gemm(a, w, out, bias=bias, rope=rope, rope_cols=2 * D, q_scale=0.125, q_cols=D, rows_per_batch=NF, num_batches=B)
    ref = (a.float() @ w.float().T + bias).view(B, NF, 3 * D // 64, 32, 2)
    c, s = rope[None, :, None, :, 0], rope[None, :, None, :, 1]
    rot = torch.stack([ref[..., 0] * c - ref[..., 1] * s, ref[..., 1] * c + ref[..., 0] * s], dim=-1)
    ref2 = ref.clone(); ref2[:, :, : 2 * D // 64] = rot[:, :, : 2 * D // 64]
    ref2 = ref2.reshape(M, 3 * D).clone(); ref2[:, :D] *= 0.125
    assert rel(out, ref2) < 4e-3


def test_gemm_gate_mask_residual_inplace():
    from f5_tts_mlx_b200 import ops
    B, NF, D = 2, 937, 1024
    M = B * NF
    a = rnd(M, 2048).bfloat16(); w = rnd(D, 2048, scale=2048 ** -0.5).bfloat16(); bias = rnd(D)
    gate = rnd(B, 6 * D); x = rnd(M, D); x0 = x.clone()
    lens = torch.tensor([937, 700], dtype=torch.int32, device=dev)
    ops.gemm(a, w, x, bias=bias, resid=x, gate=gate[:, 2 * D:3 * D], row_len=lens, rows_per_batch=NF, num_batches=B)
    ref = (a.float() @ w.float().T + bias).view(B, NF, D)
    valid = (torch.arange(NF, device=dev)[None] < lens[:, None]).float()[..., None]
    ref = x0.view(B, NF, D) + gate[:, None, 2 * D:3 * D] * (ref * valid)
    assert rel(x, ref.view(M, D)) < 1e-5


@pytest.mark.parametrize("act,fn", [(1, lambda v: F.gelu(v, approximate="tanh")), (2, F.gelu), (3, F.mish)])
def test_gemm_activations(act, fn):
    from f5_tts_mlx_b200 import ops
    a = rnd(500, 512).bfloat16(); w = rnd(1024, 512, scale=512 ** -0.5).bfloat16(); bias = rnd(1024)
    out = torch.empty(500, 1024, device=dev, dtype=torch.bfloat16)
    ops.gemm(a, w, out, bias=bias, act=act)
    assert rel(out, fn(a.float() @ w.float().T + bias)) < 4e-3


@pytest.mark.parametrize("B,N,C", [(2, 937, 1024), (1, 200, 128), (3, 31, 512), (1, 1, 64)])
def test_grouped_conv31_implicit_gemm(B, N, C):
    from f5_tts_mlx_b200 import ops
    x = rnd(B * N, C).bfloat16()
    wt = rnd(C, 64, 31, scale=(64 * 31) ** -0.5).bfloat16(); bias = rnd(C)
    wp = wt.permute(0, 2, 1).reshape(C, 31 * 64).contiguous()
    out = torch.empty(B * N, C, device=dev, dtype=torch.bfloat16)
    ops.gemm(x, wp, out, n=C, k=64, bias=bias, act=3, rows_per_batch=N, num_batches=B, batched_tiles=True,
             conv_taps=31, conv_pad=15, conv_grouped=True)
    ref = F.mish(F.conv1d(x.float().view(B, N, C).transpose(1, 2), wt.float(), bias, padding=15, groups=C // 64))
    assert rel(out, ref.transpose(1, 2).reshape(B * N, C)) < 4e-3


def _attn(B, N, H, kv_len=None, scale_in=1.0, seed=0):
    from f5_tts_mlx_b200 import _lib
    D = H * 64
    qkv = rnd(B * N, 3 * D, scale=scale_in, seed=seed).bfloat16()
    out = torch.full((B * N, D), float("nan"), device=dev, dtype=torch.bfloat16)
    kl = torch.tensor(kv_len, dtype=torch.int32, device=dev) if kv_len is not None else None
    _lib.check(_lib.load().f5_attention_fwd(qkv.data_ptr(), 3 * D, out.data_ptr(), D, B, N, H, 64,
                                            kl.data_ptr() if kl is not None else None,
                                            torch.cuda.current_stream().cuda_stream))
    q, k, v = [t.float().view(B, N, H, 64).permute(0, 2, 1, 3) for t in qkv.split(D, dim=1)]
    s = q @ k.transpose(-1, -2)
    if kl is not None:
        m = torch.arange(N, device=dev)[None] < kl[:, None]
        s = s.masked_fill(~m[:, None, None, :], float("-inf"))
    ref = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(B * N, D)
    return out, ref


@pytest.mark.parametrize("B,N,H,kv,sc", [(1, 128, 1, None, 1.0), (1, 100, 1, None, 1.0), (2, 937, 16, None, 0.35),
                                         (2, 937, 16, [937, 500], 0.35), (3, 300, 8, [300, 129, 1], 1.0),
                                         (1, 1500, 4, None, 0.5), (1, 1, 2, None, 1.0)])
def test_attention(B, N, H, kv, sc):
    out, ref = _attn(B, N, H, kv, sc)
    assert torch.isfinite(out.float()).all()
    assert rel(out, ref) < 6e-3


def test_attention_long_sequence_properties():
    """N = 5625 (60 s): rows of softmax sum to one -> attention of constant V returns that constant."""
    from f5_tts_mlx_b200 import _lib
    B, N, H = 1, 5625, 16
    D = H * 64
    qkv = rnd(B * N, 3 * D, scale=0.3).bfloat16()
    qkv[:, 2 * D:] = 0.5
    out = torch.empty(B * N, D, device=dev, dtype=torch.bfloat16)
    _lib.check(_lib.load().f5_attention_fwd(qkv.data_ptr(), 3 * D, out.data_ptr(), D, B, N, H, 64, None,
                                            torch.cuda.current_stream().cuda_stream))
    assert (out.float() - 0.5).abs().max().item() < 4e-3


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


# ---------------- fused AdaLayerNormZero (f5_gemm_args.ln_*) ----------------
def _ln_tab(scale, shift, w):
    """What f5_dit_precompute's table GEMM produces for one time: rows c1_hi, c1_lo, c2_hi, c2_lo from the bf16
    hi/lo split of (1 + scale) and shift against the bf16 weight."""
    a = 1 + scale
    ah = a.bfloat16().float(); al = (a - ah).bfloat16().float()
    bh = shift.bfloat16().float(); bl = (shift - bh).bfloat16().float()
    return torch.stack([ah @ w.float().T, al @ w.float().T, bh @ w.float().T, bl @ w.float().T]).contiguous()


@pytest.mark.parametrize("M,D,K,variant,tile", [(1874, 1024, 1024, 1, 0), (1874, 1024, 2048, 1, 0), (300, 512, 512, 1, 64),
                                                (700, 1024, 1024, 2, 256), (40000, 1024, 2048, 0, 0)])
def test_gemm_fused_ln_producer(M, D, K, variant, tile):
    """out-proj / FF2 shape: x = resid + gate * (a W^T + bias) in fp32, plus the bf16 operand x * (1 + s) and the
    per-row unit statistics (sum, sum of squares per 64 columns) of x — all three against fp32 torch."""
    from f5_tts_mlx_b200 import ops
    a = rnd(M, K).bfloat16(); w = rnd(D, K, scale=K ** -0.5).bfloat16(); bias = rnd(D)
    gate = rnd(1, D); x = rnd(M, D) * 2 + 0.3; x0 = x.clone(); s = rnd(D, seed=5) * 0.3
    xt = torch.full((M, D), float("nan"), device=dev, dtype=torch.bfloat16)
    stats = torch.full((M, D // 64, 2), float("nan"), device=dev)
    ops.gemm(a, w, x, bias=bias, resid=x, gate=gate[0], out2=xt, ln_scale=s, ln_stats=stats, variant=variant, tile_n=tile)
    ref = x0 + gate * (a.float() @ w.float().T + bias)
    assert rel(x, ref) < 1e-5
    assert rel(xt, ref * (1 + s)) < 4e-3
    units = ref.view(M, D // 64, 64)
    assert (stats[..., 0] - units.sum(-1)).abs().max().item() < 2e-3
    assert rel(stats[..., 1], (units ** 2).sum(-1)) < 1e-5


@pytest.mark.parametrize("M,D,N,act,rope", [(1874, 1024, 3072, 0, True), (1874, 1024, 2048, 1, False), (937, 1024, 100, 0, False),
                                            (300, 512, 1536, 0, True), (40000, 1024, 2048, 1, False)])
def test_gemm_fused_ln_consumer(M, D, N, act, rope):
    """QKV / FF1 / proj_out shape: Linear(LayerNorm(x) * (1 + s) + b) from the producer's operand x~ = bf16(x (1+s)),
    its chunk statistics and the c1/c2 table, against fp32 torch on the un-normalised x."""
    from f5_tts_mlx_b200 import ops
    from f5_tts_mlx_b200.dit import rope_table
    x = rnd(M, D) * 1.7 + 0.4
    s = rnd(D, seed=7) * 0.3; b = rnd(D, seed=8) * 0.5
    w = rnd(N, D, scale=D ** -0.5).bfloat16(); bias = rnd(N)
    xt = (x * (1 + s)).bfloat16()
    units = x.view(M, D // 64, 64)
    stats = torch.stack([units.sum(-1), (units ** 2).sum(-1)], dim=-1).contiguous()
    tab = _ln_tab(s, b, w)
    f32 = N == 100
    out = torch.full((M, N), float("nan"), device=dev, dtype=torch.float32 if f32 else torch.bfloat16)
    kw = {}
    if rope:
        kw = dict(rope=rope_table(M).to(dev), rope_cols=2 * N // 3, q_scale=0.125, q_cols=N // 3, rows_per_batch=M, num_batches=1)
    ops.gemm(xt, w, out, bias=bias, act=act, ln_in_stats=stats, ln_tab=tab, **kw)
    ref = (F.layer_norm(x, (D,), eps=1e-6) * (1 + s) + b) @ w.float().T + bias
    if act == 1:
        ref = F.gelu(ref, approximate="tanh")
    if rope:
        r = ref.view(M, N // 64, 32, 2)
        c, sn = kw["rope"][:, None, :, 0], kw["rope"][:, None, :, 1]
        rot = torch.stack([r[..., 0] * c - r[..., 1] * sn, r[..., 1] * c + r[..., 0] * sn], dim=-1)
        r2 = r.clone(); r2[:, : kw["rope_cols"] // 64] = rot[:, : kw["rope_cols"] // 64]
        ref = r2.reshape(M, N).clone(); ref[:, : N // 3] *= 0.125
    # the operand is bf16(x (1+s)): its rounding error is relative to |x| (not |x - mean|); mean/std here is 0.24
    assert rel(out, ref) < 6e-3


# ---------------- FP8 mode (e4m3 operands, e4m3 wgmma) ----------------
def _e4m3(x):
    return x.clamp(-448, 448).to(torch.float8_e4m3fn)


@pytest.mark.parametrize("M,N,K,variant,tile,act", [(1874, 3072, 1024, 0, 0, 0), (1874, 2048, 1024, 0, 0, 1), (300, 256, 128, 1, 0, 0),
                                                     (257, 512, 256, 1, 64, 0), (700, 1024, 1024, 2, 256, 0), (40000, 2048, 1024, 0, 0, 1)])
def test_gemm_fp8_operands(M, N, K, variant, tile, act):
    """f5_gemm_args.ab_fp8: A and W as e4m3 bytes, fp32 accumulation, accumulator x acc_scale + bias (+ GELU), bf16 out —
    against the fp32 product of the SAME e4m3 values (exact products, so only the summation order differs)."""
    from f5_tts_mlx_b200 import ops
    a8 = _e4m3(rnd(M, K) * 1.5); wf = rnd(N, K, scale=K ** -0.5); bias = rnd(N)
    sc = float(wf.abs().max()) / 448.0
    w8 = _e4m3(wf / sc)
    out = torch.full((M, N), float("nan"), device=dev, dtype=torch.bfloat16)
    ops.gemm(a8, w8, out, bias=bias, act=act, ab_fp8=True, acc_scale=sc, variant=variant, tile_n=tile)
    ref = (a8.float() @ w8.float().T) * sc + bias
    if act == 1:
        ref = F.gelu(ref, approximate="tanh")
    assert rel(out, ref) < 4e-3


def test_gemm_fp8_second_output_and_consumer_chain():
    """Producer writes the fused-LN operand as e4m3 (out2_fp8), an FP8-mode consumer multiplies it: the chain the
    DiT block runs in FP8 mode, against fp32 torch on the same quantised values."""
    from f5_tts_mlx_b200 import ops
    M, D, K, N = 1874, 1024, 1024, 2048
    a = rnd(M, K).bfloat16(); w = rnd(D, K, scale=K ** -0.5).bfloat16(); bias = rnd(D)
    gate = rnd(1, D); x = rnd(M, D) * 2 + 0.3; x0 = x.clone(); s = rnd(D, seed=5) * 0.3
    xt8 = torch.zeros(M, D, device=dev, dtype=torch.uint8)
    stats = torch.zeros(M, D // 64, 2, device=dev)
    ops.gemm(a, w, x, bias=bias, resid=x, gate=gate[0], out2=xt8, ln_scale=s, ln_stats=stats, out2_fp8=True)
    xref = x0 + gate * (a.float() @ w.float().T + bias)
    want = _e4m3(xref * (1 + s))
    got = xt8.view(torch.float8_e4m3fn)
    assert (got.float() == want.float()).float().mean().item() > 0.995          # ties / 1-ulp fp32 differences only
    assert rel(got.float(), want.float()) < 5e-3
    # consumer in FP8 mode on that operand
    b2 = rnd(D, seed=8) * 0.5
    w2f = rnd(N, D, scale=D ** -0.5); bias2 = rnd(N); sc = float(w2f.abs().max()) / 448.0
    w28 = _e4m3(w2f / sc)
    tab = _ln_tab(s, b2, w2f.bfloat16())
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    ops.gemm(xt8, w28, out, bias=bias2, act=1, ln_in_stats=stats, ln_tab=tab, ab_fp8=True, acc_scale=sc)
    mu = xref.mean(-1, keepdim=True); rstd = torch.rsqrt(xref.var(-1, unbiased=False, keepdim=True) + 1e-6)
    acc = (got.float() @ w28.float().T) * sc
    c1 = (1 + s) @ w2f.bfloat16().float().T; c2 = b2 @ w2f.bfloat16().float().T + bias2
    ref = F.gelu(rstd * (acc - mu * c1) + c2, approximate="tanh")
    assert rel(out, ref) < 6e-3


def test_gemm_fp8_primary_output_and_attention_e4m3_output():
    """FF1 in FP8 mode writes its GELU output as e4m3 (the A operand of FF2); the attention kernel writes e4m3 for the
    out-projection: both against the e4m3 rounding of the fp32 reference."""
    from f5_tts_mlx_b200 import _lib, ops
    M, K, N = 1874, 1024, 2048
    a8 = _e4m3(rnd(M, K) * 1.5); wf = rnd(N, K, scale=K ** -0.5); bias = rnd(N)
    sc = float(wf.abs().max()) / 448.0
    w8 = _e4m3(wf / sc)
    out8 = torch.zeros(M, N, device=dev, dtype=torch.uint8)
    ops.gemm(a8, w8, out8, bias=bias, act=1, ab_fp8=True, acc_scale=sc, out_fp8=True)
    ref = F.gelu((a8.float() @ w8.float().T) * sc + bias, approximate="tanh")
    got = out8.view(torch.float8_e4m3fn).float()
    assert (got == _e4m3(ref).float()).float().mean().item() > 0.99
    assert rel(got, ref) < 4e-2                                   # e4m3 rounding of the output itself (2^-4 relative)
    # attention with e4m3 output
    B, NF, H = 2, 937, 16
    D = H * 64
    qkv = (rnd(B * NF, 3 * D) * 0.5).bfloat16()
    o16 = torch.empty(B * NF, D, device=dev, dtype=torch.bfloat16)
    o8 = torch.zeros(B * NF, D, device=dev, dtype=torch.uint8)
    lib = _lib.load(); st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.f5_attention_fwd(qkv.data_ptr(), 3 * D, o16.data_ptr(), D, B, NF, H, 64, None, st))
    _lib.check(lib.f5_attention_fwd_e4m3(qkv.data_ptr(), 3 * D, o8.data_ptr(), D, B, NF, H, 64, None, st))
    g8 = o8.view(torch.float8_e4m3fn).float()
    assert rel(g8, o16.float()) < 4e-2 and (g8 - o16.float()).abs().max().item() <= 0.07 * o16.float().abs().max().item() + 2e-3
