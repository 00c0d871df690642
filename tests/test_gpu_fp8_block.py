"""-m gpu: the block-scaled FP8 mode (DESIGN.md section 8) — the scaled GEMM on exact known answers, the block-scaled
producers bitwise against the scale rule, the scaled attention output, and the DiT in that mode against its emulation.

Exact GEMM answers: A and W hold e4m3 codes from {0, +-1, +-2} with power-of-two scales (A per (row, 64 columns), W per
output channel).  Every unit partial is an integer below 2^9, every scaled sum a multiple of 2^-6 below 2^17: fp32
represents each step exactly in any order, so fp32 outputs must equal the float64 reference bitwise."""
import pytest
import torch

import fp8_block_emul as E
from helpers import ocfg_of, rel
from kernel_check import Guarded, assert_exact, assert_within, gemm_tiles, instantiation, round_to
from oracle import f5_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
F8 = torch.float8_e4m3fn

# instantiations of dispatch_scaled (gemm.cu) these cases launch: (ACT, OUT_BF16, ROPE, FP8, RESID, BN)
INSTANTIATIONS = []


def _declare(**kw):
    for tile in (64, 128):
        INSTANTIATIONS.append(instantiation(fp8=True, tile=tile, **kw))


def _codes(rows, cols, g, density=0.5):
    v = torch.randint(-2, 3, (rows, cols), generator=g).float()
    v[torch.rand(rows, cols, generator=g) > density] = 0
    return v


def _pow2(shape, g, lo=-3, hi=3):
    return torch.pow(2.0, torch.randint(lo, hi + 1, shape, generator=g).float())


def _operands(M, N, K, g):
    a, w = _codes(M, K, g), _codes(N, K, g)
    sa = _pow2((K // 64, M), g)                     # [K/64][M] unit-major
    sw = _pow2((N,), g)
    a_deq = (a.reshape(M, K // 64, 64) * sa.T[..., None]).reshape(M, K)
    return a, w, sa, sw, a_deq.double() @ (w.double() * sw.double()[:, None]).T


_declare(out_dtype=torch.float32, resid=True)


@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("M,N,K,batched", [(300, 200, 256, False), (256, 128, 128, False), (2 * 150, 192, 384, True)])
def test_scaled_gemm_exact(tile, M, N, K, batched):
    """fp32 out = acc (per-unit A scales, per-channel W scales) + bias + residual; M / N / K tails, batched tiles that
    end mid-utterance (150 frames: the second tile of each utterance runs past it) and a row mask."""
    g = torch.Generator().manual_seed(M + N + K + tile)
    a, w, sa, sw, ref = _operands(M, N, K, g)
    bias = torch.randint(-4, 5, (N,), generator=g).float()
    resid = torch.randint(-8, 9, (M, N), generator=g).float()
    kw = {}
    want = ref + bias.double() + resid.double()
    if batched:
        rl = torch.tensor([150, 97], dtype=torch.int32)
        kw = dict(rows_per_batch=150, num_batches=2, batched_tiles=True, row_len=rl.to(DEV))
        pos = torch.arange(M) % 150
        valid = pos < rl.repeat_interleave(150)
        want = torch.where(valid[:, None], ref + bias.double(), torch.zeros_like(ref)) + resid.double()
    go = Guarded(M, N, torch.float32, DEV)
    go.view.copy_(resid)
    sab = Guarded(K // 64, M, torch.float32, DEV, lr=False)
    sab.view.copy_(sa)
    ops().gemm(a.to(F8).to(DEV), w.to(F8).to(DEV), go.view, bias=bias.to(DEV), resid=go.view, ab_fp8=True, tile_n=tile,
               a_scale=sab.view, w_scale=sw.to(DEV), w_static=True, **kw)
    assert_exact(go.view.cpu(), round_to(want, torch.float32), gemm_tiles(tile, 150, batched), "scaled gemm")
    go.check("scaled gemm guard")


def ops():
    from f5_tts_mlx_b200 import ops as _ops
    return _ops


_declare(out_dtype=torch.float32, resid=True)   # the producer form: fp32 out + block-scaled e4m3 out2


@pytest.mark.parametrize("tile", [64, 128])
def test_scaled_producer_codes_and_scales_bitwise(tile):
    """out2 = e4m3(out * (1 + s) / scale) with one power-of-two scale per (row, 64 columns): codes and scales equal the
    host rule applied to the kernel's own fp32 output, bitwise.  Large values (beyond 448) and a masked row included."""
    g = torch.Generator().manual_seed(11 + tile)
    M, N, K = 300, 256, 256
    a, w, sa, sw, ref = _operands(M, N, K, g)
    sa[:, :40] *= 64.0                                      # rows far beyond 448
    s = (torch.randn(N, generator=g) * 0.3).float()
    go, g2 = Guarded(M, N, torch.float32, DEV), Guarded(M, N, torch.uint8, DEV)
    st = Guarded(M, N // 64 * 2, torch.float32, DEV, lr=False)
    s2 = Guarded(N // 64, M, torch.float32, DEV, lr=False)
    sab = Guarded(K // 64, M, torch.float32, DEV, lr=False)
    sab.view.copy_(sa)
    rl = torch.tensor([M - 5], dtype=torch.int32, device=DEV)
    ops().gemm(a.to(F8).to(DEV), w.to(F8).to(DEV), go.view, ab_fp8=True, tile_n=tile, a_scale=sab.view,
               w_scale=sw.to(DEV), out2=g2.view, out2_fp8=True, out2_scale=s2.view, ln_scale=s.to(DEV),
               ln_stats=st.view.view(M, N // 64, 2), row_len=rl, rows_per_batch=M, num_batches=1)
    torch.cuda.synchronize()
    out = go.view.cpu()
    from f5_tts_mlx_b200.weights import quantize_e4m3_blocks
    q, sc = quantize_e4m3_blocks(out * (1 + s), 64)
    assert_exact(s2.view.cpu().T.contiguous(), sc, gemm_tiles(tile), "out2 scales")
    assert_exact(g2.view.cpu(), q, gemm_tiles(tile), "out2 codes")
    assert (s2.view.cpu()[:, M - 5:] == 1).all()            # masked rows: zero, scale 1 (no residual here)
    for gd, what in ((go, "out"), (g2, "out2"), (s2, "out2 scales"), (st, "stats")):
        gd.check(what + " guard")


_declare(act=1)                                      # FF1: GELU, block-scaled e4m3 out, no residual


@pytest.mark.parametrize("tile", [64, 128])
def test_scaled_gelu_e4m3_output(tile):
    """FF1's form: GELU output quantised per (row, 64 columns).  Each unit's largest code magnitude is in [224, 448]
    (the scale is the smallest power of two that fits), and codes * scales are within half an e4m3 ulp (relative
    2^-4) plus the GELU approximation of the float64 GELU."""
    g = torch.Generator().manual_seed(5 + tile)
    M, N, K = 260, 320, 256
    a, w, sa, sw, ref = _operands(M, N, K, g)
    bias = torch.randn(N, generator=g)
    go = Guarded(M, N, torch.uint8, DEV)
    so = Guarded(N // 64, M, torch.float32, DEV, lr=False)
    sab = Guarded(K // 64, M, torch.float32, DEV, lr=False)
    sab.view.copy_(sa)
    ops().gemm(a.to(F8).to(DEV), w.to(F8).to(DEV), go.view, bias=bias.to(DEV), act=1, ab_fp8=True, out_fp8=True,
               tile_n=tile, a_scale=sab.view, w_scale=sw.to(DEV), out_scale=so.view)
    torch.cuda.synchronize()
    codes = go.view.cpu().view(F8).float()
    sc = so.view.cpu().T
    deq = (codes.reshape(M, N // 64, 64) * sc[..., None]).reshape(M, N)
    v = ref + bias.double()
    want = 0.5 * v * (1 + torch.tanh(0.7978845608028654 * (v + 0.044715 * v ** 3)))
    amax = codes.abs().reshape(M, N // 64, 64).amax(-1)
    nz = want.abs().reshape(M, N // 64, 64).amax(-1) > 0
    assert ((amax >= 224) & (amax <= 448))[nz].all()
    bound = 2.0 ** -4 * want.abs() + 2.0 ** -9 * sc.repeat_interleave(64, 1).double() + 1e-3 * (1 + v.abs())
    assert_within(deq, want, bound, gemm_tiles(tile), "scaled gelu e4m3")
    go.check("gelu out guard"); so.check("gelu scale guard")


_declare(rope=True, scaled=True)                     # the RoPE QKV: bf16 out, no residual


@pytest.mark.parametrize("tile", [64, 128])
def test_scaled_fused_ln_consumer_exact(tile):
    """The fused-LN consumer form of the scaled epilogue, rstd * w_s[col] * acc - mu_r * c1 + c2 — what the QKV and FF1
    GEMMs of the mode compute — on an exact known answer.  The row statistics make mean and rstd powers of two (mean 2,
    variance 2^20: rstd 2^-10; mean -4, variance 2^16: rstd 2^-8; the 1e-6 of the LayerNorm is below half an ulp of
    the variance), c1 / c2 / bias are integers and A / W block-scaled codes, so every fp32 step is exact; bf16 out.
    Runs the RoPE QKV instantiation with rope_cols = q_cols = 0 (no rotation), M and N tails, NaN-guarded output."""
    from f5_tts_mlx_b200.dit import rope_table
    g = torch.Generator().manual_seed(31 + tile)
    M, N, K = 300, 192, 256
    a, w, sa, sw, _ = _operands(M, N, K, g)
    kind = torch.rand(M, generator=g) < 0.5
    mean = torch.where(kind, 2.0, -4.0).double()
    var = torch.where(kind, 2.0 ** 20, 2.0 ** 16).double()
    stats = torch.empty(M, K // 64, 2)
    stats[..., 0] = (mean * 64)[:, None].float()
    stats[..., 1] = ((var + mean * mean) * 64)[:, None].float()
    tab = torch.randint(-8, 9, (4, N + 8), generator=g).float()
    bias = torch.randint(-8, 9, (N,), generator=g).float()
    rstd = var.rsqrt()
    acc = (a.reshape(M, K // 64, 64) * sa.T[..., None]).reshape(M, K).double() @ w.double().T
    c1 = (tab[0] + tab[1])[:N].double()
    c2 = (bias + (tab[2] + tab[3])[:N]).double()
    want = rstd[:, None] * sw.double()[None] * acc - (mean * rstd)[:, None] * c1[None] + c2[None]
    go = Guarded(M, N, torch.bfloat16, DEV)
    sab = Guarded(K // 64, M, torch.float32, DEV, lr=False)
    sab.view.copy_(sa)
    ops().gemm(a.to(F8).to(DEV), w.to(F8).to(DEV), go.view, bias=bias.to(DEV), ab_fp8=True, tile_n=tile,
               a_scale=sab.view, w_scale=sw.to(DEV), ln_in_stats=stats.to(DEV), ln_tab=tab.to(DEV),
               rope=rope_table(M).to(DEV), rope_cols=0, q_scale=0.125, q_cols=0, rows_per_batch=M, num_batches=1)
    torch.cuda.synchronize()
    assert_exact(go.view.cpu(), round_to(want, torch.bfloat16), gemm_tiles(tile), "scaled fused-LN consumer")
    go.check("scaled fused-LN consumer guard")
_declare(act=3, out_dtype=torch.float32, resid=True)  # the Mish conv-position GEMM (bf16 operands, scaled out2)


@pytest.mark.parametrize("tile", [64, 128])
def test_scaled_qkv_rope_and_mish_producer(tile):
    """The remaining two epilogues of the mode: the RoPE QKV with block-scaled A and per-channel W (against the unscaled
    FP8 launch on pre-multiplied exact operands), and the Mish producer on bf16 operands with a block-scaled out2."""
    from f5_tts_mlx_b200.dit import rope_table
    from f5_tts_mlx_b200.weights import quantize_e4m3_blocks
    g = torch.Generator().manual_seed(23 + tile)
    M, D, K = 270, 256, 256
    a, w, sa, sw, ref = _operands(M, 3 * D, K, g)
    tab = rope_table(M).to(DEV)
    sab = Guarded(K // 64, M, torch.float32, DEV, lr=False)
    sab.view.copy_(sa)
    got = Guarded(M, 3 * D, torch.bfloat16, DEV)
    kw = dict(rope=tab, rope_cols=2 * D, q_scale=0.125, q_cols=D, rows_per_batch=M, num_batches=1, tile_n=tile)
    ops().gemm(a.to(F8).to(DEV), w.to(F8).to(DEV), got.view, ab_fp8=True, a_scale=sab.view, w_scale=sw.to(DEV), **kw)
    # the same product with the scales folded into exact bf16 operands, on the bf16 instantiation
    a_deq = (a.reshape(M, K // 64, 64) * sa.T[..., None]).reshape(M, K)
    want = Guarded(M, 3 * D, torch.bfloat16, DEV)
    ops().gemm(a_deq.bfloat16().to(DEV), (w * sw[:, None]).bfloat16().to(DEV), want.view, **kw)
    torch.cuda.synchronize()
    assert_exact(got.view.cpu(), want.view.cpu(), gemm_tiles(tile), "scaled rope qkv")
    got.check("qkv guard")
    # Mish, fp32 out, bf16 operands, block-scaled e4m3 out2 (bitwise against the rule on the kernel's own fp32 out)
    ab, wb = torch.randn(M, K, generator=g).bfloat16(), (torch.randn(D, K, generator=g) * K ** -0.5).bfloat16()
    s = (torch.randn(D, generator=g) * 0.3).float()
    go, g2 = Guarded(M, D, torch.float32, DEV), Guarded(M, D, torch.uint8, DEV)
    st = Guarded(M, D // 64 * 2, torch.float32, DEV, lr=False)
    s2 = Guarded(D // 64, M, torch.float32, DEV, lr=False)
    h = (torch.randn(M, D, generator=g) * 300).to(DEV)
    ops().gemm(ab.to(DEV), wb.to(DEV), go.view, act=3, resid=h, out2=g2.view, out2_fp8=True, out2_scale=s2.view,
               ln_scale=s.to(DEV), ln_stats=st.view.view(M, D // 64, 2), tile_n=tile)
    torch.cuda.synchronize()
    q, sc = quantize_e4m3_blocks(go.view.cpu() * (1 + s), 64)
    assert_exact(s2.view.cpu().T.contiguous(), sc, gemm_tiles(tile), "mish out2 scales")
    assert_exact(g2.view.cpu(), q, gemm_tiles(tile), "mish out2 codes")
    g2.check("mish out2 guard"); s2.check("mish scale guard")


def test_scaled_attention_output():
    """f5_attention_fwd_e4m3_scaled: e4m3 codes with one power-of-two scale per (row, head).  The dequantised output is
    within the bf16 output's derived bound plus half an e4m3 ulp of each row-head's scale range, and every nonzero
    row-head has its largest code magnitude in [224, 448]."""
    import ctypes as C
    from f5_tts_mlx_b200 import _lib
    from kernel_check import attention_bound, attention_ref
    B, N, H = 2, 300, 4
    D = H * 64
    g = torch.Generator().manual_seed(9)
    qkv = (torch.randn(B * N, 3 * D, generator=g) * 0.5)
    qkv[:, 2 * D:] *= torch.pow(2.0, torch.randint(-8, 9, (1, D), generator=g).float())   # wide range of V per head
    qkv = qkv.bfloat16()
    kv = torch.tensor([300, 201], dtype=torch.int32)
    out = Guarded(B * N, D, torch.uint8, DEV)
    sc = Guarded(H, B * N, torch.float32, DEV, lr=False)
    qd = qkv.to(DEV)
    _lib.check(_lib.load().f5_attention_fwd_e4m3_scaled(qd.data_ptr(), 3 * D, out.view.data_ptr(), out.view.stride(0), B, N,
                                                        H, 64, kv.to(DEV).data_ptr(), sc.view.data_ptr(),
                                                        C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    codes = out.view.cpu().view(F8).float().reshape(B * N, H, 64)
    s = sc.view.cpu().T                                              # [rows, H]
    deq = (codes * s[..., None]).reshape(B * N, D)
    split = lambda t: t.float().reshape(B, N, H, 64).permute(0, 2, 1, 3)
    q, k, v = split(qkv[:, :D]), split(qkv[:, D:2 * D]), split(qkv[:, 2 * D:])
    o, pv, qk = attention_ref(q, k, v, kv)
    flat = lambda t: t.permute(0, 2, 1, 3).reshape(B * N, D)
    bd = flat(attention_bound(o, pv, qk, qk.max().item(), 3, torch.float32)) + \
        (2.0 ** -4 * flat(o).abs() + 2.0 ** -9 * s.repeat_interleave(64, 1).double())
    from kernel_check import attn_tiles
    assert_within(deq, flat(o), bd, attn_tiles(N), "scaled attention")
    amax = codes.abs().amax(-1)
    nz = flat(o).abs().reshape(B * N, H, 64).amax(-1) > 0
    assert ((amax >= 224) & (amax <= 448))[nz].all()
    out.check("attention out guard"); sc.check("attention scale guard")


# ---------------------------------------------------------------- the DiT in block mode
def _dit(cfg, W, **kw):
    from f5_tts_mlx_b200 import DiT
    return DiT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult, mel_dim=cfg.mel_dim,
               text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim, conv_layers=cfg.conv_layers, device=DEV,
               **kw).load_weights(W)


@pytest.mark.parametrize("construction", ["random", "outlier"])
def test_block_mode_forward_within_emulated_drift(construction):
    """DiT(fp8=True, fp8_scaling="block") stays within 3x the drift of its CPU emulation (fp8_block_emul) from the fp32
    oracle, on the seeded random weights and on the outlier construction (residual rows far beyond 448)."""
    from f5_tts_mlx_b200.weights import GATE_CONFIG, random_dit_weights
    cfg = GATE_CONFIG
    W = random_dit_weights(cfg, seed=1234)
    N = 300
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1, N, 100, generator=g); cond = torch.randn(1, N, 100, generator=g) * 2 - 1
    text = torch.randint(0, 2545, (1, 60), generator=g, dtype=torch.int32)
    if construction == "outlier":
        x, cond = E.outlier_inputs(1, N)
    t = torch.tensor(0.25)
    ref = O.dit_forward(x, cond, text, t, False, False, None, W, ocfg_of(cfg))
    emu = E.dit_forward_block8(x, cond, text, t, False, False, None, W, ocfg_of(cfg))
    m = _dit(cfg, W, fp8=True, fp8_scaling="block")
    got = m(x.to(DEV), cond.to(DEV), text.to(DEV), t).cpu()
    drift, r = rel(emu, ref), rel(got, ref)
    print(f"{construction}: block-mode rel {r:.3e}, emulated drift {drift:.3e}")
    assert torch.isfinite(got).all() and r < 3 * drift, (r, drift)


def test_block_mode_sample_through_from_pretrained():
    """from_pretrained("random", fp8="block"): sample() with batch > 1 (ragged durations) and with frame bucketing."""
    from f5_tts_mlx_b200 import F5TTS
    from f5_tts_mlx_b200.pretrained import from_pretrained
    f5 = from_pretrained(F5TTS, "random", fp8="block", vocoder=False)
    assert f5.transformer.fp8_block
    g = torch.Generator().manual_seed(4)
    cond = (torch.randn(2, 120, 100, generator=g) * 2 - 1).to(DEV)
    text = torch.randint(0, 2545, (2, 40), generator=g, dtype=torch.int32)
    text[1, 30:] = -1
    out, _ = f5.sample(cond, text, torch.tensor([300, 260]), steps=4, method="euler", cfg_strength=2.0, seed=1)
    assert out.shape[0] == 2 and torch.isfinite(out).all()
    one, _ = f5.sample(cond[:1], text[:1], 250, steps=4, method="euler", cfg_strength=2.0, seed=1, frame_bucket=128)
    assert one.shape[1] == 250 and torch.isfinite(one).all()
    assert f5.last_plan.session.frames == 256 and f5.last_plan.session.a_fp8_scale is not None


def test_dit_forward_rejects_a_partly_bound_mode():
    """f5_dit_forward checks the mode its buffers and weights select instead of inferring one from whichever pointers
    are set: a partly bound fused-AdaLN, FP8 or block-scaled set is F5_ERR_INVALID naming what is missing."""
    import ctypes as C
    from f5_tts_mlx_b200 import _lib
    from f5_tts_mlx_b200.dit import DitBuffersC
    from f5_tts_mlx_b200.weights import GATE_CONFIG, DitBlockWeightsC, DitWeightsC, random_dit_weights
    cfg = GATE_CONFIG
    W = random_dit_weights(cfg, seed=1234)
    lib = _lib.load()

    def forward(model, unbind=(), unbind_block=None):
        s = model.session(1, 128, 1, False, 16, False)
        b = DitBuffersC.from_buffer_copy(s.c)
        for name in unbind:
            setattr(b, name, None)
        w = DitWeightsC.from_buffer_copy(model.packed.c_struct())
        blks = (DitBlockWeightsC * cfg.depth)(*[DitBlockWeightsC.from_buffer_copy(w.blocks[i])
                                                for i in range(cfg.depth)])
        if unbind_block is not None:
            i, names = unbind_block
            for name in names:
                setattr(blks[i], name, None)
        w.blocks = blks
        rc = lib.f5_dit_forward(C.byref(w), C.byref(b), 0, C.c_void_p(torch.cuda.current_stream().cuda_stream))
        return rc, lib.f5_last_error().decode()

    bf16, tensor, block = _dit(cfg, W), _dit(cfg, W, fp8=True), _dit(cfg, W, fp8=True, fp8_scaling="block")
    rc, msg = forward(bf16, unbind=("ln_prep",))
    assert rc == -1 and "fused AdaLN needs ln_prep" in msg, msg
    rc, msg = forward(tensor, unbind=("ln_stats", "ln_tab", "ln_prep"))
    assert rc == -1 and "FP8 needs the fused AdaLN" in msg, msg
    rc, msg = forward(tensor, unbind_block=(1, ("out_w8", "ff2_w8")))
    assert rc == -1 and "FP8 needs out_w8, ff2_w8 of blocks[1]" in msg, msg
    rc, msg = forward(block, unbind=("attn_scale",))
    assert rc == -1 and "block-scaled FP8 needs attn_scale" in msg, msg
    rc, msg = forward(block, unbind=("a_fp8",))
    assert rc == -1 and "FP8 needs a_fp8" in msg, msg
    rc, msg = forward(block, unbind=("a_fp8_scale", "attn_scale", "ff_scale"))
    assert rc == -1 and "blocks[0] has per-channel weight scales" in msg, msg
    rc, msg = forward(block, unbind_block=(0, ("ff1_ws",)))
    assert rc == -1 and "block-scaled FP8 needs ff1_ws of blocks[0]" in msg, msg
