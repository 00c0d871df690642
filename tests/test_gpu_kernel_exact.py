"""-m gpu: known-answer tests of the wgmma GEMM and the flash attention.

The GEMM operands are small integers (bf16) or e4m3 values from {0, +-1, +-2}; bias and residual are integers, gates
and 1 + ln_scale powers of two, q_scale = 0.125 and the RoPE table holds quarter turns only.  Every partial sum is
then an integer (or a dyadic fraction with few bits) below 2^20, so the fp32 result is exact in ANY summation order:
fp32 outputs must equal the float64 reference bitwise, bf16 / e4m3 outputs its round-to-nearest, ln_stats exactly.
Any indexing, masking, tail or ring-phase mistake is a nonzero difference, reported with its tile, row and column.
Every output is written into a NaN-filled buffer with guard rows and columns (ld > n), which must stay untouched.

INSTANTIATIONS lists the kernel instantiation (gemm.cu dispatch_epi) each GEMM case launches; a CPU test checks it
against gemm.cu so that no instantiation and tile width goes untested.
"""
import pytest
import torch
import torch.nn.functional as F

from kernel_check import Guarded, assert_exact, attn_tiles, gemm_tiles, instantiation, round_to, rope_ref

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


def run_exact(*, M, N, K, tile, w_static, out="bf16", seed=0, amax=4, density=1.0, rpb=0, nb=1, batched=False,
              row_len=False, gate=None, resid=None, out2=None, ln_scale=False, rope=False, ab8=False, pad_cols=0):
    """One GEMM launch against its float64 reference.  out: 'bf16' | 'f32' | 'e4m3'; gate: None | 'shared' (one [N]
    vector for every utterance);
    resid: None | 'alias' (resid is out itself) | 'sep'; out2: None | 'bf16' | 'e4m3'."""
    from f5_tts_mlx_b200 import ops
    odt = {"bf16": torch.bfloat16, "f32": torch.float32, "e4m3": torch.uint8}[out]
    rpb_e = rpb or M
    if ab8:
        A, W = ints((M, K), 2, seed, density, F8), ints((N, K), 2, seed + 1, density, F8)
        acc_scale = 0.5
    else:
        A, W = ints((M, K), amax, seed, density), ints((N, K), amax, seed + 1, density)
        acc_scale = 1.0
    bias = ints((N,), 8, seed + 2, dtype=torch.float32)
    rows = torch.arange(M, device=DEV)
    bidx, pos = rows // rpb_e, rows % rpb_e
    A64, W64 = A.float().double(), W.float().double()
    v = (A64 @ W64.T) * acc_scale + bias.double()
    vb = (A64.abs() @ W64.abs().T) * acc_scale + bias.double().abs()      # bounds every partial sum
    kw = dict(bias=bias, tile_n=tile, w_static=bool(w_static), ab_fp8=ab8, acc_scale=acc_scale)
    if rpb:
        kw.update(rows_per_batch=rpb, num_batches=nb, batched_tiles=batched)
    if rope:
        tab = quarter_turns(rpb_e, seed + 3)
        rc, qc = 2 * N // 3, N // 3
        v = rope_ref(v, tab, pos, rc)
        v[:, :qc] *= 0.125
        kw.update(rope=tab, rope_cols=rc, q_scale=0.125, q_cols=qc)
    if row_len:
        lens = row_lens(nb, rpb_e)
        v = torch.where((pos < lens.long()[bidx])[:, None], v, torch.zeros_like(v))
        kw.update(row_len=lens)
    g_out = Guarded(M, N, odt, DEV, pad_cols=pad_cols)
    if gate is not None:
        assert gate == "shared"
        gt = pow2((N,), seed + 4)
        gm = gt.double()[None]
        v, vb = v * gm, vb * gm.abs()
        kw.update(gate=gt)
    if resid is not None:
        r = ints((M, N), 16, seed + 5, dtype=torch.float32)
        v, vb = v + r.double(), vb + r.double().abs()
        if resid == "alias":
            assert odt == torch.float32
            g_out.view.copy_(r)
            kw.update(resid=g_out.view)
        else:
            kw.update(resid=r)
    assert (vb < EXACT_LIMIT).all(), "operands too large for an exact test"
    g2 = st = None
    if out2 is not None:
        g2 = Guarded(M, N, torch.uint8 if out2 == "e4m3" else torch.bfloat16, DEV)
        kw.update(out2=g2.view, out2_fp8=out2 == "e4m3")
        if ln_scale:
            s = pow2((N,), seed + 6).abs() - 1          # 1 + s in {0.5, 1, 2}
            st = Guarded(M, N // 64 * 2, torch.float32, DEV, lr=False)
            kw.update(ln_scale=s, ln_stats=st.view.view(M, N // 64, 2))
            want2 = v * (1 + s.double())
            assert (64 * vb.view(M, N // 64, 64).amax(-1) ** 2 < 2 ** 24).all(), "ln_stats would not be exact"
        else:
            want2 = v
    ops.gemm(A, W, g_out.view, out_fp8=out == "e4m3", **kw)
    torch.cuda.synchronize()
    loc = gemm_tiles(tile, rpb_e, batched)
    what = f"M={M} N={N} K={K} tile={tile} w_static={w_static}"
    assert_exact(g_out.view, round_to(v, odt), loc, what + " out")
    g_out.check(what + " out guard")
    if g2 is not None:
        assert_exact(g2.view, round_to(want2, g2.view.dtype), loc, what + " out2")
        g2.check(what + " out2 guard")
    if st is not None:
        u = v.view(M, N // 64, 64)
        want = torch.stack([u.sum(-1), (u * u).sum(-1)], -1).reshape(M, N // 64 * 2)
        assert_exact(st.view, round_to(want, torch.float32), lambda r, c: f"row {r} unit {c // 2}", what + " ln_stats")
        st.check(what + " ln_stats guard")


def inst_of(c: dict) -> tuple:
    return instantiation(act=0, out_dtype={"bf16": torch.bfloat16, "f32": torch.float32, "e4m3": torch.uint8}[c.get("out", "bf16")],
                         rope=c.get("rope", False), fp8=c.get("ab8", False) or c.get("out") == "e4m3" or c.get("out2") == "e4m3",
                         resid=c.get("resid") is not None, tile=c["tile"])


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
    for c in PROD.values():
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
