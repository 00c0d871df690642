"""-m gpu: known-answer tests of the wgmma GEMM at launches with more output tiles than the GPU has SMs.

The production launches at batch 1 fit in about one wave of 128 x BN tiles; batched requests and the convolutions do
not.  These cases size the problem from the SM count so that every CTA of a one-CTA-per-SM launch would own 2, 3 or 8+
tiles, exactly one, or one tile more than the SMs, with ragged M / N tails, and so that an in-place residual, a fused-LN
producer and a 31-tap grouped convolution run over many waves.  Operands are small integers (run_exact of
test_gpu_kernel_exact): every output must equal the float64 reference bitwise, whatever the order in which tiles run.

WAVES holds one case per (instantiation, BN) of both dispatchers at 3 to 4 tiles per CTA (a CPU test in
test_kernel_check.py fails when an instantiation has none), and the DiT block's GEMM chain runs with programmatic
dependent launch live, eagerly and as a replayed CUDA graph.
"""
import pytest
import torch
import torch.nn.functional as F

from kernel_check import STAGES, Guarded, assert_exact, cdiv, gemm_bn, gemm_num_kb, gemm_tile_count, gemm_tiles
from test_gpu_kernel_exact import DEV, ints, round_to, run_exact

pytestmark = pytest.mark.gpu


def sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("per_sm", [2, 3, 9])
def test_many_tiles_per_sm_ragged(per_sm, tile):
    """per_sm x SMs tiles (or a few more) with a 40-column N tail and a 37-row M tail."""
    nt = 8
    N = nt * tile - 40
    mt = cdiv(per_sm * sms(), nt)
    run_exact(M=mt * 128 - 37, N=N, K=192, tile=tile, w_static=per_sm % 2, seed=per_sm)


@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("extra", [0, 1])
def test_sm_count_tiles(extra, tile):
    """Exactly SMs tiles (one column tile, SMs row tiles), then one more row tile holding a single row."""
    run_exact(M=sms() * 128 + extra, N=56, K=128, tile=tile, w_static=1, out="f32", seed=10 + extra)


@pytest.mark.parametrize("tile", [64, 128])
def test_in_place_residual_over_many_waves(tile):
    """Out-projection / FF2 form over >= 3 tiles per SM: fp32 stream updated in place (each tile reads its residual
    before any store to it), shared gate, row mask, bf16 operand and LN statistics of the next block."""
    N = 1024
    rpb = cdiv(3 * sms(), N // tile) * 64 + 5          # two utterances, each ending mid-tile
    run_exact(M=2 * rpb, N=N, K=256, tile=tile, w_static=1, rpb=rpb, nb=2, row_len=True, gate="shared",
              resid="alias", out="f32", out2="bf16", ln_scale=True, amax=1, density=0.125, seed=20)


@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("form", ["qkv_rope", "fp8_qkv_rope", "fp8_out_proj", "fp8_e4m3_out"])
def test_block_forms_over_many_waves(form, tile):
    """The block GEMMs' epilogue forms at >= 3 tiles per SM, batched rows (tiles never straddle utterances)."""
    N = {"qkv_rope": 768, "fp8_qkv_rope": 768, "fp8_out_proj": 512, "fp8_e4m3_out": 512}[form]
    rt = cdiv(3 * sms(), N // tile)
    rpb = cdiv(rt, 3) * 128 - 17
    kw = dict(M=3 * rpb, N=N, K=256, tile=tile, w_static=1, rpb=rpb, nb=3, batched=True, seed=30)
    if form == "qkv_rope":
        kw.update(rope=True, amax=2)
    elif form == "fp8_qkv_rope":
        kw.update(rope=True, ab8=True, density=0.5)
    elif form == "fp8_out_proj":
        kw.update(row_len=True, gate="shared", resid="alias", out="f32", out2="e4m3", ln_scale=True, ab8=True,
                  density=0.125)
    else:
        kw.update(ab8=True, out="e4m3", density=0.25)
    run_exact(**kw)


# ---------------------------------------------------------------- every instantiation over many waves
# One case per (instantiation, BN) of dispatch_epi and dispatch_scaled (gemm.cu), in the form a production path launches
# it (or the closest form where none does).  Each is sized from the SM count S so that the launch has 3 S + r tiles,
# 0 < r < S: every CTA runs 3 or 4 tiles on both consumer warpgroups, the last wave is ragged.  K makes num_kb not a
# multiple of the ring depth, so that consecutive tiles of a CTA start at different ring stages and phases.  `rows`:
# "flat" (one matrix), ("utt", nb) (nb utterances, flat tiles straddling them) or ("batched", nb) (tiles never straddle).
# The fused-LN consumer needs K / 64 a power of two (ln_row_stats), hence its K of 128 / 256 at BN 128.
_QKV = dict(N=960, rope=True, ln_in=True, rows=("utt", 3))                       # D = 320: N ragged at BN 128
_OUT_PROJ = dict(N=320, row_len=True, gate="shared", resid="alias", out="f32", ln_scale=True, rows=("utt", 2))
_FF1 = dict(N=704, act=1, ln_in=True, rows="flat")
_CONV31 = dict(N=512, K=64, conv_taps=31, conv_pad=15, conv_grouped=True, act=3, rows=("batched", 6))
_MISH_PRODUCER = dict(N=512, act=3, resid="sep", out="f32", ln_scale=True, amax=1, density=0.25)
WAVES = {
    # ---- bf16: the DiT, text ConvNeXt, Vocos and the duration model
    "qkv_64": dict(_QKV, tile=64, K=512),
    "qkv_128": dict(_QKV, tile=128, K=128),
    "plain_bf16_64": dict(N=1000, K=320, tile=64, row_len=True, resid="sep", rows=("utt", 3)),     # no production caller
    "plain_bf16_128": dict(N=1000, K=448, tile=128, row_len=True, resid="sep", rows=("utt", 3)),
    "out_proj_64": dict(_OUT_PROJ, tile=64, K=320, out2="bf16", amax=1, density=0.125),
    "vocos_conv7_128": dict(N=456, K=128, tile=128, conv_taps=7, conv_pad=3, out="f32", rows=("batched", 3)),
    "ff1_64": dict(_FF1, tile=64, K=512),
    "ff1_128": dict(_FF1, tile=128, K=128),
    "gelu_resid_64": dict(N=1000, K=320, tile=64, act=1, resid="sep", rows="flat"),               # no production caller
    "gelu_resid_128": dict(N=1000, K=448, tile=128, act=1, resid="sep", rows="flat"),
    "pw1_erf_64": dict(N=1000, K=320, tile=64, act=2, rows="flat"),
    "pw1_erf_128": dict(N=1000, K=448, tile=128, act=2, rows="flat"),
    "conv_pos1_64": dict(_CONV31, tile=64, row_len=True),
    "mish_bf16_128": dict(N=1000, K=320, tile=128, act=3, row_len=True, rows=("utt", 6)),          # plain-GEMM form
    "conv_pos2_64": {**_CONV31, **_MISH_PRODUCER, "tile": 64, "out2": "bf16"},
    "mish_producer_128": dict(_MISH_PRODUCER, K=320, tile=128, out2="bf16", rows="flat"),
    # ---- per-tensor FP8: e4m3 operands (acc_scale 0.5), e4m3 second / FF1 outputs
    "fp8_qkv_64": dict(_QKV, tile=64, K=1024, ab8=True, density=0.5),
    "fp8_qkv_128": dict(_QKV, tile=128, K=256, ab8=True, density=0.5),
    "fp8_e4m3_out_64": dict(N=1008, K=640, tile=64, ab8=True, out="e4m3", density=0.25, row_len=True, rows=("utt", 3)),
    "fp8_e4m3_out_128": dict(N=1008, K=1152, tile=128, ab8=True, out="e4m3", density=0.25, rows="flat"),
    "fp8_out_proj_64": dict(_OUT_PROJ, tile=64, K=640, ab8=True, out2="e4m3", density=0.0625),
    "fp8_ff2_128": dict(_OUT_PROJ, tile=128, K=1152, ab8=True, out2="e4m3", density=0.0625, row_len=False),
    "fp8_ff1_64": dict(_FF1, tile=64, K=1024, ab8=True, out="e4m3", density=0.5),
    "fp8_ff1_128": dict(_FF1, tile=128, K=256, ab8=True, out="e4m3", density=0.5),
    "fp8_gelu_resid_64": dict(N=1000, K=640, tile=64, ab8=True, act=1, resid="sep", density=0.5, rows="flat"),
    "fp8_gelu_resid_128": dict(N=1000, K=1152, tile=128, ab8=True, act=1, resid="sep", density=0.5, rows="flat"),
    "fp8_conv_pos2_64": {**_CONV31, **_MISH_PRODUCER, "tile": 64, "out2": "e4m3"},
    "fp8_mish_producer_128": dict(_MISH_PRODUCER, K=320, tile=128, out2="e4m3", rows="flat"),
    # ---- block-scaled FP8: per-(row, 64-column) A scales, per-channel W scales, block-scaled e4m3 outputs
    "s_qkv_64": dict(_QKV, tile=64, K=1024, scaled=True, density=0.5),
    "s_qkv_128": dict(_QKV, tile=128, K=256, scaled=True, density=0.5),
    # FF2: A is FF1's e4m3 output, its scales in FF1's [K/64][M] out_scale layout (ld = M); no row mask
    "s_ff2_64": dict(_OUT_PROJ, tile=64, K=2048, scaled=True, a_scale_ld=-1, out2="e4m3", density=0.0625,
                     scale_exp=(-1, 1), row_len=False),
    "s_out_proj_128": dict(_OUT_PROJ, tile=128, K=640, scaled=True, out2="e4m3", density=0.0625, scale_exp=(-1, 1)),
    "s_ff1_64": dict(_FF1, tile=64, K=1024, scaled=True, out="e4m3", density=0.5),
    "s_ff1_128": dict(_FF1, tile=128, K=256, scaled=True, out="e4m3", density=0.5),
    "s_conv_pos2_64": {**_CONV31, **_MISH_PRODUCER, "tile": 64, "out2": "e4m3", "out_blocks": True},
    "s_mish_producer_128": dict(_MISH_PRODUCER, K=320, tile=128, out2="e4m3", out_blocks=True, rows="flat"),
}


def wave_case(name: str, sms: int) -> dict:
    """WAVES[name] as run_exact arguments for a GPU with `sms` SMs: M (and rows per utterance) such that the launch has
    3 sms + r output tiles, 0 < r < sms, with ragged M tails; w_static alternates over the table."""
    c = dict(WAVES[name])
    rows = c.pop("rows")
    tiles_n = cdiv(c["N"], 64 if c.get("conv_grouped") else c["tile"])
    mt = cdiv(3 * sms + 1, tiles_n)                      # row tiles wanted
    if rows == "flat":
        c.update(M=mt * 128 - 37)
    elif rows[0] == "utt":
        nb = rows[1]
        rpb = (mt * 128 - 37) // nb
        c.update(M=nb * rpb, rpb=rpb, nb=nb)
    else:
        nb = rows[1]
        rpb = cdiv(mt, nb) * 128 - 50
        c.update(M=nb * rpb, rpb=rpb, nb=nb, batched=True)
    if c.get("a_scale_ld") == -1:
        c["a_scale_ld"] = c["M"]
    c["w_static"] = list(WAVES).index(name) % 2
    c["seed"] = 100 + list(WAVES).index(name)
    return c


def wave_geometry(c: dict, sms: int) -> dict:
    """Tiles, tiles per CTA (persistent grid min(tiles, sms)), num_kb and the ring depth of a run_exact case."""
    bn = gemm_bn(c["N"], c["M"], tile_n=c["tile"], rows_per_batch=c.get("rpb", 0), num_batches=c.get("nb", 1),
                 batched=c.get("batched", False), conv_grouped=c.get("conv_grouped", False), sms=sms)
    tiles = gemm_tile_count(c["N"], c["M"], bn, rows_per_batch=c.get("rpb", 0), num_batches=c.get("nb", 1),
                            batched=c.get("batched", False))
    grid = min(tiles, sms)
    num_kb = gemm_num_kb(c["K"], conv_taps=c.get("conv_taps", 1), ab8=c.get("ab8", False) or c.get("scaled", False))
    return dict(bn=bn, tiles=tiles, per_cta=(tiles // grid, cdiv(tiles, grid)), num_kb=num_kb, stages=STAGES[bn])


@pytest.mark.parametrize("name", list(WAVES))
def test_every_instantiation_over_many_waves(name):
    """Each (instantiation, BN) at 3 SMs + r tiles: exact answers (or, after an activation, the float64 bound and bitwise
    equality with one-wave slices), NaN guards around every output."""
    S = sms()
    c = wave_case(name, S)
    geo = wave_geometry(c, S)
    assert 3 * S < geo["tiles"] < 4 * S and geo["num_kb"] % geo["stages"] != 0, geo
    print(f"{name}: M={c['M']} N={c['N']} K={c['K']} BN={geo['bn']}: {geo['tiles']} tiles on {S} SMs, "
          f"{geo['per_cta'][0]}-{geo['per_cta'][1]} per CTA, num_kb {geo['num_kb']}, {geo['stages']} stages")
    run_exact(**c)


@pytest.mark.parametrize("ws", [0, 1])
def test_grouped_conv31_many_waves(ws):
    """The conv position embedding's grouped Conv1d(k=31, pad 15) over three utterances whose row tiles spread over
    >= 3 tiles per SM, the last row tile of each utterance ragged."""
    from f5_tts_mlx_b200 import ops
    Cc, B = 256, 3
    NF = cdiv(3 * sms(), B * (Cc // 64)) * 128 - 50
    x = ints((B * NF, Cc), 4, 41)
    wt = ints((Cc, 64, 31), 2, 42)
    wp = wt.permute(0, 2, 1).reshape(Cc, 31 * 64).contiguous()
    bias = ints((Cc,), 8, 43, dtype=torch.float32)
    g = Guarded(B * NF, Cc, torch.bfloat16, DEV)
    ops.gemm(x, wp, g.view, n=Cc, k=64, bias=bias, rows_per_batch=NF, num_batches=B, batched_tiles=True,
             conv_taps=31, conv_pad=15, conv_grouped=True, w_static=bool(ws))
    torch.cuda.synchronize()
    ref = F.conv1d(x.double().view(B, NF, Cc).transpose(1, 2), wt.double(), bias.double(), padding=15, groups=Cc // 64)
    assert_exact(g.view, round_to(ref.transpose(1, 2).reshape(B * NF, Cc), torch.bfloat16), gemm_tiles(64, NF, True),
                 "conv31")
    g.check("conv31 guard")


# ---------------------------------------------------------------- a DiT block's GEMM chain with PDL live
@pytest.mark.parametrize("mode", ["bf16", "block"])
def test_block_gemm_chain_pdl_and_graph(mode):
    """One DiT block's GEMMs as f5_dit_forward chains them — out-projection producer (in-place residual, gate, row mask,
    LN operand and statistics) -> FF1 consumer (GELU) -> FF2 producer -> QKV consumer (RoPE, q_scale) — in bf16 or
    block-scaled FP8 mode, every launch at >= 3 tiles per CTA with static weights.  Launched back to back on one stream
    (each kernel's prologue overlaps its predecessor's tail under programmatic dependent launch) and as a captured,
    replayed CUDA graph, the results must be bitwise equal to the same sequence with a synchronize after every launch."""
    from f5_tts_mlx_b200 import ops
    from f5_tts_mlx_b200.dit import rope_table
    from f5_tts_mlx_b200.weights import quantize_e4m3_blocks
    S, D, Fi, nb = sms(), 512, 1024, 2
    rpb = (cdiv(3 * S + 1, D // 128) * 128 - 37) // nb
    R = nb * rpb
    for n in (D, Fi, 3 * D):      # the launcher picks 128-wide tiles here; the narrowest GEMM still has >= 3 per CTA
        bn = gemm_bn(n, R, rows_per_batch=rpb, num_batches=nb, sms=S)
        assert gemm_tile_count(n, R, bn) >= 3 * S, (n, bn)
    g = torch.Generator(device=DEV).manual_seed(5)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    blk = mode == "block"

    def weight(n, k):
        wf = rn(n, k) * k ** -0.5
        if not blk:
            return wf.bfloat16(), None
        q, s = quantize_e4m3_blocks(wf, k)
        return q, s.reshape(n).contiguous()

    (w_out, ws_out), (w1, ws1), (w2, ws2), (wq, wsq) = weight(D, D), weight(Fi, D), weight(D, Fi), weight(3 * D, D)
    b_out, b1, b2, bq = rn(D), rn(Fi), rn(D), rn(3 * D)
    gate1, gate2, s1, s2 = rn(D), rn(D), rn(D) * 0.3, rn(D) * 0.3
    tab1, tabq = rn(4, Fi) * 0.1, rn(4, 3 * D) * 0.1
    lens = torch.tensor([rpb, rpb - 100], dtype=torch.int32, device=DEV)
    rope = rope_table(rpb).to(DEV)
    x0 = rn(R, D) * 2
    attn = rn(R, D)
    if blk:
        q, sc = quantize_e4m3_blocks(attn, 64)
        attn, attn_s = q, sc.T.contiguous()
    else:
        attn = attn.bfloat16()
    x = torch.empty(R, D, device=DEV)
    a = torch.empty(R, D, device=DEV, dtype=torch.uint8 if blk else torch.bfloat16)
    ff = torch.empty(R, Fi, device=DEV, dtype=torch.uint8 if blk else torch.bfloat16)
    st = torch.empty(R, D // 64, 2, device=DEV)
    qkv = torch.empty(R, 3 * D, device=DEV, dtype=torch.bfloat16)
    a_s, ff_s = torch.empty(D // 64, R, device=DEV), torch.empty(Fi // 64, R, device=DEV)
    utt = dict(rows_per_batch=rpb, num_batches=nb)
    f8 = dict(ab_fp8=True) if blk else {}

    def launches():
        ops.gemm(attn, w_out, x, bias=b_out, resid=x, gate=gate1, row_len=lens, out2=a, ln_scale=s1, ln_stats=st,
                 w_static=True, **utt, **(dict(f8, a_scale=attn_s, w_scale=ws_out, out2_fp8=True, out2_scale=a_s) if blk else {}))
        yield
        ops.gemm(a, w1, ff, bias=b1, act=1, ln_in_stats=st, ln_tab=tab1, w_static=True,
                 **(dict(f8, a_scale=a_s, w_scale=ws1, out_fp8=True, out_scale=ff_s) if blk else {}))
        yield
        ops.gemm(ff, w2, x, bias=b2, resid=x, gate=gate2, out2=a, ln_scale=s2, ln_stats=st, w_static=True, **utt,
                 **(dict(f8, a_scale=ff_s, w_scale=ws2, out2_fp8=True, out2_scale=a_s) if blk else {}))
        yield
        ops.gemm(a, wq, qkv, bias=bq, ln_in_stats=st, ln_tab=tabq, rope=rope, rope_cols=2 * D, q_scale=0.125, q_cols=D,
                 w_static=True, **utt, **(dict(f8, a_scale=a_s, w_scale=wsq) if blk else {}))
        yield

    outs = {"x": x, "operand": a, "ln_stats": st.view(R, -1), "ff": ff, "qkv": qkv}
    if blk:
        outs.update(operand_scales=a_s, ff_scales=ff_s)

    def reset():
        x.copy_(x0)
        for t in (a, ff, st, qkv, a_s, ff_s):
            t.view(torch.uint8).fill_(0xFF)       # NaN in every dtype: a missing write cannot pass as a stale one

    def snapshot():
        torch.cuda.synchronize()
        return {k: v.clone() for k, v in outs.items()}

    reset()
    for _ in launches():
        torch.cuda.synchronize()
    want = snapshot()
    reset()
    for _ in launches():
        pass
    eager = snapshot()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in launches():
            pass
    reset()
    graph.replay()
    replay = snapshot()
    loc = gemm_tiles(128)
    for k in outs:
        assert_exact(eager[k], want[k], loc, f"{mode} chain, back to back: {k}")
        assert_exact(replay[k], want[k], loc, f"{mode} chain, graph replay: {k}")
    assert torch.isfinite(want["x"]).all() and torch.isfinite(want["qkv"].float()).all()
