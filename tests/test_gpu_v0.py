"""-m gpu: F5TTS_Base (v0) on the H100 — unmasked text padding and rotary embedding on the leading heads only.

  * the QKV epilogue's second rotated range (f5_gemm_args.rope_col2), bitwise, in the bf16, per-tensor FP8 and
    block-scaled FP8 instantiations at the shapes the model launches;
  * the v0 DiT forward and sample() against the test-side restatement (tests/v0_emul.py), within 3x the drift of its
    bf16 emulation, on the gate and the base model; frame bucketing and a ragged batch; the block-scaled FP8 modes
    against their emulations composed with the v0 rotation.
"""
import ctypes as C

import pytest
import torch

from oracle import f5_oracle as O
from helpers import rel
import fp8_attn_emul as EA
import fp8_block_emul as EB
import v0_emul as V

pytestmark = pytest.mark.gpu
DEV = "cuda"


# ---------------------------------------------------------------- the epilogue, bitwise
def _qkv_operands(kind, M, D, seed):
    """A [M, D], W [3D, D] and the GEMM keywords of one QKV kind: bf16, per-tensor e4m3, block-scaled e4m3."""
    from f5_tts_mlx_b200.weights import quantize_e4m3_blocks
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = torch.randn(M, D, generator=g, device=DEV)
    w = torch.randn(3 * D, D, generator=g, device=DEV) / D ** 0.5
    kw = dict(bias=torch.randn(3 * D, generator=g, device=DEV))
    if kind == "bf16":
        return a.bfloat16(), w.bfloat16(), kw
    if kind == "fp8":
        kw.update(ab_fp8=True, acc_scale=w.abs().max().item() / 448.0)
        return (a.to(torch.float8_e4m3fn).view(torch.uint8),
                (w / kw["acc_scale"]).to(torch.float8_e4m3fn).view(torch.uint8), kw)
    qa, sa = quantize_e4m3_blocks(a, 64)                       # per (row, 64 columns)
    qw, sw = quantize_e4m3_blocks(w, D)                        # per output channel
    kw.update(ab_fp8=True, a_scale=sa.reshape(M, D // 64).t().contiguous(), w_scale=sw.reshape(-1).contiguous())
    return qa.view(torch.uint8), qw.view(torch.uint8), kw


@pytest.mark.parametrize("kind", ["bf16", "fp8", "block8"])
@pytest.mark.parametrize("D,frames,utts", [(512, 300, 2), (1024, 937, 2), (1024, 800, 1)])
def test_qkv_rope_leading_heads_bitwise(kind, D, frames, utts):
    """rope_cols = 64 h, rope_col2 = D: the rotated columns (q heads < h, k heads < h) equal today's all-heads launch
    bitwise, every other column equals the same launch with an identity table (cos 1, sin 0) bitwise, and that one
    equals q_scale x the rope-free GEMM's fp32 output rounded to bf16; h = heads is today's launch, bitwise."""
    from f5_tts_mlx_b200 import ops
    from f5_tts_mlx_b200.dit import rope_table
    heads, M = D // 64, frames * utts
    a, w, kw = _qkv_operands(kind, M, D, seed=D + frames)
    tab = rope_table(frames).to(DEV)
    ident = torch.stack([torch.ones(frames, 32), torch.zeros(frames, 32)], -1).contiguous().to(DEV)
    common = dict(rows_per_batch=frames, num_batches=utts, q_scale=0.125, q_cols=D, **kw)

    def qkv(table, rope_cols, rope_col2=0):
        out = torch.full((M, 3 * D), float("nan"), dtype=torch.bfloat16, device=DEV)
        return ops.gemm(a, w, out, rope=table, rope_cols=rope_cols, rope_col2=rope_col2, **common)

    today, plain = qkv(tab, 2 * D), qkv(ident, 2 * D)
    free = torch.full((M, 3 * D), float("nan"), device=DEV)
    ops.gemm(a, w, free, rows_per_batch=frames, num_batches=utts, **kw)
    scale = torch.ones(3 * D, device=DEV); scale[:D] = 0.125
    assert torch.equal(plain, (free * scale).bfloat16()), "identity rotation != q_scale x rope-free output"
    for h in (1, heads // 2, heads):
        got = qkv(tab, 64 * h, D)
        rot = torch.zeros(3 * D, dtype=torch.bool, device=DEV)
        rot[:64 * h] = True; rot[D:D + 64 * h] = True
        assert torch.equal(got[:, rot], today[:, rot]), f"rope_heads={h}: rotated columns"
        assert torch.equal(got[:, ~rot], plain[:, ~rot]), f"rope_heads={h}: unrotated columns"
        if h == heads:
            assert torch.equal(got, today)


def test_gemm_refuses_bad_second_rope_range():
    from f5_tts_mlx_b200 import _lib, ops
    D, M = 512, 256
    a = torch.zeros(M, D, dtype=torch.bfloat16, device=DEV)
    w = torch.zeros(3 * D, D, dtype=torch.bfloat16, device=DEV)
    out = torch.zeros(M, 3 * D, dtype=torch.bfloat16, device=DEV)
    tab = torch.zeros(M, 32, 2, device=DEV)
    for rope, rc, r2 in ((tab, 64, 32), (tab, 128, 64), (tab, 64, 3 * D), (None, 64, D), (tab, 0, D), (tab, 64, -64)):
        with pytest.raises(_lib.F5Error, match="rope_col2"):
            ops.gemm(a, w, out, rope=rope, rope_cols=rc, rope_col2=r2, q_scale=0.125, q_cols=D)


# ---------------------------------------------------------------- the DiT
def _dit(cfg, W, **kw):
    from f5_tts_mlx_b200 import DiT
    return DiT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult, mel_dim=cfg.mel_dim,
               text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim, conv_layers=cfg.conv_layers, device=DEV,
               **kw).load_weights(W)


V0 = dict(text_mask_padding=False, pe_attn_head=1)


@pytest.fixture(scope="module")
def gate():
    from f5_tts_mlx_b200.weights import GATE_CONFIG, random_dit_weights
    W = random_dit_weights(GATE_CONFIG, seed=1234)
    return GATE_CONFIG, W, _dit(GATE_CONFIG, W, **V0)


@pytest.fixture(scope="module")
def base():
    from f5_tts_mlx_b200.weights import BASE_CONFIG, random_dit_weights
    W = random_dit_weights(BASE_CONFIG, seed=1234)
    return BASE_CONFIG, W, _dit(BASE_CONFIG, W, **V0)


def within_drift(got, ref, ref16, factor=3.0, floor=2e-3):
    drift, r = rel(ref16, ref), rel(got, ref)
    assert torch.isfinite(got).all() and r < max(factor * drift, floor), f"rel {r:.3e} vs bf16 drift {drift:.3e}"
    return r, drift


def _inputs(B, N, nt, seed, pad_from=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, N, 100, generator=g); cond = torch.randn(B, N, 100, generator=g) * 2 - 1
    text = torch.randint(0, 2545, (B, nt), generator=g, dtype=torch.int32)
    if pad_from is not None:
        text[:, pad_from:] = -1                  # filler tokens inside the row, then rows past the text
    return x, cond, text


@pytest.mark.parametrize("which", ["gate", "base"])
@pytest.mark.parametrize("drops", [(False, False), (True, True), (False, True)])
def test_v0_forward_vs_restatement(which, drops, request):
    cfg, W, model = request.getfixturevalue(which)
    x, cond, text = _inputs(1, 200, 48, seed=7, pad_from=37)
    t = torch.tensor(0.37)
    ocfg = V.ocfg_v0(cfg)
    ref = V.dit_forward(x, cond, text, t, *drops, None, W, ocfg, pe_attn_head=1)
    ref16 = V.dit_forward(x, cond, text, t, *drops, None, W, ocfg, O.Precision(True), pe_attn_head=1)
    got = model(x.to(DEV), cond.to(DEV), text.to(DEV), t, *drops).cpu()
    r, drift = within_drift(got, ref, ref16)
    print(f"{which} drops={drops}: rel {r:.3e}, bf16 drift {drift:.3e}")
    # both v0 differences are visible at this size: v1 is far from the v0 answer
    assert rel(V.dit_forward(x, cond, text, t, *drops, None, W, V.ocfg_v0(cfg, True)), ref) > 10 * max(r, 1e-4)


def test_pe_attn_head_all_heads_is_v1_bitwise(gate):
    cfg, W, _ = gate
    x, cond, text = _inputs(1, 150, 30, seed=8)
    args = (x.to(DEV), cond.to(DEV), text.to(DEV), torch.tensor(0.5))
    assert torch.equal(_dit(cfg, W, pe_attn_head=cfg.heads)(*args), _dit(cfg, W)(*args))


@pytest.mark.parametrize("which", ["gate", "base"])
def test_v0_euler_cfg_sample_vs_restatement(which, request):
    from f5_tts_mlx_b200 import F5TTS
    cfg, W, model = request.getfixturevalue(which)
    g = torch.Generator().manual_seed(11)
    cond = (torch.randn(1, 60, 100, generator=g) * 2.24 - 1.27)
    text = torch.randint(0, 2545, (1, 40), generator=g, dtype=torch.int32); text[0, 33:] = -1
    N = 230
    y0 = torch.randn(1, N, 100, generator=g)
    kw = dict(steps=4, method="euler", cfg_strength=2.0, sway_sampling_coef=-1.0, y0=y0)
    out, _ = F5TTS(model).sample(cond.to(DEV), text, N, **kw)
    ocfg = V.ocfg_v0(cfg)
    ref, _ = V.sample(cond, text, N, W, ocfg, pe_attn_head=1, **kw)
    ref16, _ = V.sample(cond, text, N, W, ocfg, pe_attn_head=1, prec=O.Precision(True), **kw)
    r, drift = within_drift(out.cpu(), ref, ref16)
    print(f"{which} sample: rel {r:.3e}, bf16 drift {drift:.3e}")


def test_v0_frame_bucketing_equals_exact_shapes(gate):
    """150 / 201 / 255 frames in one 256-frame plan give the exact-shape results: the filler rows below N keep their
    embedding, the bucket rows at and past N stay zero for the text ConvNeXt and the conv position embedding."""
    from f5_tts_mlx_b200 import F5TTS
    cfg, W, model = gate
    g = torch.Generator().manual_seed(21)
    cond = (torch.randn(1, 60, 100, generator=g) * 2.24 - 1.27).to(DEV)
    kw = dict(steps=4, method="euler", cfg_strength=2.0, sway_sampling_coef=-1.0)
    exact, bucketed = F5TTS(model), F5TTS(model)
    bucketed.frame_bucket = 128
    plans = set()
    for N, nt in ((150, 20), (201, 31), (255, 27)):
        text = torch.randint(0, 2545, (1, nt), generator=g, dtype=torch.int32)
        y0 = torch.randn(1, N, 100, generator=g)
        a, _ = exact.sample(cond, text, N, y0=y0, **kw)
        b, _ = bucketed.sample(cond, text, N, y0=y0, **kw)
        plans.add(id(bucketed.last_plan))
        assert b.shape == a.shape == (1, N, 100)
        assert rel(b, a) < 1e-3, (N, rel(b, a))
        ref, _ = V.sample(cond.cpu(), text, N, W, V.ocfg_v0(cfg), pe_attn_head=1, y0=y0, **kw)
        assert rel(b.cpu(), ref) < 1e-2
    assert len(plans) == 1 and bucketed.last_plan.session.frames == 256


def test_v0_ragged_batch_vs_restatement(gate):
    from f5_tts_mlx_b200 import F5TTS
    cfg, W, model = gate
    g = torch.Generator().manual_seed(31)
    cond = (torch.randn(2, 70, 100, generator=g) * 2.24 - 1.27)
    text = torch.randint(0, 2545, (2, 45), generator=g, dtype=torch.int32); text[1, 29:] = -1
    dur = torch.tensor([260, 201])
    kw = dict(steps=4, method="euler", cfg_strength=2.0, sway_sampling_coef=-1.0, seed=3)
    out, _ = F5TTS(model).sample(cond.to(DEV), text, dur, **kw)
    ocfg = V.ocfg_v0(cfg)
    ref, _ = V.sample(cond, text, dur, W, ocfg, pe_attn_head=1, **kw)
    ref16, _ = V.sample(cond, text, dur, W, ocfg, pe_attn_head=1, prec=O.Precision(True), **kw)
    r, drift = within_drift(out.cpu(), ref, ref16)
    print(f"ragged batch: rel {r:.3e}, bf16 drift {drift:.3e}")


@pytest.mark.parametrize("mode", ["tensor", "block", "block+attn", "unfused"])
def test_v0_other_modes(gate, mode):
    """Per-tensor FP8, block FP8, block FP8 + FP8 attention and the separate-LayerNorm mode on v0.  The block modes stay
    within 3x the drift of fp8_block_emul / fp8_attn_emul composed with the v0 text embedding and rotation; per-tensor
    FP8 and the unfused mode, within 3x the drift of the oracle's FP8 / bf16 emulation of the v0 forward."""
    cfg, W, _ = gate
    kw = {"tensor": dict(fp8=True), "block": dict(fp8=True, fp8_scaling="block"),
          "block+attn": dict(fp8=True, fp8_scaling="block", fp8_attention=True), "unfused": dict(fused_adaln=False)}[mode]
    x, cond, text = _inputs(1, 300, 60, seed=2, pad_from=44)
    t = torch.tensor(0.25)
    ocfg = V.ocfg_v0(cfg)
    ref = V.dit_forward(x, cond, text, t, False, False, None, W, ocfg, pe_attn_head=1)
    if mode == "block":
        emu = V.dit_forward(x, cond, text, t, False, False, None, W, ocfg, EB.BF16, 1, block=EB.dit_block8)
    elif mode == "block+attn":
        emu = V.dit_forward(x, cond, text, t, False, False, None, W, ocfg, EA.BF16, 1, block=EA.dit_block8a)
    elif mode == "tensor":
        emu = V.dit_forward(x, cond, text, t, False, False, None, W, ocfg, O.Precision(True, True, fp8=True), 1)
    else:
        emu = V.dit_forward(x, cond, text, t, False, False, None, W, ocfg, O.Precision(True), 1)
    got = _dit(cfg, W, **V0, **kw)(x.to(DEV), cond.to(DEV), text.to(DEV), t).cpu()
    drift, r = rel(emu, ref), rel(got, ref)
    print(f"v0 {mode}: rel {r:.3e}, emulated drift {drift:.3e}")
    assert torch.isfinite(got).all() and r < max(3 * drift, 2e-3), (r, drift)


def test_dit_forward_refuses_bad_rope_heads(gate):
    from f5_tts_mlx_b200 import _lib
    cfg, W, model = gate
    x, cond, text = _inputs(1, 64, 10, seed=1)
    w = model.packed.c_struct()
    try:
        for bad, field in ((cfg.heads + 1, "rope_heads"), (-1, "rope_heads")):
            w.rope_heads = bad
            with pytest.raises(_lib.F5Error, match=field):
                model(x.to(DEV), cond.to(DEV), text.to(DEV), torch.tensor(0.5))
        w.rope_heads = 1
        w.text_unmasked = 2
        with pytest.raises(_lib.F5Error, match="text_unmasked"):
            model(x.to(DEV), cond.to(DEV), text.to(DEV), torch.tensor(0.5))
    finally:
        w.rope_heads, w.text_unmasked = 1, 1


def test_v0_through_from_pretrained_random():
    from f5_tts_mlx_b200 import F5TTS
    from f5_tts_mlx_b200.pretrained import from_pretrained
    f5 = from_pretrained(F5TTS, "random", vocoder=False, model_version="v0", fp8="block", fp8_attention=True)
    c = f5.transformer.config
    assert (c.text_mask_padding, c.pe_attn_head) == (False, 1)
    g = torch.Generator().manual_seed(4)
    cond = (torch.randn(2, 120, 100, generator=g) * 2 - 1).to(DEV)
    text = torch.randint(0, 2545, (2, 40), generator=g, dtype=torch.int32); text[1, 30:] = -1
    out, _ = f5.sample(cond, text, torch.tensor([300, 260]), steps=4, method="euler", cfg_strength=2.0, seed=1,
                       frame_bucket=128)
    assert out.shape == (2, 300, 100) and torch.isfinite(out).all()
