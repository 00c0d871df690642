"""-m gpu: the FP8 attention mode (DESIGN.md sections 5 and 8) — the quantise pass bitwise against the host rule, the FP8
attention on exact known answers and on random data within a derived bound, the DiT in that mode against its
emulation, sample() through from_pretrained, and the refusal of a partly bound mode."""
import ctypes as C

import pytest
import torch

from helpers import ocfg_of, rel
from kernel_check import (E4M3_SUB, EPS_EX2, U32, U_E4M3, Guarded, assert_exact, assert_within, attn_tiles)
from oracle import f5_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
F8 = torch.float8_e4m3fn


def _lib():
    from f5_tts_mlx_b200 import _lib as L
    return L


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _npad(n):
    return (n + 127) // 128 * 128


def run_quant(qkv, B, N, H, kv=None):
    """The quantise pass into guarded buffers: f5_qkv_quant_e4m3 (every key valid) when kv is None, else
    f5_qkv_quant_e4m3_masked with kv (device int32 [B] valid keys).  Returns (qk [R, 2D], vt [B*D, Npad],
    scales [3H, R])."""
    D, R = H * 64, B * N
    qk = Guarded(R, 2 * D, torch.uint8, DEV)
    vt = Guarded(B * D, _npad(N), torch.uint8, DEV)
    sc = Guarded(3 * H, R, torch.float32, DEV, lr=False)
    lib = _lib().load()
    args = (qkv.data_ptr(), qkv.stride(0), qk.view.data_ptr(), qk.view.stride(0), vt.view.data_ptr(), vt.view.stride(0),
            sc.view.data_ptr(), B, N, H)
    if kv is None:
        _lib().check(lib.f5_qkv_quant_e4m3(*args, _stream()))
    else:
        _lib().check(lib.f5_qkv_quant_e4m3_masked(*args, kv.data_ptr(), _stream()))
    return qk, vt, sc


def run_attention(qkv, B, N, H, kv):
    """quantise pass + f5_attention_fwd_fp8, both with kv_len kv: (dequantised output [R, D] float32, out guard, scale
    guard)."""
    D, R = H * 64, B * N
    qk, vt, sc = run_quant(qkv, B, N, H, kv)
    out = Guarded(R, D, torch.uint8, DEV)
    so = Guarded(H, R, torch.float32, DEV, lr=False)
    L = _lib()
    L.check(L.load().f5_attention_fwd_fp8(qk.view.data_ptr(), qk.view.stride(0), vt.view.data_ptr(), vt.view.stride(0),
                                          sc.view.data_ptr(), out.view.data_ptr(), out.view.stride(0), B, N, H, 64,
                                          kv.data_ptr() if kv is not None else None, so.view.data_ptr(), _stream()))
    torch.cuda.synchronize()
    codes = out.view.cpu().view(F8).float().reshape(R, H, 64)
    deq = (codes * so.view.cpu().T[..., None]).reshape(R, D)
    return deq, out, so


def expected_vt(vcodes: torch.Tensor, N: int) -> torch.Tensor:
    """V codes [N, 64] (uint8) of one (utterance, head) -> the V^T block [64, Npad] in the host key order."""
    from f5_tts_mlx_b200.weights import fp8_vt_key_order
    t = torch.zeros(64, _npad(N), dtype=torch.uint8)
    t[:, :N] = vcodes.T
    pos = torch.arange(_npad(N))
    return t[:, pos // 32 * 32 + fp8_vt_key_order()[pos % 32]]


# ---------------------------------------------------------------- the quantise pass
def expected_codes(qkv: torch.Tensor, B: int, N: int, H: int, kv_len=None):
    """The host rule applied to the bf16 qkv: q per (row, head), k and v per (utterance, head, 128-key tile)
    (weights.quantize_e4m3_blocks with one block spanning the tile's rows), the keys at or beyond kv_len [B] (None: N,
    clamped to [1, N] as the kernels do) read as zero.  Returns codes uint8 [R, 3D] and scales [3H, R], every key
    carrying its tile's scale."""
    from f5_tts_mlx_b200.weights import E4M3_MAX, e4m3_block_scale, quantize_e4m3_blocks
    D, T = H * 64, (N + 127) // 128
    x = qkv.float()
    codes = torch.empty(B * N, 3 * D, dtype=torch.uint8)
    scales = torch.empty(3 * H, B * N)
    codes[:, :D], sq = quantize_e4m3_blocks(x[:, :D], 64)
    scales[:H] = sq.T
    # k and v: [B, T, 128, 2, H, 64] with the padding and masked keys zero (they do not move a tile's amax)
    kvx = x[:, D:].reshape(B, N, 2 * D)
    if kv_len is not None:
        valid = torch.arange(N)[None] < kv_len.cpu().long().clamp(1, N)[:, None]
        kvx = torch.where(valid[..., None], kvx, torch.zeros(()))
    kv = torch.nn.functional.pad(kvx, (0, 0, 0, T * 128 - N)).reshape(B, T, 128, 2, H, 64)
    s = e4m3_block_scale(kv.abs().amax(dim=(2, 5)))                                  # [B, T, 2, H]
    q = (kv * (1.0 / s)[:, :, None, :, :, None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    codes[:, D:] = q.view(torch.uint8).reshape(B, T * 128, 2 * D)[:, :N].reshape(B * N, 2 * D)
    per_key = s[:, :, None].expand(B, T, 128, 2, H).reshape(B, T * 128, 2 * H)[:, :N]  # [B, N, 2H]
    scales[H:] = per_key.reshape(B * N, 2 * H).T
    return codes, scales


_QUANT_N = [129, 300, 937, 5625, 8192]


@pytest.mark.parametrize("N,ragged", [(n, False) for n in _QUANT_N] + [(n, True) for n in _QUANT_N],
                         ids=[str(n) for n in _QUANT_N] + [f"{n}-ragged" for n in _QUANT_N])
def test_quantise_pass_bitwise(N, ragged):
    """Codes and scales of Q (per row and head) and of K and V (per 128-key tile and head) equal the host rule on the
    bf16 input; V^T holds the transposed V codes in the host key order, zero codes on the padding keys; guard bands
    untouched.  B = 3, H = 4 up to N = 937; B = 2, H = 16 at 60 s (N = 5625) and max_duration (8192).
    ragged: B = 4 with kv_len = (N, ending inside a key tile, ending at a multiple of 128, 1) and every row at or
    beyond kv_len +-3e4: those keys do not move their tile's k and v scales (the valid keys keep the codes they would
    have without them) and have zero K and V codes; Q is quantised on every row."""
    B, H = (3, 4) if N < 1000 else (2, 16)
    kv = None
    if ragged:
        B = 4
        mid = N // 2 + 5 if (N // 2 + 5) % 128 else N // 2 + 6
        kv = torch.tensor([N, mid, (N - 1) // 128 * 128, 1], dtype=torch.int32)
    D, R = H * 64, B * N
    g = torch.Generator().manual_seed(N)
    x = torch.randn(R, 3 * D, generator=g) * torch.pow(2.0, torch.randint(-12, 13, (R, 3 * H), generator=g).float()
                                                        ).repeat_interleave(64, 1)
    x[::17, :64] = 0                                              # all-zero units: scale 1
    x[5, 2 * D + 64:2 * D + 128] = 3e4                            # beyond 448
    x[N:N + 128, D + 64:D + 128] = 0                              # an all-zero k tile of utterance 1
    if ragged:
        for b in range(B):
            rows = slice(b * N + int(kv[b]), (b + 1) * N)
            x[rows] = 3e4 * (torch.randint(0, 2, x[rows].shape, generator=g) * 2 - 1)
    qkv = x.bfloat16()
    qk, vt, sc = run_quant(qkv.to(DEV), B, N, H, kv.to(DEV) if kv is not None else None)
    torch.cuda.synchronize()
    codes, scales = expected_codes(qkv, B, N, H, kv)
    assert_exact(qk.view.cpu(), codes[:, :2 * D].contiguous(), attn_tiles(N), "q|k codes")
    assert_exact(sc.view.cpu(), scales, lambda r, c: f"unit {r} row {c}", "scales")
    vt_got = vt.view.cpu()
    for b in range(B):
        for h in range(H):
            want = expected_vt(codes[b * N:(b + 1) * N, 2 * D + h * 64:2 * D + (h + 1) * 64], N)
            got = vt_got[b * D + h * 64:b * D + (h + 1) * 64]
            assert_exact(got, want, lambda r, c: f"utt {b} head {h} d {r} position {c}", "V^T")
    for gd, what in ((qk, "qk"), (vt, "vt"), (sc, "scales")):
        gd.check(what + " guard")


# ---------------------------------------------------------------- the attention: exact known answers
_VALS = torch.tensor([1.0, -1.0, 1.5, -1.5, 2.0, -2.0, 3.0, -3.0])


@pytest.mark.parametrize("case", list(range(6)) + ["last"])
def test_fp8_attention_one_hot_key(case):
    """One key per (utterance, head) has logit 64, every other valid key 0, so every query's output is V[hot] exactly
    (the others weigh below e^-64).  Across the cases the hot keys cover every residue mod 32 and the first five 128-key
    tiles (positions 0, 127 and 128 are fixed points of the key order and would miss a layout error).  Keys beyond
    kv_len have logit 128: a leak would dominate."""
    B, N, H = 2, 937, 3
    D = H * 64
    kv = torch.tensor([937, 700], dtype=torch.int32)
    g = torch.Generator().manual_seed(41)
    qkv = torch.zeros(B * N, 3 * D)
    qkv[:, :D] = 1.0
    qkv[:, 2 * D:] = _VALS[torch.randint(0, 8, (B * N, D), generator=g)]
    kk = qkv[:, D:2 * D].view(B, N, H, 64)
    vv = qkv[:, 2 * D:].view(B, N, H, 64)
    want = torch.empty(B, N, H, 64)
    for b in range(B):
        L = int(kv[b])
        kk[b, L:] = 2.0
        for h in range(H):
            i = b * H + h
            idx = L - 1 - 37 * i if case == "last" else (6 * case + i) % 32 + 32 * ((7 * case + i) % 4) + 128 * ((case + i) % 5)
            kk[b, idx, h] = 1.0
            want[b, :, h] = vv[b, idx, h]
    deq, out, so = run_attention(qkv.bfloat16().to(DEV), B, N, H, kv.to(DEV))
    assert_exact(deq, want.reshape(B * N, D), attn_tiles(N), f"one-hot {case}")
    out.check("one-hot out guard"); so.check("one-hot scale guard")


def test_fp8_attention_uniform_mean():
    """Q = 0: every valid key weighs the same, and with V constant per column (per-head magnitudes from 2^-6 to 2^6)
    the output is that constant exactly, for full and masked utterances."""
    B, N, H = 2, 300, 4
    D = H * 64
    kv = torch.tensor([201, 300], dtype=torch.int32)
    g = torch.Generator().manual_seed(5)
    col = _VALS[torch.randint(0, 8, (D,), generator=g)] * torch.pow(2.0, torch.tensor([-6.0, 0.0, 3.0, 6.0])
                                                                      ).repeat_interleave(64)
    qkv = torch.zeros(B * N, 3 * D)
    qkv[:, D:2 * D] = torch.randn(B * N, D, generator=g)
    qkv[:, 2 * D:] = col
    deq, out, so = run_attention(qkv.bfloat16().to(DEV), B, N, H, kv.to(DEV))
    assert_exact(deq, col.expand(B * N, D).contiguous(), attn_tiles(N), "uniform mean")
    out.check("uniform out guard"); so.check("uniform scale guard")


# ---------------------------------------------------------------- the attention: random data, derived bound
def fp8_attention_bound(q, k, v, kv_len):
    """Reference and bound for the FP8 attention on [B, H, N, 64] operands that are already the dequantised e4m3 values
    the kernel multiplies (the quantise pass is checked bitwise above).

    With p_j = exp(s_j - m) and O = sum p_j v_j / l, a relative error d_j of each p_j in the numerator moves O by at most
    max|d| p|v| (p|v| = sum p_j |v_j| / l).  Sources of d: the e4m3 rounding of P~ = 2^8 p (U_E4M3); the S accumulation
    (a 64-product e4m3 wgmma partial, 2 k-steps of one 2^-12 truncation each of sum |q||k|, as gemm_acc_bound_fp8); the
    fp32 exponent argument (3u |s| log2 e, times ln 2) and ex2.approx (EPS_EX2); the running-max rescale, 2 (EPS_EX2 +
    u) per tile, which also perturbs l.  The P V partial of a tile (128 products, 4 k-steps) is off by 2^-10 of its sum
    |P~||codes|, the fp32 promotion adds 2u per tile.  Below 2^-6 P~ has the absolute e4m3 floor E4M3_SUB: key j adds
    at most E4M3_SUB |v_j| / (2^8 l) to O (v_j = sv_t codes_j; the running rescale only shrinks it).  1 / l and the
    products add 3u |O|."""
    from kernel_check import attention_ref
    o, pv, qk = attention_ref(q, k, v, kv_len)
    B, H, N, _ = q.shape
    tiles = (N + 127) // 128
    s = q.double() @ k.double().transpose(-1, -2)
    valid = torch.arange(N)[None] < kv_len[:, None].long()
    s = s.masked_fill(~valid[:, None, None, :], float("-inf"))
    l = torch.exp(s - s.amax(-1, keepdim=True)).sum(-1, keepdim=True)           # [B, H, N, 1], >= 1
    floor = (v.double().abs() * valid[:, None, :, None]).sum(-2, keepdim=True)  # [B, H, 1, 64]
    logit_max = s.masked_fill(torch.isinf(s), 0).abs().max().item()
    d = U_E4M3 + 2.0 ** -11 * qk + 3 * U32 * logit_max * 1.4427 * 0.6932 + EPS_EX2 + 2 * tiles * (EPS_EX2 + U32)
    b = 2 * d * pv + (2.0 ** -10 * (1 + U_E4M3) + 2 * U32 * (tiles + 1)) * pv + E4M3_SUB * floor / (256.0 * l) \
        + 3 * U32 * o.abs()
    return o, b


def test_fp8_attention_random_within_bound():
    """Random Q, K, V against float64 softmax on the same e4m3 operands, within fp8_attention_bound plus the block-scaled
    output rounding (relative 2^-4, absolute half the subnormal spacing of the row-head's scale).  V heads at widely
    different magnitudes, and two heads whose keys carry per-key magnitudes 2^-6 .. 2^6, so that a tile's scale is set
    by its largest keys and the small ones reach the e4m3 subnormal range; kv_len masking and N not a multiple of 128."""
    B, N, H = 2, 300, 4
    D = H * 64
    g = torch.Generator().manual_seed(9)
    x = torch.randn(B * N, 3 * D, generator=g)
    x[:, :D] *= 0.5
    x[:, 2 * D:] *= torch.pow(2.0, torch.tensor([-8.0, 0.0, 5.0, 0.0])).repeat_interleave(64)
    x[:, 2 * D + 128:] *= torch.pow(2.0, torch.randint(-6, 7, (B * N, 1), generator=g).float())
    qkv = x.bfloat16()
    kv = torch.tensor([300, 201], dtype=torch.int32)
    deq, out, so = run_attention(qkv.to(DEV), B, N, H, kv.to(DEV))
    codes, scales = expected_codes(qkv, B, N, H, kv)
    dq = (codes.view(F8).float().reshape(B * N, 3 * H, 64) * scales.T[..., None]).reshape(B * N, 3 * D)
    split = lambda t: t.reshape(B, N, H, 64).permute(0, 2, 1, 3)
    q, k, v = split(dq[:, :D]), split(dq[:, D:2 * D]), split(dq[:, 2 * D:])
    o, b = fp8_attention_bound(q, k, v, kv)
    flat = lambda t: t.permute(0, 2, 1, 3).reshape(B * N, D)
    o, b = flat(o), flat(b)
    s_out = so.view.cpu().T.repeat_interleave(64, 1).double()
    bound = b + U_E4M3 * (o.abs() + b) + E4M3_SUB * s_out
    assert_within(deq, o, bound, attn_tiles(N), "fp8 attention")
    out.check("out guard"); so.check("scale guard")


# ---------------------------------------------------------------- the DiT in FP8 attention mode
def _dit(cfg, W, **kw):
    from f5_tts_mlx_b200 import DiT
    return DiT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult, mel_dim=cfg.mel_dim,
               text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim, conv_layers=cfg.conv_layers, device=DEV,
               **kw).load_weights(W)


@pytest.mark.parametrize("construction", ["random", "outlier"])
def test_fp8_attention_forward_within_emulated_drift(construction):
    """DiT(fp8=True, fp8_scaling="block", fp8_attention=True) stays within 3x the drift of its CPU emulation
    (fp8_attn_emul) from the fp32 oracle, on the seeded random weights and on the outlier construction."""
    import fp8_attn_emul as A
    import fp8_block_emul as E
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
    emu = A.dit_forward_block8a(x, cond, text, t, False, False, None, W, ocfg_of(cfg))
    m = _dit(cfg, W, fp8=True, fp8_scaling="block", fp8_attention=True)
    got = m(x.to(DEV), cond.to(DEV), text.to(DEV), t).cpu()
    drift, r = rel(emu, ref), rel(got, ref)
    print(f"{construction}: fp8-attention rel {r:.3e}, emulated drift {drift:.3e}")
    assert torch.isfinite(got).all() and r < 3 * drift, (r, drift)


def test_fp8_attention_sample_through_from_pretrained():
    """from_pretrained("random", fp8="block", fp8_attention=True): sample() with a ragged batch (seq_len masking), with
    frame bucketing (valid_len), and again on the captured CUDA graph of the same plan."""
    from f5_tts_mlx_b200 import F5TTS
    from f5_tts_mlx_b200.pretrained import from_pretrained
    f5 = from_pretrained(F5TTS, "random", fp8="block", fp8_attention=True, vocoder=False)
    assert f5.transformer.fp8_attention
    g = torch.Generator().manual_seed(4)
    cond = (torch.randn(2, 120, 100, generator=g) * 2 - 1).to(DEV)
    text = torch.randint(0, 2545, (2, 40), generator=g, dtype=torch.int32)
    text[1, 30:] = -1
    out, _ = f5.sample(cond, text, torch.tensor([300, 260]), steps=4, method="euler", cfg_strength=2.0, seed=1)
    assert out.shape == (2, 300, 100) and torch.isfinite(out).all()
    assert f5.last_plan.session.seq_len is not None and f5.last_plan.session.qk_fp8 is not None
    one, _ = f5.sample(cond[:1], text[:1], 250, steps=4, method="euler", cfg_strength=2.0, seed=1, frame_bucket=128)
    assert one.shape == (1, 250, 100) and torch.isfinite(one).all()
    assert f5.last_plan.session.frames == 256 and f5.last_plan.session.vt_fp8.shape == (2, 1024, 256)
    again, _ = f5.sample(cond[:1], text[:1], 250, steps=4, method="euler", cfg_strength=2.0, seed=1, frame_bucket=128)
    assert torch.equal(again, one)                                   # the plan's graph replayed: same result


def test_dit_forward_rejects_a_partly_bound_fp8_attention():
    """A partial set of qk_fp8 / vt_fp8 / qkv_scale, or the full set without the block-scaled buffers, is F5_ERR_INVALID
    naming what is missing."""
    from f5_tts_mlx_b200.dit import DitBuffersC
    from f5_tts_mlx_b200.weights import GATE_CONFIG, random_dit_weights
    cfg = GATE_CONFIG
    W = random_dit_weights(cfg, seed=1234)
    L = _lib()
    lib = L.load()
    m = _dit(cfg, W, fp8=True, fp8_scaling="block", fp8_attention=True)
    s = m.session(1, 128, 1, False, 16, False)

    def forward(unbind):
        b = DitBuffersC.from_buffer_copy(s.c)
        for name in unbind:
            setattr(b, name, None)
        rc = lib.f5_dit_forward(C.byref(m.packed.c_struct()), C.byref(b), 0, _stream())
        return rc, lib.f5_last_error().decode()

    rc, msg = forward(("vt_fp8",))
    assert rc == -1 and "FP8 attention needs vt_fp8" in msg, msg
    rc, msg = forward(("qk_fp8", "qkv_scale"))
    assert rc == -1 and "FP8 attention needs qk_fp8, qkv_scale" in msg, msg
    rc, msg = forward(("a_fp8_scale", "attn_scale", "ff_scale"))
    assert rc == -1 and "FP8 attention needs the block-scaled FP8 mode" in msg, msg
