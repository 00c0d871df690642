"""CPU emulation of the block-scaled FP8 mode of the DiT (DiT(fp8=True, fp8_scaling="block"), DESIGN.md section 8).

It runs the oracle's DiT forward with exactly the rounding points of the CUDA path in that mode:
  * weights: e4m3 with one power-of-two scale per output channel;
  * activations: e4m3 with one power-of-two scale per (row, 64 columns), each computed from the fp32 value the kernel
    quantises: x * (1 + s) of the residual stream (the fused-LN operand of QKV / FF1), the attention output O / l (one
    scale per row and head) and the GELU output of FF1;
  * the fused-LN correction rstd * (acc - mean * c1) + c2 with c1 / c2 from the bf16 weights, as in the other modes;
  * everything else as Precision(emulate_bf16=True, ln_by_linearity=True).

The scale rule is restated here from its definition (the smallest power of two s >= 2^-126 with amax <= 448 s, found by
float64 comparisons), independently of the bit manipulation the package and the kernels use (weights.e4m3_block_scale,
ptx.cuh e4m3_block_scale), so the emulation does not share code with what it checks.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle import f5_oracle as O

BF16 = O.Precision(True, True)


def block_scale(amax: torch.Tensor) -> torch.Tensor:
    """The smallest power of two s >= 2^-126 with amax <= 448 s (1 for amax = 0, amax itself when not finite)."""
    a = amax.double()
    _, e = torch.frexp(torch.where(torch.isfinite(a) & (a > 0), a, torch.ones_like(a)))   # a = m 2^e, m in [0.5, 1)
    k = (e - 9).double()                                     # 448 2^(e-9) = 0.875 2^e: within one step of the answer
    k = torch.where(a > 448.0 * torch.exp2(k), k + 1, k)
    k = torch.where(a <= 448.0 * torch.exp2(k - 1), k - 1, k)
    s = torch.exp2(k.clamp_min(-126.0))
    s = torch.where(a == 0, torch.ones_like(s), s)
    return torch.where(torch.isfinite(a), s, a).float()


def _quant(x: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """e4m3 codes (as fp32) of x / s, s broadcast over the block, rounded to nearest even."""
    return (x.double() / s.double()).clamp(-448.0, 448.0).to(torch.float8_e4m3fn).float()


def q_rows(x: torch.Tensor) -> torch.Tensor:
    """Block-scaled e4m3 round trip of the last dimension in units of 64 columns: codes * scale."""
    shp = x.shape
    g = x.float().reshape(-1, shp[-1] // 64, 64)
    s = block_scale(g.abs().amax(dim=-1))[..., None]
    return (_quant(g, s) * s).reshape(shp)


def q_channels(w: torch.Tensor):
    """Per-output-channel e4m3 weight: (codes as fp32, scale per row)."""
    s = block_scale(w.float().abs().amax(dim=1))
    return _quant(w.float(), s[:, None]), s


def linear8(a_deq: torch.Tensor, w: torch.Tensor, b) -> torch.Tensor:
    wq, ws = q_channels(w)
    out = F.linear(a_deq, wq) * ws
    return out + b if b is not None else out


def adaln8(x, scale, shift, w, b, eps=1e-6):
    """The fused-LN consumer on a block-scaled e4m3 operand: rstd * (w_s * (x~ W~^T) - mean * c1) + c2."""
    mu = x.mean(dim=-1, keepdim=True)
    rstd = torch.rsqrt(x.var(dim=-1, unbiased=False, keepdim=True) + eps)
    wb = BF16.op(w)
    c1 = F.linear(1 + scale, wb)[:, None]
    c2 = F.linear(shift, wb, b)[:, None]
    acc = linear8(q_rows(x * (1 + scale[:, None])), w, None)
    return rstd * (acc - mu * c1) + c2


def attention8(x, mask, rope, W, pfx, heads, scale_msa, shift_msa):
    b, n, _ = x.shape
    wqkv = torch.cat([W[pfx + f"to_{c}.weight"] for c in "qkv"], 0)
    bqkv = torch.cat([W[pfx + f"to_{c}.bias"] for c in "qkv"], 0)
    qkv = adaln8(x, scale_msa, shift_msa, wqkv, bqkv)
    q, k, v = qkv.chunk(3, dim=-1)
    q, k, v = [t.reshape(b, n, heads, -1).permute(0, 2, 1, 3) for t in (q, k, v)]
    q = O.apply_rotary_pos_emb(q, rope, 1.0)
    k = O.apply_rotary_pos_emb(k, rope, 1.0)
    s = torch.matmul(BF16.op(q / math.sqrt(q.shape[-1])), BF16.op(k).transpose(-1, -2))
    if mask is not None:
        s = s.masked_fill(~mask[:, None, None, :], float("-inf"))
    m = s.max(dim=-1, keepdim=True).values
    e = torch.exp(s - m)
    o = torch.matmul(BF16.op(e), BF16.op(v)) / e.sum(dim=-1, keepdim=True)
    o = o.permute(0, 2, 1, 3).reshape(b, n, -1)
    o = linear8(q_rows(o), W[pfx + "to_out.layers.0.weight"], W[pfx + "to_out.layers.0.bias"])
    if mask is not None:
        o = o * mask[:, :, None]
    return o


def dit_block8(x, t, mask, rope, W, i, cfg):
    p = f"transformer.transformer_blocks.{i}."
    emb = O.linear(F.silu(t), W[p + "attn_norm.linear.weight"], W[p + "attn_norm.linear.bias"], BF16)
    shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp = emb.chunk(6, dim=1)
    x = x + gate_msa[:, None] * attention8(x, mask, rope, W, p + "attn.", cfg.heads, scale_msa, shift_msa)
    h = adaln8(x, scale_mlp, shift_mlp, W[p + "ff.ff.layers.0.layers.0.weight"], W[p + "ff.ff.layers.0.layers.0.bias"])
    h = F.gelu(h, approximate="tanh")
    ff = linear8(q_rows(h), W[p + "ff.ff.layers.2.weight"], W[p + "ff.ff.layers.2.bias"])
    return x + gate_mlp[:, None] * ff


def dit_forward_block8(x, cond, text, time, drop_audio_cond, drop_text, mask, W, cfg):
    """oracle.dit_forward with the rounding points of the block-scaled FP8 mode."""
    batch, seq_len = x.shape[0], x.shape[1]
    if time.ndim == 0:
        time = time.repeat(batch)
    t = O.timestep_embedding(time.float(), W)
    text_embed = O.text_embedding(text, seq_len, drop_text, W, cfg, BF16)
    x = O.input_embedding(x, cond, text_embed, drop_audio_cond, W, BF16)
    rope = O.rotary_freqs(seq_len, cfg.dim_head)
    for i in range(cfg.depth):
        x = dit_block8(x, t, mask, rope, W, i, cfg)
    emb = O.linear(F.silu(t), W["transformer.norm_out.linear.weight"], W["transformer.norm_out.linear.bias"], BF16)
    scale, shift = emb.chunk(2, dim=1)
    return O.adaln_linear(x, scale, shift, W["transformer.proj_out.weight"], W["transformer.proj_out.bias"], BF16)


def outlier_weights(W: dict, cfg, seed: int = 7) -> dict:
    """A few output channels of the V, out-projection, FF1 and FF2 weights of every block 40x larger than the rest (the
    outlier channels of real checkpoints; q and k are left alone, where they would sharpen the softmax).  Recorded in
    DESIGN.md section 8: it does not separate the two FP8 modes, because the 64-column activation units that carry an
    outlier channel lose the same precision under either scaling."""
    g = torch.Generator().manual_seed(seed)
    W = dict(W)
    for i in range(cfg.depth):
        p = f"transformer.transformer_blocks.{i}."
        for name in ("attn.to_v", "attn.to_out.layers.0", "ff.ff.layers.0.layers.0", "ff.ff.layers.2"):
            w = W[p + name + ".weight"].clone()
            rows = torch.randperm(w.shape[0], generator=g)[:3]
            w[rows] *= 40.0
            W[p + name + ".weight"] = w
    return W


def outlier_inputs(B: int, N: int, seed: int = 3):
    """A construction that per-tensor scaling handles badly: noise whose first 24 frames are 3e5 times larger, so that
    in those rows the residual stream (and the fused-LN operand x (1 + s)) lies far beyond 448, where an unscaled e4m3
    activation saturates."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, N, 100, generator=g)
    x[:, :24] *= 3e5
    cond = torch.randn(B, N, 100, generator=g) * 2 - 1
    return x, cond
