"""CPU emulation of the FP8 attention mode of the DiT (DiT(fp8=True, fp8_scaling="block", fp8_attention=True), DESIGN.md
section 8), composed from the block mode's emulation (fp8_block_emul), whose rounding points it keeps everywhere else.

The attention's rounding points:
  * q, k, v: the bf16 values the QKV GEMM writes (q rotated and scaled by 1/8, k rotated), quantised to e4m3 with the
    block mode's power-of-two rule: q with one scale per (row, head), k and v with one scale per (utterance, head,
    128-key tile) (the amax of the tile's 128 x 64 values);
  * S from the codes times the scales (exact in float64 here);
  * p = exp(S - m) and l = sum p in full precision (the kernel sums the fp32 p);
  * P~ = e4m3(2^8 p), and O = sum_t (sv_t / 2^8) P~_t V-codes_t / l;
  * the output quantised per (row, head), as in the block mode.

m here is the FINAL row max.  The kernel's online softmax forms P~ against the running max of the tiles seen so far and
rescales later, so a tile read before the row's max arrives rounds p exp(m - m_run) instead of p: the same relative
rounding (2^-4) on values up to exp(m - m_run) times larger, which moves only where P~ is near the e4m3 subnormal range.
The emulation takes the final max, the single-pass answer that does not depend on the tile order.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

import fp8_block_emul as E
from oracle import f5_oracle as O

BF16 = E.BF16
TILE = 128


def q_heads(x: torch.Tensor):
    """Per-(row, head) block-scaled e4m3 of [..., 64]: (codes as float64, scales [..., 1])."""
    s = E.block_scale(x.float().abs().amax(-1, keepdim=True))
    return E._quant(x.float(), s).double(), s.double()


def q_tiles(x: torch.Tensor, mask=None):
    """Per-(utterance, head, 128-key tile) block-scaled e4m3 of [b, h, n, 64]: (codes as float64, scales [b, h, n, 1],
    every key carrying its tile's scale).  mask [b, n] bool or None: masked keys are zero, so they neither move their
    tile's amax nor carry a code (the quantise pass reads keys at or beyond kv_len as zero)."""
    b, h, n, _ = x.shape
    x = x.float()
    if mask is not None:
        x = torch.where(mask.bool().to(x.device)[:, None, :, None], x, torch.zeros((), device=x.device))
    pad = (-n) % TILE
    a = F.pad(x.abs(), (0, 0, 0, pad)).reshape(b, h, (n + pad) // TILE, TILE * 64).amax(-1)
    s = E.block_scale(a).repeat_interleave(TILE, -1)[..., :n, None]
    return E._quant(x, s).double(), s.double()


def attention_fp8(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, mask, heads_per_chunk: int = 4) -> torch.Tensor:
    """q, k, v: [b, h, n, 64] bf16 values (q already scaled by 1/8); mask [b, n] bool or None -> O [b, h, n, 64].
    The float64 scores are formed `heads_per_chunk` heads at a time (a [b, h, n, n] tensor is 8 GB at n = 5625), on
    the GPU when there is one (the result returns to q's device)."""
    qc, sq = q_heads(q)
    kc, sk = q_tiles(k, mask)
    vc, sv = q_tiles(v, mask)
    b, h, n, _ = q.shape
    dev = "cuda" if torch.cuda.is_available() else "cpu"
    valid = (mask.bool() if mask is not None else torch.ones(b, n, dtype=torch.bool)).to(dev)
    out = torch.empty(b, h, n, q.shape[-1])
    for h0 in range(0, h, heads_per_chunk):
        c = lambda t: t[:, h0:h0 + heads_per_chunk].to(dev)
        s = (c(qc) @ c(kc).transpose(-1, -2)) * c(sq) * c(sk).transpose(-1, -2)
        s = s.masked_fill(~valid[:, None, None, :], float("-inf"))
        p = torch.exp(s - s.amax(-1, keepdim=True))
        pt = E._quant(p * 256.0, torch.ones((), device=dev)).double()
        o = pt @ (c(vc) * c(sv) / 256.0)    # sv is constant over each tile: sum_t (sv_t / 2^8) P~_t V-codes_t
        out[:, h0:h0 + heads_per_chunk] = (o / p.sum(-1, keepdim=True)).float().cpu()
    return out.to(q.device)


def attention8a(x, mask, rope, W, pfx, heads, scale_msa, shift_msa):
    b, n, _ = x.shape
    wqkv = torch.cat([W[pfx + f"to_{c}.weight"] for c in "qkv"], 0)
    bqkv = torch.cat([W[pfx + f"to_{c}.bias"] for c in "qkv"], 0)
    qkv = E.adaln8(x, scale_msa, shift_msa, wqkv, bqkv)
    q, k, v = qkv.chunk(3, dim=-1)
    q, k, v = [t.reshape(b, n, heads, -1).permute(0, 2, 1, 3) for t in (q, k, v)]
    q = O.apply_rotary_pos_emb(q, rope, 1.0)
    k = O.apply_rotary_pos_emb(k, rope, 1.0)
    o = attention_fp8(BF16.op(q / 8.0), BF16.op(k), BF16.op(v), mask)
    o = o.permute(0, 2, 1, 3).reshape(b, n, -1)
    o = E.linear8(E.q_rows(o), W[pfx + "to_out.layers.0.weight"], W[pfx + "to_out.layers.0.bias"])
    if mask is not None:
        o = o * mask[:, :, None]
    return o


def dit_block8a(x, t, mask, rope, W, i, cfg):
    p = f"transformer.transformer_blocks.{i}."
    emb = O.linear(F.silu(t), W[p + "attn_norm.linear.weight"], W[p + "attn_norm.linear.bias"], BF16)
    shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp = emb.chunk(6, dim=1)
    x = x + gate_msa[:, None] * attention8a(x, mask, rope, W, p + "attn.", cfg.heads, scale_msa, shift_msa)
    h = E.adaln8(x, scale_mlp, shift_mlp, W[p + "ff.ff.layers.0.layers.0.weight"], W[p + "ff.ff.layers.0.layers.0.bias"])
    h = F.gelu(h, approximate="tanh")
    ff = E.linear8(E.q_rows(h), W[p + "ff.ff.layers.2.weight"], W[p + "ff.ff.layers.2.bias"])
    return x + gate_mlp[:, None] * ff


def dit_forward_block8a(x, cond, text, time, drop_audio_cond, drop_text, mask, W, cfg):
    """oracle.dit_forward with the rounding points of the FP8 attention mode."""
    batch, seq_len = x.shape[0], x.shape[1]
    if time.ndim == 0:
        time = time.repeat(batch)
    t = O.timestep_embedding(time.float(), W)
    text_embed = O.text_embedding(text, seq_len, drop_text, W, cfg, BF16)
    x = O.input_embedding(x, cond, text_embed, drop_audio_cond, W, BF16)
    rope = O.rotary_freqs(seq_len, cfg.dim_head)
    for i in range(cfg.depth):
        x = dit_block8a(x, t, mask, rope, W, i, cfg)
    emb = O.linear(F.silu(t), W["transformer.norm_out.linear.weight"], W["transformer.norm_out.linear.bias"], BF16)
    scale, shift = emb.chunk(2, dim=1)
    return O.adaln_linear(x, scale, shift, W["transformer.proj_out.weight"], W["transformer.proj_out.bias"], BF16)
