"""F5TTS_Base (v0) restated test-side by composing the oracle (oracle/f5_oracle.py stays the fixed restatement of the
reference, which only has the v1 rotation).

v0 differs from v1 in two places:
  * TextEmbedding(mask_padding=False) (dit.py:182-229) — reference code, reached here through the oracle's own
    `text_embedding(mask_padding=False)` and pinned to the unmodified reference by tests/golden/ref_dit_v0.npz;
  * rotary embedding on the first `pe_attn_head` heads of q and k only (upstream's pe_attn_head; v0 = 1).  Upstream v0
    rotated the un-split [b, n, heads*64] q and k projections with a 64-wide table, so only their first 64 columns
    (head 0) turned.  The oracle's attention rotates every head with one [n, 64] table; a per-head [heads, n, 64] angle
    table whose rows past pe_attn_head are zero composes the v0 rotation from it exactly (cos 0 = 1, sin 0 = 0).
    `upstream_v0_attention` states the upstream form independently, for tests/test_v0.py to check the composition.
"""
from __future__ import annotations

import math
from typing import Callable, Optional

import torch
import torch.nn.functional as F

from oracle import f5_oracle as O


def head_rope(seq_len: int, heads: int, pe_attn_head: Optional[int], dim_head: int = 64) -> torch.Tensor:
    """[heads, seq_len, dim_head] rotary angles: the oracle's table for the first pe_attn_head heads (None: all), zero
    (the identity) for the rest.  O.apply_rotary_pos_emb slices the table's leading axis with [-seq_len:], which keeps
    every head as long as seq_len >= heads."""
    assert seq_len >= heads, "the per-head table needs seq_len >= heads (O.apply_rotary_pos_emb slices [-seq_len:])"
    t = O.rotary_freqs(seq_len, dim_head)[None].repeat(heads, 1, 1)
    if pe_attn_head is not None:
        t[pe_attn_head:] = 0.0
    return t


def oracle_block(prec: O.Precision = O.FP32) -> Callable:
    return lambda x, t, mask, rope, W, i, cfg: O.dit_block(x, t, mask, rope, W, i, cfg, prec)


def dit_forward(x, cond, text, time, drop_audio_cond: bool, drop_text: bool, mask, W, cfg: O.DiTConfig,
                prec: O.Precision = O.FP32, pe_attn_head: Optional[int] = None, block: Optional[Callable] = None):
    """O.dit_forward (dit.py:374-401) with TextEmbedding(mask_padding=cfg.text_mask_padding) and the rotation on the
    first pe_attn_head heads.  `block(x, t, mask, rope, W, i, cfg)`: the transformer block (default the oracle's at
    `prec`; the FP8 emulations pass theirs)."""
    block = block or oracle_block(prec)
    batch, seq_len = x.shape[0], x.shape[1]
    if time.ndim == 0:
        time = time.repeat(batch)
    t = O.timestep_embedding(time.float(), W)
    text_embed = O.text_embedding(text, seq_len, drop_text, W, cfg, prec, mask_padding=cfg.text_mask_padding)
    x = O.input_embedding(x, cond, text_embed, drop_audio_cond, W, prec)
    rope = head_rope(seq_len, cfg.heads, pe_attn_head, cfg.dim_head)
    for i in range(cfg.depth):
        x = block(x, t, mask, rope, W, i, cfg)
    emb = O.linear(F.silu(t), W["transformer.norm_out.linear.weight"], W["transformer.norm_out.linear.bias"], prec)
    scale, shift = emb.chunk(2, dim=1)
    return O.adaln_linear(x, scale, shift, W["transformer.proj_out.weight"], W["transformer.proj_out.bias"], prec)


def sample(cond, text, duration, W, cfg: O.DiTConfig, *, pe_attn_head: Optional[int] = None, steps: int = 8,
           method: str = "rk4", cfg_strength: float = 2.0, sway_sampling_coef: Optional[float] = -1.0,
           seed: Optional[int] = None, y0: Optional[torch.Tensor] = None, prec: O.Precision = O.FP32,
           block: Optional[Callable] = None):
    """O.sample (cfm.py:264-402) on the forward above; the same prologue, noise and solvers."""
    prep = O.sample_prologue(cond, text, duration, W)
    step_cond, txt, mask = prep.step_cond, prep.text, prep.mask

    def fn(t, x):
        pred = dit_forward(x, step_cond, txt, t, False, False, mask, W, cfg, prec, pe_attn_head, block)
        if cfg_strength < 1e-5:
            return pred
        null_pred = dit_forward(x, step_cond, txt, t, True, True, mask, W, cfg, prec, pe_attn_head, block)
        return pred + (pred - null_pred) * cfg_strength

    if y0 is None:
        ys = []
        for dur in prep.duration.tolist():
            gen = torch.Generator().manual_seed(seed if seed is not None else 0)
            ys.append(torch.randn(100, int(dur), generator=gen))
        y0 = O.pad_sequence(ys, padding_value=0).permute(0, 2, 1)
    t = O.time_grid(steps, sway_sampling_coef)
    solver = {"euler": O.odeint_euler, "midpoint": O.odeint_midpoint, "rk4": O.odeint_rk4}[method]
    trajectory = solver(fn, y0.float(), t)
    return torch.where(prep.cond_mask, prep.cond, trajectory[-1]), trajectory


def upstream_v0_attention(x: torch.Tensor, mask: Optional[torch.Tensor], W, pfx: str, heads: int) -> torch.Tensor:
    """Upstream v0's attention, stated independently of the per-head table: the un-split projections q, k [b, n, D] are
    rotated with the [n, 64] table, which turns their first 64 columns only; then the heads are split."""
    b, n, D = x.shape
    q = F.linear(x, W[pfx + "to_q.weight"], W[pfx + "to_q.bias"])
    k = F.linear(x, W[pfx + "to_k.weight"], W[pfx + "to_k.bias"])
    v = F.linear(x, W[pfx + "to_v.weight"], W[pfx + "to_v.bias"])
    freqs = O.rotary_freqs(n, 64)
    rot = lambda u: torch.cat([u[..., :64] * freqs.cos() + O.rotate_half(u[..., :64]) * freqs.sin(), u[..., 64:]], -1)
    q, k = rot(q), rot(k)
    q, k, v = [u.reshape(b, n, heads, -1).permute(0, 2, 1, 3) for u in (q, k, v)]
    s = torch.matmul(q, k.transpose(-1, -2)) / math.sqrt(q.shape[-1])
    if mask is not None:
        s = s.masked_fill(~mask[:, None, None, :], float("-inf"))
    o = torch.matmul(torch.softmax(s, dim=-1), v).permute(0, 2, 1, 3).reshape(b, n, D)
    o = F.linear(o, W[pfx + "to_out.layers.0.weight"], W[pfx + "to_out.layers.0.bias"])
    if mask is not None:
        o = o * mask[:, :, None]
    return o


def ocfg_v0(cfg, text_mask_padding: bool = False) -> O.DiTConfig:
    return O.DiTConfig(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult,
                       text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim, conv_layers=cfg.conv_layers,
                       text_mask_padding=text_mask_padding)
