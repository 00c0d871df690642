"""E2TTS_Base's UNetT (upstream F5-TTS f5_tts/model/backbones/unett.py, skip_connect_type "concat") restated test-side,
composed from the oracle's pieces (oracle/f5_oracle.py stays untouched).  Neither upstream's source nor a checkpoint is
available offline: this restatement of the model definition is what the CUDA path is checked against.

  * TimestepEmbedding, the text embedding (conv_layers = 0: a plain gather, no position table, filler rows unmasked) and
    InputEmbedding are the oracle's, reached through the MLX parameter names (weights.convert_upstream_keys);
  * the time token is row 0 of each utterance, the key mask gets a leading True, RoPE covers positions 0..n on the first
    pe_attn_head heads (v0_emul.head_rope);
  * layer i < depth/2 pushes x, layer i >= depth/2 pops (LIFO) and replaces x by skip_proj([x | skip]);
  * RMSNorm is x_transformers': F.normalize(x) * sqrt(D) * g.

`prec = O.Precision(True)` emulates the GPU's rounding points: bf16 GEMM operands, the folded weight bf16(W diag(g)) of
every Linear that consumes a norm with the row scale sqrt(D) / max(||x||, 1e-12) applied to the fp32 accumulator, fp32
elsewhere.  `skip_order` / `x_first` exist only to show that the pairing and the concat order matter.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn.functional as F

from oracle import f5_oracle as O
from v0_emul import head_rope


def rms_norm(x: torch.Tensor, g: torch.Tensor) -> torch.Tensor:
    """x_transformers.RMSNorm: F.normalize(x, dim=-1) * sqrt(D) * g."""
    return F.normalize(x, dim=-1) * math.sqrt(x.shape[-1]) * g


def rms_linear(x, g, w, b, prec: O.Precision = O.FP32):
    """Linear(RMSNorm(x)).  With bf16 emulation: bf16(x) @ bf16(W diag(g))^T * sqrt(D) / max(||x||, 1e-12) + b."""
    if not prec.emulate_bf16:
        return F.linear(rms_norm(x, g), w, b)
    scale = math.sqrt(x.shape[-1]) / x.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    out = F.linear(prec.op(x), prec.op(w * g[None, :])) * scale
    return out + b if b is not None else out


def attention(x, g, mask, rope, W, pfx, heads, prec: O.Precision = O.FP32):
    """upstream Attention on RMSNorm(x): to_q/k/v with bias, rotary on the table's heads, scale 1/8, key mask, to_out,
    padded rows' output zero (the oracle's attention with the norm folded into the projections)."""
    b, n, _ = x.shape
    q, k, v = (rms_linear(x, g, W[pfx + f"to_{c}.weight"], W[pfx + f"to_{c}.bias"], prec) for c in "qkv")
    q, k, v = (u.reshape(b, n, heads, -1).permute(0, 2, 1, 3) for u in (q, k, v))
    q = O.apply_rotary_pos_emb(q, rope, 1.0)
    k = O.apply_rotary_pos_emb(k, rope, 1.0)
    s = torch.matmul(prec.op(q / 8.0), prec.op(k).transpose(-1, -2))
    if mask is not None:
        s = s.masked_fill(~mask[:, None, None, :], float("-inf"))
    if prec.emulate_bf16:
        m = s.max(dim=-1, keepdim=True).values
        e = torch.exp(s - m)
        o = torch.matmul(prec.op(e), prec.op(v)) / e.sum(dim=-1, keepdim=True)
    else:
        o = torch.matmul(torch.softmax(s, dim=-1), v)
    o = o.permute(0, 2, 1, 3).reshape(b, n, -1)
    o = O.linear(prec.op(o), W[pfx + "to_out.0.weight"], W[pfx + "to_out.0.bias"], prec)
    if mask is not None:
        o = o * mask[:, :, None]
    return o


def ocfg(cfg) -> O.DiTConfig:
    """The oracle config of the pieces reused here (text embedding without ConvNeXt, unmasked)."""
    return O.DiTConfig(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult,
                       text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim, conv_layers=0,
                       text_mask_padding=False)


def unett_forward(x, cond, text, time, drop_audio_cond: bool, drop_text: bool, mask: Optional[torch.Tensor], W, cfg,
                  prec: O.Precision = O.FP32, skip_order: str = "lifo", x_first: bool = True, keep_time_row=False):
    """UNetT.forward of x, cond [b, n, mel], text [b, nt] (pad -1), time (scalar or [b]); W: upstream names."""
    from f5_tts_mlx_b200.weights import convert_upstream_keys
    M = convert_upstream_keys(W)            # the oracle's pieces read MLX names
    b, n = x.shape[:2]
    if time.ndim == 0:
        time = time.repeat(b)
    t = O.timestep_embedding(time.to(x.dtype), M)
    te = O.text_embedding(text, n, drop_text, M, ocfg(cfg), prec, mask_padding=False)
    h = O.input_embedding(x, cond, te, drop_audio_cond, M, prec)
    h = torch.cat([t[:, None].to(h.dtype), h], dim=1)                 # the time token at row 0
    mask1 = F.pad(mask, (1, 0), value=True) if mask is not None else None
    rope = head_rope(n + 1, cfg.heads, cfg.pe_attn_head, cfg.dim_head)
    skips = []
    T = "transformer."
    for i in range(cfg.depth):
        p = T + f"layers.{i}."
        if i < cfg.depth // 2:
            skips.append(h)
        else:
            s = skips.pop() if skip_order == "lifo" else skips.pop(0)
            h = O.linear(torch.cat([h, s] if x_first else [s, h], dim=-1), W[p + "0.weight"], None, prec)
        h = attention(h, W[p + "1.g"], mask1, rope, W, p + "2.", cfg.heads, prec) + h
        f = F.gelu(rms_linear(h, W[p + "3.g"], W[p + "4.ff.0.0.weight"], W[p + "4.ff.0.0.bias"], prec),
                   approximate="tanh")
        h = O.linear(f, W[p + "4.ff.2.weight"], W[p + "4.ff.2.bias"], prec) + h
    out = rms_linear(h, W[T + "norm_out.g"], W[T + "proj_out.weight"], W[T + "proj_out.bias"], prec)
    return out if keep_time_row else out[:, 1:]


def sample(cond, text, duration, W, cfg, *, steps: int = 8, method: str = "rk4", cfg_strength: float = 2.0,
           sway_sampling_coef: Optional[float] = -1.0, seed: Optional[int] = None, y0: Optional[torch.Tensor] = None,
           prec: O.Precision = O.FP32):
    """O.sample (cfm.py:264-402) on the UNetT forward: the same prologue, noise and solvers."""
    prep = O.sample_prologue(cond, text, duration, W)
    step_cond, txt, mask = prep.step_cond, prep.text, prep.mask

    def fn(t, x):
        pred = unett_forward(x, step_cond, txt, t, False, False, mask, W, cfg, prec)
        if cfg_strength < 1e-5:
            return pred
        null_pred = unett_forward(x, step_cond, txt, t, True, True, mask, W, cfg, prec)
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
