"""CPU oracle for the f5-tts-mlx hot path — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A torch-CPU fp32 restatement of the reference's arithmetic, op for op, for the path
BASELINE.json names: F5TTS.sample() -> DiT forward (+ log-mel front-end, + Vocos back-end).
Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` legs
may import this module.  The product package (f5_tts_mlx_b200) never does.

PARITY UNPINNED: the reference ships no tests, golden vectors or fixtures for this path
and its runtime (mlx, vocos-mlx) is not installable in this image, so this
restatement cannot be checked against outputs of the reference itself.  It is pinned instead
against independent library implementations of the same operators (torchaudio MelSpectrogram,
torch.nn.functional conv1d / layer_norm / scaled_dot_product_attention / gelu / mish, torch.istft)
in tests/test_oracle_*.py.

Every function cites the reference lines (relative to /root/reference/f5_tts_mlx/) it follows,
INCLUDING the reference's inefficiencies (two unbatched CFG passes per evaluation, text embedding
recomputed on every forward, AdaLN linears recomputed per block per forward, full trajectory kept),
because the same code is the CPU baseline that bench.py times.

Weights are a flat dict name -> torch.Tensor using the MLX parameter-tree names and MLX layouts
(Linear: (out, in); Conv1d: (out, k, in/groups)).

`emulate_bf16=True` rounds every tensor-core operand (GEMM/conv inputs and weights, q/k/v, softmax
probabilities, attention output) to bf16 while accumulating in fp32 — the precision model of the
CUDA path — and is used to DERIVE the parity tolerance rather than guess it.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from functools import lru_cache
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

Tensor = torch.Tensor
Weights = Dict[str, Tensor]


# ---------------------------------------------------------------------------------------------
# precision model
# ---------------------------------------------------------------------------------------------
class Precision:
    """fp32 everywhere (the reference), or bf16-rounded tensor-core operands (the CUDA path)."""

    def __init__(self, emulate_bf16: bool = False, ln_by_linearity: bool = False, fp8: bool = False):
        self.emulate_bf16 = emulate_bf16
        # rounding points of the CUDA path's fused AdaLN (see adaln_linear below); only meaningful with emulate_bf16
        self.ln_by_linearity = ln_by_linearity
        # FP8 mode of the CUDA path (DiT(fp8=True)): the four GEMMs of every DiT block multiply e4m3 operands — weights
        # quantised per tensor (scale = max|w| / 448), activations rounded to e4m3 by the producing kernel (no scale)
        self.fp8 = fp8

    @staticmethod
    def e4m3(x: Tensor) -> Tensor:
        return x.clamp(-448.0, 448.0).to(torch.float8_e4m3fn).float()

    def op(self, x: Tensor) -> Tensor:
        return x.bfloat16().float() if self.emulate_bf16 else x


FP32 = Precision(False)


def linear(x: Tensor, w: Tensor, b: Optional[Tensor], prec: Precision = FP32) -> Tensor:
    """mlx.nn.Linear: x @ W^T + b."""
    return F.linear(prec.op(x), prec.op(w), b)


def adaln_linear(x: Tensor, scale: Tensor, shift: Tensor, w: Tensor, b: Optional[Tensor], prec: Precision = FP32,
                 eps: float = 1e-6, fp8_scale: Optional[float] = None) -> Tensor:
    """Linear(LayerNorm(x) * (1 + scale) + shift) — dit.py:270 + the Linear that consumes it (dit.py:136-143, 94,
    398).  fp32: exactly that.  With `prec.ln_by_linearity` it applies the CUDA path's operand rounding point: the
    producer GEMM's epilogue stores bf16(x * (1 + scale)) and the consumer GEMM multiplies that operand and finishes
    the LayerNorm in its epilogue by linearity,
        out = rstd * (x~ @ W^T - mean * c1) + c2,   c1 = (1 + scale) @ W^T,  c2 = shift @ W^T + b   (fp32 tables).
    The mean and rstd here are exact two-pass statistics of x.  The kernels do not compute those: the producer stores
    the fp32 (sum, sum of squares) of every 64-column unit and the consumer forms var = E[x^2] - mean^2 from them,
    whose error grows like r^2 with r = |mean| / std (tests/adaln_emul.py emulates that; below r ~ 1000 at D = 1024
    the operand rounding, which this emulation does include, dominates)."""
    d = x.shape[-1]
    if not (prec.emulate_bf16 and prec.ln_by_linearity):
        norm = F.layer_norm(x, (d,), eps=eps) * (1 + scale[:, None]) + shift[:, None]
        return linear(norm, w, b, prec)
    mu = x.mean(dim=-1, keepdim=True)
    rstd = torch.rsqrt(x.var(dim=-1, unbiased=False, keepdim=True) + eps)
    wb = prec.op(w)
    xt = prec.op(x * (1 + scale[:, None]))
    c1 = F.linear(1 + scale, wb)[:, None]          # the tables always come from the bf16 weights
    c2 = F.linear(shift, wb, b)[:, None]
    if prec.fp8 and fp8_scale is not None:
        # FP8 mode: e4m3 activation (unscaled) x e4m3 weight (per-tensor scale), fp32 accumulation
        acc = F.linear(Precision.e4m3(x * (1 + scale[:, None])), Precision.e4m3(w / fp8_scale)) * fp8_scale
        return rstd * (acc - mu * c1) + c2
    return rstd * (F.linear(xt, wb) - mu * c1) + c2


def conv1d_nlc(x: Tensor, w_mlx: Tensor, b: Optional[Tensor], padding: int, groups: int,
               prec: Precision = FP32) -> Tensor:
    """mlx.nn.Conv1d on channels-last input (b, n, c) with MLX weight layout (out, k, in/groups),
    zero padding."""
    w = w_mlx.permute(0, 2, 1)  # -> torch (out, in/groups, k)
    y = F.conv1d(prec.op(x).transpose(1, 2), prec.op(w), b, padding=padding, groups=groups)
    return y.transpose(1, 2)


# ---------------------------------------------------------------------------------------------
# utils.py
# ---------------------------------------------------------------------------------------------
def lens_to_mask(t: Tensor, length: Optional[int] = None) -> Tensor:
    """utils.py:39-47 — mask[b, n] = n < t[b]."""
    if length is None:
        length = int(t.max().item())
    seq = torch.arange(length)
    return seq[None, :] < t[:, None]


def pad_to_length(t: Tensor, length: int, value=0) -> Tensor:
    """utils.py:93-103."""
    seq_len = t.shape[-1]
    if length > seq_len:
        t = F.pad(t, (0, length - seq_len), value=value)
    return t[..., :length]


def pad_sequence(ts: Sequence[Tensor], padding_value=0) -> Tensor:
    """utils.py:106-109."""
    max_len = max(i.shape[-1] for i in ts)
    return torch.stack([pad_to_length(i, max_len, padding_value) for i in ts])


def list_str_to_tensor(text: List[str], padding_value=-1) -> Tensor:
    """utils.py:115-118 — utf-8 byte tokenizer."""
    ts = [torch.tensor([*bytes(t, "UTF-8")], dtype=torch.int32) for t in text]
    return pad_sequence(ts, padding_value=-1)


def list_str_to_idx(text: List[Sequence[str]], vocab_char_map: Dict[str, int], padding_value=-1) -> Tensor:
    """utils.py:124-133 — char tokenizer, unknown -> 0, pad -1."""
    ts = [torch.tensor([vocab_char_map.get(c, 0) for c in t], dtype=torch.int32) for t in text]
    return pad_sequence(ts, padding_value=padding_value)


# ---------------------------------------------------------------------------------------------
# audio.py
# ---------------------------------------------------------------------------------------------
@lru_cache(maxsize=None)
def mel_filters(sample_rate: int, n_fft: int, n_mels: int) -> Tensor:
    """audio.py:12-98 with norm=None, mel_scale='htk' (the only mode the path uses, audio.py:187-189).
    Returns (n_mels, n_fft//2+1)."""
    def hz_to_mel(f):
        return 2595.0 * math.log10(1.0 + f / 700.0)

    f_max = sample_rate / 2
    n_freqs = n_fft // 2 + 1
    all_freqs = torch.linspace(0, sample_rate // 2, n_freqs, dtype=torch.float32)       # :70
    m_pts = torch.linspace(hz_to_mel(0.0), hz_to_mel(f_max), n_mels + 2, dtype=torch.float32)  # :74-76
    f_pts = 700.0 * (10.0 ** (m_pts / 2595.0) - 1.0)                                    # :77
    f_diff = f_pts[1:] - f_pts[:-1]                                                    # :81
    slopes = f_pts[None, :] - all_freqs[:, None]                                       # :82
    down = (-slopes[:, :-2]) / f_diff[:-1]                                             # :86
    up = slopes[:, 2:] / f_diff[1:]                                                    # :87
    fb = torch.clamp(torch.minimum(down, up), min=0.0)                                 # :88-90
    return fb.T.contiguous()                                                           # :96 moveaxis


@lru_cache(maxsize=None)
def hanning(size: int) -> Tensor:
    """audio.py:101-112 — np.hanning(size+1)[:-1] (periodic Hann)."""
    return torch.from_numpy(np.hanning(size + 1)[:-1].astype(np.float32))


def stft(x: Tensor, window: Tensor, nperseg: int, noverlap: int) -> Tensor:
    """audio.py:115-159 — zero ('constant') centre padding, frames at hop `noverlap`, rfft."""
    nfft = nperseg
    padding = nperseg // 2
    x = F.pad(x, (padding, padding))                       # :143-153
    t = (x.numel() - nperseg + noverlap) // noverlap       # :156
    frames = x.unfold(0, nfft, noverlap)[:t]               # :158 as_strided
    return torch.fft.rfft(frames * window)                 # :159


def log_mel_spectrogram(audio: Tensor, sample_rate=24_000, n_mels=100, n_fft=1024, hop_length=256) -> Tensor:
    """audio.py:162-210 — returns (b, frames, n_mels) (frames-major)."""
    if audio.ndim == 1:
        audio = audio[None]
    filters = mel_filters(sample_rate, n_fft, n_mels)
    outs = []
    for i in range(audio.shape[0]):
        freqs = stft(audio[i].float(), hanning(n_fft), nperseg=n_fft, noverlap=hop_length)
        magnitudes = freqs[:-1, :].abs()                   # :203 drops the last frame
        mel_spec = magnitudes @ filters.T                  # :205
        outs.append(torch.clamp(mel_spec, min=1e-5).log())  # :206
    return torch.stack(outs, 0)


# ---------------------------------------------------------------------------------------------
# rope.py
# ---------------------------------------------------------------------------------------------
def rotary_freqs(seq_len: int, dim: int = 64, base: float = 10000.0) -> Tensor:
    """rope.py:12-53 — forward_from_seq_len: freqs[n] = [nθ0,nθ0,nθ1,nθ1,...] (N, dim); xpos off."""
    inv_freq = 1.0 / (base ** (torch.arange(0, dim, 2, dtype=torch.float32) / dim))   # :24
    t = torch.arange(seq_len, dtype=torch.float32)
    freqs = torch.einsum("i,j->ij", t, inv_freq)                                      # :45-47
    return torch.stack((freqs, freqs), dim=-1).reshape(seq_len, dim)                  # :49-50


def precompute_freqs_cis(dim: int, end: int, theta: float = 10000.0) -> Tensor:
    """rope.py:63-73 — text positional table [cos | sin] (end, dim)."""
    freqs = 1.0 / (theta ** (torch.arange(0, dim, 2)[: dim // 2].float() / dim))
    t = torch.arange(end, dtype=torch.float32)
    freqs = torch.outer(t, freqs).float()
    return torch.cat([freqs.cos(), freqs.sin()], dim=-1)


def get_pos_embed_indices(start: Tensor, length: int, max_pos: int, scale: float = 1.0) -> Tensor:
    """rope.py:76-84 — positions clamped to max_pos-1."""
    sc = scale * torch.ones_like(start, dtype=torch.float32)
    pos = start[:, None] + (torch.arange(length)[None, :] * sc[:, None]).to(torch.int32)
    return torch.where(pos < max_pos, pos, torch.full_like(pos, max_pos - 1))


def rotate_half(x: Tensor) -> Tensor:
    """rope.py:87-91 — (x0,x1) -> (-x1,x0) on adjacent pairs."""
    x = x.reshape(*x.shape[:-1], -1, 2)
    x1, x2 = x[..., 0], x[..., 1]
    return torch.stack([-x2, x1], dim=-1).reshape(*x.shape[:-2], -1)


def apply_rotary_pos_emb(t: Tensor, freqs: Tensor, scale: float = 1.0) -> Tensor:
    """rope.py:94-107."""
    rot_dim, seq_len = freqs.shape[-1], t.shape[-2]
    freqs = freqs[-seq_len:, :]
    t_rot, t_un = t[..., :rot_dim], t[..., rot_dim:]
    t_rot = (t_rot * freqs.cos() * scale) + (rotate_half(t_rot) * freqs.sin() * scale)
    return torch.cat((t_rot, t_un), dim=-1)


# ---------------------------------------------------------------------------------------------
# convnext_v2.py
# ---------------------------------------------------------------------------------------------
def grn(x: Tensor, gamma: Tensor, beta: Tensor) -> Tensor:
    """convnext_v2.py:15-18 — L2 norm over the sequence axis (axis=1), INCLUDING padded rows."""
    Gx = torch.linalg.norm(x, ord=2, dim=1, keepdim=True)
    Nx = Gx / (Gx.mean(dim=-1, keepdim=True) + 1e-6)
    return gamma * (x * Nx) + beta + x


def convnext_v2_block(x: Tensor, W: Weights, pfx: str, prec: Precision = FP32) -> Tensor:
    """convnext_v2.py:46-54 (dilation 1, k=7, pad 3, groups=dim)."""
    dim = x.shape[-1]
    residual = x
    x = conv1d_nlc(x, W[pfx + "dwconv.weight"], W[pfx + "dwconv.bias"], padding=3, groups=dim)   # fp32 in the CUDA path too
    x = F.layer_norm(x, (dim,), W[pfx + "norm.weight"], W[pfx + "norm.bias"], eps=1e-6)
    x = linear(x, W[pfx + "pwconv1.weight"], W[pfx + "pwconv1.bias"], prec)
    x = F.gelu(x)                                     # nn.GELU() exact erf
    x = prec.op(x)                                    # the CUDA path stores this activation in bf16
    x = grn(x, W[pfx + "grn.gamma"], W[pfx + "grn.beta"])
    x = linear(x, W[pfx + "pwconv2.weight"], W[pfx + "pwconv2.bias"], prec)
    return residual + x


# ---------------------------------------------------------------------------------------------
# dit.py
# ---------------------------------------------------------------------------------------------
@dataclass
class DiTConfig:
    dim: int = 1024
    depth: int = 22
    heads: int = 16
    dim_head: int = 64
    ff_mult: int = 2
    mel_dim: int = 100
    text_num_embeds: int = 2545
    text_dim: int = 512
    conv_layers: int = 4
    text_mask_padding: bool = True


def sinus_position_embedding(x: Tensor, dim: int = 256, scale: float = 1000.0) -> Tensor:
    """dit.py:56-67."""
    half = dim // 2
    emb = math.log(10000) / (half - 1)
    emb = torch.exp(torch.arange(half, dtype=torch.float32) * -emb)
    emb = scale * x[:, None] * emb[None, :]
    return torch.cat([emb.sin(), emb.cos()], dim=-1)


def timestep_embedding(time: Tensor, W: Weights) -> Tensor:
    """dit.py:73-82 — fp32 in both precision models (tiny)."""
    h = sinus_position_embedding(time)
    h = linear(h, W["transformer.time_embed.time_mlp.layers.0.weight"], W["transformer.time_embed.time_mlp.layers.0.bias"])
    h = F.silu(h)
    return linear(h, W["transformer.time_embed.time_mlp.layers.2.weight"], W["transformer.time_embed.time_mlp.layers.2.bias"])


def text_embedding(text: Tensor, seq_len: int, drop_text: bool, W: Weights, cfg: DiTConfig,
                   prec: Precision = FP32, prefix: str = "transformer.", mask_padding: bool = True) -> Tensor:
    """dit.py:196-229 (mask_padding=False is how DurationTransformer builds it, duration.py:118-120)."""
    batch, text_len = text.shape
    text = text + 1                                                     # :200
    text = text[:, :seq_len]                                            # :203
    text = F.pad(text, (0, max(seq_len - text_len, 0)), value=0)        # :205
    text_mask = (text == 0)[..., None]                                  # :207 (before the drop)
    if drop_text:
        text = torch.zeros_like(text)                                   # :210
    x = W[prefix + "text_embed.text_embed.weight"][text.long()]          # :211
    if cfg.conv_layers > 0:
        max_pos = 4096                                                  # :190
        table = precompute_freqs_cis(cfg.text_dim, max_pos)
        pos_idx = get_pos_embed_indices(torch.zeros(batch, dtype=torch.int32), seq_len, max_pos)
        x = x + table[pos_idx.long()]                                   # :216-218
        if mask_padding:
            x = torch.where(text_mask, torch.zeros_like(x), x)          # :222
        for i in range(cfg.conv_layers):
            x = convnext_v2_block(x, W, prefix + f"text_embed.text_blocks.layers.{i}.", prec)
            if mask_padding:
                x = torch.where(text_mask, torch.zeros_like(x), x)      # :223-225 (else :227)
    return x


def conv_position_embedding(x: Tensor, W: Weights, prec: Precision = FP32, prefix: str = "transformer.") -> Tensor:
    """dit.py:29-50 with mask=None (dit.py:251): Conv1d(k31,g16) Mish Conv1d Mish."""
    p = prefix + "input_embed.conv_pos_embed.conv1d.layers."
    h = F.mish(conv1d_nlc(x, W[p + "0.weight"], W[p + "0.bias"], padding=15, groups=16, prec=prec))
    return F.mish(conv1d_nlc(h, W[p + "2.weight"], W[p + "2.bias"], padding=15, groups=16, prec=prec))


def input_embedding(x: Tensor, cond: Tensor, text_embed: Tensor, drop_audio_cond: bool, W: Weights,
                    prec: Precision = FP32) -> Tensor:
    """dit.py:241-252."""
    if drop_audio_cond:
        cond = torch.zeros_like(cond)
    h = linear(torch.cat((x, cond, text_embed), dim=-1), W["transformer.input_embed.proj.weight"],
               W["transformer.input_embed.proj.bias"], prec)
    return conv_position_embedding(h, W, prec) + h


def attention(x: Tensor, mask: Optional[Tensor], rope: Tensor, W: Weights, pfx: str, heads: int,
              prec: Precision = FP32, adaln: Optional[Tuple[Tensor, Tensor]] = None) -> Tensor:
    """dit.py:126-175.  `mask` (b, n) bool = key-padding mask with the INTENDED semantics of
    dit.py:161-166 (the reference's `.expand` call is not an mx.array method)."""
    b, n, _ = x.shape
    if adaln is not None:   # x is the un-normalised stream; AdaLayerNormZero (dit.py:270) feeds to_q/k/v (dit.py:313-316)
        s8 = None
        if prec.fp8:        # ONE scale for the fused [3D, D] weight, as the CUDA pack quantises it
            s8 = max(float(W[pfx + f"to_{n}.weight"].abs().max()) for n in "qkv") / 448.0
        lin = lambda w, bb: adaln_linear(x, adaln[0], adaln[1], w, bb, prec, fp8_scale=s8)
    else:
        lin = lambda w, bb: linear(x, w, bb, prec)
    q = lin(W[pfx + "to_q.weight"], W[pfx + "to_q.bias"])
    k = lin(W[pfx + "to_k.weight"], W[pfx + "to_k.bias"])
    v = lin(W[pfx + "to_v.weight"], W[pfx + "to_v.bias"])
    q = q.reshape(b, n, heads, -1).permute(0, 2, 1, 3)
    k = k.reshape(b, n, heads, -1).permute(0, 2, 1, 3)
    v = v.reshape(b, n, heads, -1).permute(0, 2, 1, 3)
    q = apply_rotary_pos_emb(q, rope, 1.0)
    k = apply_rotary_pos_emb(k, rope, 1.0)
    scale = 1.0 / math.sqrt(q.shape[-1])
    # mx.fast.scaled_dot_product_attention(scale=..., mask=bool key mask); fp32 softmax
    s = torch.matmul(prec.op(q * scale), prec.op(k).transpose(-1, -2))
    if mask is not None:
        s = s.masked_fill(~mask[:, None, None, :], float("-inf"))
    p = torch.softmax(s, dim=-1)
    if prec.emulate_bf16:
        # flash-attention order of operations: un-normalised bf16 probabilities, fp32 row sum
        m = s.max(dim=-1, keepdim=True).values
        e = torch.exp(s - m)
        o = torch.matmul(prec.op(e), prec.op(v)) / e.sum(dim=-1, keepdim=True)
    else:
        o = torch.matmul(p, v)
    o = o.permute(0, 2, 1, 3).reshape(b, n, -1)
    if prec.fp8:   # FP8 mode: the attention output leaves the kernel as e4m3, the out-projection weight is e4m3 (per tensor)
        wo = W[pfx + "to_out.layers.0.weight"]
        so = float(wo.abs().max()) / 448.0
        o = F.linear(Precision.e4m3(o), Precision.e4m3(wo / so)) * so + W[pfx + "to_out.layers.0.bias"]
    else:
        o = linear(prec.op(o), W[pfx + "to_out.layers.0.weight"], W[pfx + "to_out.layers.0.bias"], prec)
    if mask is not None:
        o = o * mask[:, :, None]                                          # :172-173
    return o


def dit_block(x: Tensor, t: Tensor, mask: Optional[Tensor], rope: Tensor, W: Weights, i: int,
              cfg: DiTConfig, prec: Precision = FP32) -> Tensor:
    """dit.py:311-325 with AdaLayerNormZero dit.py:266-271 and FeedForward dit.py:88-99."""
    p = f"transformer.transformer_blocks.{i}."
    dim = cfg.dim
    emb = linear(F.silu(t), W[p + "attn_norm.linear.weight"], W[p + "attn_norm.linear.bias"], prec)
    shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp = emb.chunk(6, dim=1)
    attn_out = attention(x, mask, rope, W, p + "attn.", cfg.heads, prec, adaln=(scale_msa, shift_msa))
    x = x + gate_msa[:, None] * attn_out
    w1 = W[p + "ff.ff.layers.0.layers.0.weight"]
    h = adaln_linear(x, scale_mlp, shift_mlp, w1, W[p + "ff.ff.layers.0.layers.0.bias"], prec,
                     fp8_scale=(float(w1.abs().max()) / 448.0) if prec.fp8 else None)
    h = F.gelu(h, approximate="tanh")
    if prec.fp8:   # FF1's epilogue writes e4m3, FF2's weight is e4m3 (per tensor)
        w2 = W[p + "ff.ff.layers.2.weight"]
        s2 = float(w2.abs().max()) / 448.0
        ff = F.linear(Precision.e4m3(h), Precision.e4m3(w2 / s2)) * s2 + W[p + "ff.ff.layers.2.bias"]
    else:
        ff = linear(h, W[p + "ff.ff.layers.2.weight"], W[p + "ff.ff.layers.2.bias"], prec)
    return x + gate_mlp[:, None] * ff


def dit_forward(x: Tensor, cond: Tensor, text: Tensor, time: Tensor, drop_audio_cond: bool,
                drop_text: bool, mask: Optional[Tensor], W: Weights, cfg: DiTConfig,
                prec: Precision = FP32) -> Tensor:
    """dit.py:374-401."""
    batch, seq_len = x.shape[0], x.shape[1]
    if time.ndim == 0:
        time = time.repeat(batch)                                          # :385-386
    t = timestep_embedding(time.float(), W)                                # :389
    text_embed = text_embedding(text, seq_len, drop_text, W, cfg, prec)    # :390 (recomputed each call)
    x = input_embedding(x, cond, text_embed, drop_audio_cond, W, prec)     # :391
    rope = rotary_freqs(seq_len, cfg.dim_head)                             # :393
    for i in range(cfg.depth):
        x = dit_block(x, t, mask, rope, W, i, cfg, prec)                   # :395-396
    emb = linear(F.silu(t), W["transformer.norm_out.linear.weight"], W["transformer.norm_out.linear.bias"], prec)
    scale, shift = emb.chunk(2, dim=1)                                     # dit.py:287 (scale FIRST)
    return adaln_linear(x, scale, shift, W["transformer.proj_out.weight"], W["transformer.proj_out.bias"], prec)


# ---------------------------------------------------------------------------------------------
# duration.py — DurationPredictor: runs once before the ODE loop when
# `duration=None` (cfm.py:253-262, 307-308).
# ---------------------------------------------------------------------------------------------
@dataclass
class DurationConfig:
    dim: int = 512
    depth: int = 8
    heads: int = 8
    dim_head: int = 64
    ff_mult: int = 2
    mel_dim: int = 100
    text_num_embeds: int = 2545
    text_dim: int = 512
    conv_layers: int = 2

    def as_dit(self) -> "DiTConfig":
        return DiTConfig(dim=self.dim, depth=self.depth, heads=self.heads, dim_head=self.dim_head, ff_mult=self.ff_mult,
                         mel_dim=self.mel_dim, text_num_embeds=self.text_num_embeds, text_dim=self.text_dim,
                         conv_layers=self.conv_layers)


def duration_transformer(x: Tensor, text: Tensor, W: Weights, cfg: DurationConfig, prec: Precision = FP32) -> Tensor:
    """duration.py:133-158.  Note: DurationPredictor calls it WITHOUT a mask (duration.py:245), so the
    attention is unmasked; TextEmbedding is built with mask_padding=False."""
    P = "duration.transformer."
    b, n, _ = x.shape
    text_embed = text_embedding(text, n, False, W, cfg.as_dit(), prec, prefix=P, mask_padding=False)
    h = linear(torch.cat((x, text_embed), dim=-1), W[P + "input_embed.proj.weight"], W[P + "input_embed.proj.bias"], prec)
    h = conv_position_embedding(h, W, prec, prefix=P) + h                       # duration.py:55-57
    rope = rotary_freqs(n, cfg.dim_head)
    for i in range(cfg.depth):                                                   # duration.py:81-94
        p = P + f"transformer_blocks.{i}."
        norm = F.layer_norm(h, (cfg.dim,), eps=1e-6)
        h = h + attention(norm, None, rope, W, p + "attn.", cfg.heads, prec)
        norm = F.layer_norm(h, (cfg.dim,), eps=1e-6)
        f = linear(norm, W[p + "ff.ff.layers.0.layers.0.weight"], W[p + "ff.ff.layers.0.layers.0.bias"], prec)
        f = F.gelu(f, approximate="tanh")
        h = h + linear(f, W[p + "ff.ff.layers.2.weight"], W[p + "ff.ff.layers.2.bias"], prec)
    # nn.RMSNorm(dim): x * rsqrt(mean(x^2) + 1e-5) * weight
    return h * torch.rsqrt(h.pow(2).mean(dim=-1, keepdim=True) + 1e-5) * W[P + "norm_out.weight"]


def duration_predictor(inp: Tensor, text: Tensor, W: Weights, cfg: DurationConfig, lens: Optional[Tensor] = None,
                       prec: Precision = FP32) -> Tensor:
    """duration.py:198-253 (inference branch): mel (b, n, 100) -> seconds (b,)."""
    batch, seq_len = inp.shape[:2]
    if seq_len < text.shape[1]:                                                  # :218-220
        seq_len = text.shape[1]
        inp = F.pad(inp, (0, 0, 0, seq_len - inp.shape[1]))
    if lens is None:
        lens = torch.full((batch,), seq_len)                                     # :224-225
    mask = lens_to_mask(lens, length=seq_len)                                    # :231
    inp = torch.where(mask[..., None], inp, torch.zeros_like(inp))               # :241-243
    x = duration_transformer(inp, text, W, cfg, prec)                            # :245 (no mask passed)
    x = torch.where(mask[..., None], x, torch.zeros_like(x))                     # maybe_masked_mean utils.py:82-90
    x = x.sum(dim=1) / mask.sum(dim=1).clamp(min=1)[:, None]
    return F.softplus(linear(x, W["duration.to_pred.layers.0.weight"], None, prec))[..., 0]   # :187-189


# ---------------------------------------------------------------------------------------------
# cfm.py — solvers and sample()
# ---------------------------------------------------------------------------------------------
def odeint_euler(func: Callable, y0: Tensor, t: Tensor) -> Tensor:
    """cfm.py:38-61."""
    ys = [y0]
    y = y0
    for i in range(len(t) - 1):
        dt = t[i + 1] - t[i]
        y = y + dt * func(t[i], y)
        ys.append(y)
    return torch.stack(ys)


def odeint_midpoint(func: Callable, y0: Tensor, t: Tensor) -> Tensor:
    """cfm.py:64-91."""
    ys = [y0]
    y = y0
    for i in range(len(t) - 1):
        dt = t[i + 1] - t[i]
        k1 = func(t[i], y)
        mid = y + 0.5 * dt * k1
        k2 = func(t[i] + 0.5 * dt, mid)
        y = y + dt * k2
        ys.append(y)
    return torch.stack(ys)


def odeint_rk4(func: Callable, y0: Tensor, t: Tensor) -> Tensor:
    """cfm.py:94-122."""
    ys = [y0]
    y = y0
    for i in range(len(t) - 1):
        dt = t[i + 1] - t[i]
        k1 = func(t[i], y)
        k2 = func(t[i] + 0.5 * dt, y + 0.5 * dt * k1)
        k3 = func(t[i] + 0.5 * dt, y + 0.5 * dt * k2)
        k4 = func(t[i] + dt, y + dt * k3)
        y = y + (dt / 6) * (k1 + 2 * k2 + 2 * k3 + k4)
        ys.append(y)
    return torch.stack(ys)


def time_grid(steps: int, sway_sampling_coef: Optional[float]) -> Tensor:
    """cfm.py:377-381 — `steps` is the number of GRID POINTS (steps-1 intervals)."""
    t = torch.linspace(0, 1, steps, dtype=torch.float32)
    if sway_sampling_coef is not None:
        t = t + sway_sampling_coef * (torch.cos(math.pi / 2 * t) - 1 + t)
    return t


@dataclass
class SamplePrep:
    cond: Tensor          # (b, N, 100) padded
    cond_mask: Tensor     # (b, N, 1) bool
    step_cond: Tensor     # (b, N, 100)
    text: Tensor          # (b, nt) int
    duration: Tensor      # (b,) int64
    mask: Optional[Tensor]  # (b, N) bool or None


def sample_prologue(cond: Tensor, text, duration, W: Weights, *, lens: Optional[Tensor] = None,
                    vocab_char_map: Optional[Dict[str, int]] = None, max_duration: int = 4096,
                    duration_predictor: Optional[Callable] = None, speed: float = 1.0) -> SamplePrep:
    """cfm.py:279-336."""
    if cond.ndim == 2:                                                     # raw wave :283-286
        assert cond.shape[0] == 1
        cond = log_mel_spectrogram(cond[0])
        assert cond.shape[-1] == 100
    batch, cond_seq_len = cond.shape[:2]
    if lens is None:
        lens = torch.full((batch,), cond_seq_len, dtype=torch.float32)     # :288-290
    if isinstance(text, list):                                             # :294-299
        text = list_str_to_idx(text, vocab_char_map) if vocab_char_map is not None else list_str_to_tensor(text)
        assert text.shape[0] == batch
    if text is not None:
        text_lens = (text != -1).sum(dim=-1)
        lens = torch.maximum(text_lens.to(lens.dtype), lens)               # :301-303
    if duration is None and duration_predictor is not None:
        duration = duration_predictor(cond, text, speed)
    elif duration is None:
        raise ValueError("Duration must be provided or a duration predictor must be set.")  # :309-310
    cond_mask = lens_to_mask(lens)                                         # :312
    if isinstance(duration, int):
        duration = torch.full((batch,), duration, dtype=lens.dtype)
    duration = torch.maximum(lens + 1, duration.to(lens.dtype))            # :317
    duration = torch.clip(duration, 0, max_duration)                       # :318
    N = int(duration.max().item())                                         # :319
    cond = F.pad(cond, (0, 0, 0, N - cond_seq_len))                        # :321
    cond_mask = F.pad(cond_mask, (0, N - cond_mask.shape[-1]), value=False)[..., None]
    step_cond = torch.where(cond_mask, cond, torch.zeros_like(cond))       # :331
    mask = lens_to_mask(duration) if batch > 1 else None                   # :333-336
    return SamplePrep(cond, cond_mask, step_cond, text, duration.long(), mask)


def sample(cond: Tensor, text, duration, W: Weights, cfg: DiTConfig, *, lens: Optional[Tensor] = None,
           steps: int = 8, method: str = "rk4", cfg_strength: float = 2.0, speed: float = 1.0,
           sway_sampling_coef: Optional[float] = -1.0, seed: Optional[int] = None,
           max_duration: int = 4096, y0: Optional[Tensor] = None,
           vocab_char_map: Optional[Dict[str, int]] = None, vocoder: Optional[Callable] = None,
           prec: Precision = FP32, cfg_batched: bool = False) -> Tuple[Tensor, Tensor]:
    """cfm.py:264-402.  Returns (out, trajectory) exactly like the reference.

    `y0` injects the initial noise (b, N, 100): MLX's threefry stream cannot be reproduced without
    MLX, so "identical seeds" parity is defined on injected noise.  Without `y0` a
    torch generator is seeded per element like cfm.py:369-375 (same seed for every element, noise
    drawn as (100, dur) then transposed)."""
    prep = sample_prologue(cond, text, duration, W, lens=lens, vocab_char_map=vocab_char_map,
                           max_duration=max_duration)
    step_cond, txt, mask = prep.step_cond, prep.text, prep.mask

    def fn(t, x):                                                          # :340-365
        pred = dit_forward(x, step_cond, txt, t, False, False, mask, W, cfg, prec)
        if cfg_strength < 1e-5:
            return pred
        null_pred = dit_forward(x, step_cond, txt, t, True, True, mask, W, cfg, prec)
        return pred + (pred - null_pred) * cfg_strength

    if y0 is None:                                                         # :369-375
        ys = []
        for dur in prep.duration.tolist():
            gen = torch.Generator().manual_seed(seed if seed is not None else 0)
            ys.append(torch.randn(100, int(dur), generator=gen))
        y0 = pad_sequence(ys, padding_value=0).permute(0, 2, 1)
    t = time_grid(steps, sway_sampling_coef)                               # :377-381
    solver = {"euler": odeint_euler, "midpoint": odeint_midpoint, "rk4": odeint_rk4}.get(method)
    if solver is None:
        raise ValueError(f"Unknown method: {method}")                      # :389-390
    trajectory = solver(fn, y0.float(), t)                                 # :393
    out = torch.where(prep.cond_mask, prep.cond, trajectory[-1])           # :395-397
    if vocoder is not None:
        out = vocoder(out)                                                 # :399-400
    return out, trajectory


def dit_forwards_per_sample(steps: int, method: str, cfg_strength: float) -> int:
    per = {"euler": 1, "midpoint": 2, "rk4": 4}[method]
    return (steps - 1) * per * (2 if cfg_strength >= 1e-5 else 1)


# ---------------------------------------------------------------------------------------------
# Vocos (third-party vocos-mlx, NOT in /root/reference; call sites cfm.py:19,399-400,446,471).
# Restated from the public Vocos "mel-24khz" design: ConvNeXt backbone + ISTFT head.
# Parity of this block is against this oracle only.
# ---------------------------------------------------------------------------------------------
@dataclass
class VocosConfig:
    n_mels: int = 100
    dim: int = 512
    intermediate_dim: int = 1536
    num_layers: int = 8
    n_fft: int = 1024
    hop_length: int = 256
    istft_norm: str = "window"   # "window": ÷Σw (vocos-mlx per-frame OLA); "window_sq": ÷Σw² (torch.istft)
    istft_trim: bool = False     # True: drop n_fft//2 samples each side (torch.istft center=True)


def vocos_backbone(mel: Tensor, W: Weights, vc: VocosConfig, prec: Precision = FP32) -> Tensor:
    """(b, n, 100) -> (b, n, 512): Conv1d(100->512,k7,p3) LN 8x[dwconv7 LN Linear GELU Linear γ· +res] LN."""
    x = conv1d_nlc(mel, W["vocos.backbone.embed.weight"], W["vocos.backbone.embed.bias"], padding=3, groups=1, prec=prec)
    x = F.layer_norm(x, (vc.dim,), W["vocos.backbone.norm.weight"], W["vocos.backbone.norm.bias"], eps=1e-6)
    for i in range(vc.num_layers):
        p = f"vocos.backbone.convnext.{i}."
        r = x
        h = conv1d_nlc(x, W[p + "dwconv.weight"], W[p + "dwconv.bias"], padding=3, groups=vc.dim)
        h = F.layer_norm(h, (vc.dim,), W[p + "norm.weight"], W[p + "norm.bias"], eps=1e-6)
        h = F.gelu(linear(h, W[p + "pwconv1.weight"], W[p + "pwconv1.bias"], prec))
        h = linear(h, W[p + "pwconv2.weight"], W[p + "pwconv2.bias"], prec)
        x = r + W[p + "gamma"] * h
    return F.layer_norm(x, (vc.dim,), W["vocos.backbone.final_layer_norm.weight"],
                        W["vocos.backbone.final_layer_norm.bias"], eps=1e-6)


def istft(spec: Tensor, vc: VocosConfig) -> Tensor:
    """Per-frame irfft, windowed overlap-add, envelope normalisation.  spec: (frames, n_fft//2+1) complex."""
    n_frames = spec.shape[0]
    win = hanning(vc.n_fft)
    frames = torch.fft.irfft(spec, n=vc.n_fft, dim=-1) * win
    length = (n_frames - 1) * vc.hop_length + vc.n_fft
    out = torch.zeros(length)
    env = torch.zeros(length)
    wenv = win if vc.istft_norm == "window" else win * win
    for i in range(n_frames):
        s = i * vc.hop_length
        out[s:s + vc.n_fft] += frames[i]
        env[s:s + vc.n_fft] += wenv
    out = torch.where(env > 1e-11, out / env.clamp_min(1e-11), out)
    if vc.istft_trim:
        out = out[vc.n_fft // 2: length - vc.n_fft // 2]
    return out


def vocos_head(x: Tensor, W: Weights, vc: VocosConfig, prec: Precision = FP32) -> Tensor:
    """(n, 512) -> waveform: Linear(512->n_fft+2), split (log-mag, phase), exp/clip 1e2, cos/sin, ISTFT."""
    h = linear(x, W["vocos.head.out.weight"], W["vocos.head.out.bias"], prec)
    nb = vc.n_fft // 2 + 1
    mag = torch.clamp(torch.exp(h[..., :nb]), max=1e2)
    ph = h[..., nb:]
    spec = torch.complex(mag * torch.cos(ph), mag * torch.sin(ph))
    return istft(spec, vc)


def vocos_decode(mel: Tensor, W: Weights, vc: VocosConfig = VocosConfig(), prec: Precision = FP32) -> Tensor:
    """vocoder(out) as called at cfm.py:399-400: (1, n, 100) -> 1-D waveform (batch-1, squeeze)."""
    assert mel.shape[0] == 1
    x = vocos_backbone(mel, W, vc, prec)
    return vocos_head(x[0], W, vc, prec)


# ---------------------------------------------------------------------------------------------
# FLOP accounting — used by bench.py for the roofline
# ---------------------------------------------------------------------------------------------
def dit_forward_flops(n: int, cfg: DiTConfig) -> float:
    D, L = cfg.dim, cfg.depth
    return (L * (n * (16 * D * D + 4 * n * D) + 12 * D * D)
            + n * (2 * 712 * D + 2 * (2 * 31 * (D // 16) * D) + 2 * D * 100)
            + (2 * 256 * D + 2 * D * D) + 4 * D * D)
