"""Model configs, synthetic (seeded) initialisation and weight packing for the CUDA path.

Parameter dictionaries use the reference's MLX parameter-tree names and layouts (Linear (out, in), Conv1d (out, k, in/groups)), i.e. exactly what `F5TTS.from_pretrained`
(cfm.py:475-517) feeds `load_weights` after its key conversion.  `pack_dit` turns such a dict into
the packed device layout libf5b200 consumes (include/f5_b200.h: f5_dit_weights), inside ONE
contiguous device buffer so that the multi-GPU path is a single broadcast of that buffer.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import Dict, Optional

import numpy as np
import torch


Weights = Dict[str, torch.Tensor]


@dataclass(frozen=True)
class DiTConfig:
    """Constructor arguments of the reference DiT (dit.py:332-346); defaults = F5-TTS base
    (cfm.py:459-469)."""
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
    # rotary embedding on the first pe_attn_head heads of q and k only (upstream's name; F5TTS_Base v0 = 1), None = all
    pe_attn_head: Optional[int] = None

    @property
    def ff_inner(self) -> int:
        return int(self.dim * self.ff_mult)


BASE_CONFIG = DiTConfig()
GATE_CONFIG = DiTConfig(dim=512, depth=4, heads=8)   # BASELINE.json configs[0] numerics gate


@dataclass(frozen=True)
class VocosConfig:
    n_mels: int = 100
    dim: int = 512
    intermediate_dim: int = 1536
    num_layers: int = 8
    n_fft: int = 1024
    hop_length: int = 256
    istft_norm: str = "window"
    istft_trim: bool = False


# ---------------------------------------------------------------------------------------------
# synthetic initialisation (no checkpoints are reachable: no network)
# ---------------------------------------------------------------------------------------------
def _uniform(rng: np.random.Generator, shape, fan_in: int, gain: float = 1.0) -> torch.Tensor:
    b = gain / math.sqrt(fan_in)
    return torch.from_numpy(rng.uniform(-b, b, size=shape).astype(np.float32))


def _normal(rng: np.random.Generator, shape, std: float, mean: float = 0.0) -> torch.Tensor:
    return torch.from_numpy((mean + std * rng.standard_normal(size=shape)).astype(np.float32))


def random_dit_weights(cfg: DiTConfig, seed: int = 1234, adaln_gain: float = 4.0) -> Weights:
    """Seeded random-init weights with the reference's parameter names.

    Linear/Conv: U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for weight and bias (MLX default scale).
    Deviations chosen so that every code path is numerically exercised (documented in DESIGN.md):
    GRN gamma/beta ~ N(0, 0.5^2) (reference init is zeros = identity), LayerNorm affine
    ~ (1 + 0.1 N, 0.1 N), AdaLN linears scaled by `adaln_gain` so the gates are O(0.1-0.5) instead
    of O(0.03) (otherwise 22 blocks contribute almost nothing to the output and a wrong block
    would hide below the tolerance)."""
    rng = np.random.default_rng(seed)
    D, F, Ct = cfg.dim, cfg.ff_inner, cfg.text_dim
    W: Weights = {}

    def lin(name, out_f, in_f, gain=1.0):
        W[name + ".weight"] = _uniform(rng, (out_f, in_f), in_f, gain)
        W[name + ".bias"] = _uniform(rng, (out_f,), in_f, gain)

    lin("transformer.time_embed.time_mlp.layers.0", D, 256)
    lin("transformer.time_embed.time_mlp.layers.2", D, D)
    W["transformer.text_embed.text_embed.weight"] = _normal(rng, (cfg.text_num_embeds + 1, Ct), math.sqrt(1.0 / Ct))
    for i in range(cfg.conv_layers):
        p = f"transformer.text_embed.text_blocks.layers.{i}."
        W[p + "dwconv.weight"] = _uniform(rng, (Ct, 7, 1), 7)
        W[p + "dwconv.bias"] = _uniform(rng, (Ct,), 7)
        W[p + "norm.weight"] = _normal(rng, (Ct,), 0.1, 1.0)
        W[p + "norm.bias"] = _normal(rng, (Ct,), 0.1)
        lin(p + "pwconv1", 2 * Ct, Ct)
        W[p + "grn.gamma"] = _normal(rng, (1, 1, 2 * Ct), 0.5)
        W[p + "grn.beta"] = _normal(rng, (1, 1, 2 * Ct), 0.5)
        lin(p + "pwconv2", Ct, 2 * Ct)
    lin("transformer.input_embed.proj", D, 2 * cfg.mel_dim + Ct)
    for j in (0, 2):
        p = f"transformer.input_embed.conv_pos_embed.conv1d.layers.{j}."
        W[p + "weight"] = _uniform(rng, (D, 31, D // 16), 31 * (D // 16))
        W[p + "bias"] = _uniform(rng, (D,), 31 * (D // 16))
    W["transformer.rotary_embed.inv_freq"] = 1.0 / (10000.0 ** (torch.arange(0, 64, 2, dtype=torch.float32) / 64))
    for i in range(cfg.depth):
        p = f"transformer.transformer_blocks.{i}."
        lin(p + "attn_norm.linear", 6 * D, D, adaln_gain)
        lin(p + "attn.to_q", D, D)
        lin(p + "attn.to_k", D, D)
        lin(p + "attn.to_v", D, D)
        lin(p + "attn.to_out.layers.0", D, D)
        lin(p + "ff.ff.layers.0.layers.0", F, D)
        lin(p + "ff.ff.layers.2", D, F)
    lin("transformer.norm_out.linear", 2 * D, D, adaln_gain)
    lin("transformer.proj_out", cfg.mel_dim, D)
    return W


def random_duration_weights(dim: int = 512, depth: int = 8, ff_mult: int = 2, text_dim: int = 512, conv_layers: int = 2,
                            text_num_embeds: int = 2545, mel_dim: int = 100, seed: int = 777) -> Weights:
    """Seeded random-init DurationPredictor weights with the MLX parameter names of duration_v2
    (cfm.py:428-442): `transformer.…`, `to_pred.layers.0.weight`."""
    rng = np.random.default_rng(seed)
    D, F, Ct = dim, dim * ff_mult, text_dim
    W: Weights = {}

    def lin(name, out_f, in_f, bias=True):
        W[name + ".weight"] = _uniform(rng, (out_f, in_f), in_f)
        if bias:
            W[name + ".bias"] = _uniform(rng, (out_f,), in_f)

    T = "transformer."
    W[T + "text_embed.text_embed.weight"] = _normal(rng, (text_num_embeds + 1, Ct), math.sqrt(1.0 / Ct))
    for i in range(conv_layers):
        p = T + f"text_embed.text_blocks.layers.{i}."
        W[p + "dwconv.weight"] = _uniform(rng, (Ct, 7, 1), 7); W[p + "dwconv.bias"] = _uniform(rng, (Ct,), 7)
        W[p + "norm.weight"] = _normal(rng, (Ct,), 0.1, 1.0); W[p + "norm.bias"] = _normal(rng, (Ct,), 0.1)
        lin(p + "pwconv1", 2 * Ct, Ct)
        W[p + "grn.gamma"] = _normal(rng, (1, 1, 2 * Ct), 0.5); W[p + "grn.beta"] = _normal(rng, (1, 1, 2 * Ct), 0.5)
        lin(p + "pwconv2", Ct, 2 * Ct)
    lin(T + "input_embed.proj", D, mel_dim + Ct)
    for j in (0, 2):
        p = T + f"input_embed.conv_pos_embed.conv1d.layers.{j}."
        W[p + "weight"] = _uniform(rng, (D, 31, D // 16), 31 * (D // 16)); W[p + "bias"] = _uniform(rng, (D,), 31 * (D // 16))
    for i in range(depth):
        p = T + f"transformer_blocks.{i}."
        for n in "qkv":
            lin(p + f"attn.to_{n}", D, D)
        lin(p + "attn.to_out.layers.0", D, D)
        lin(p + "ff.ff.layers.0.layers.0", F, D)
        lin(p + "ff.ff.layers.2", D, F)
    W[T + "norm_out.weight"] = _normal(rng, (D,), 0.1, 1.0)
    W["to_pred.layers.0.weight"] = _uniform(rng, (1, D), D, gain=8.0)
    return W


def random_vocos_weights(vc: VocosConfig = VocosConfig(), seed: int = 4321) -> Weights:
    rng = np.random.default_rng(seed)
    W: Weights = {}
    W["vocos.backbone.embed.weight"] = _uniform(rng, (vc.dim, 7, vc.n_mels), 7 * vc.n_mels)
    W["vocos.backbone.embed.bias"] = _uniform(rng, (vc.dim,), 7 * vc.n_mels)
    W["vocos.backbone.norm.weight"] = _normal(rng, (vc.dim,), 0.1, 1.0)
    W["vocos.backbone.norm.bias"] = _normal(rng, (vc.dim,), 0.1)
    for i in range(vc.num_layers):
        p = f"vocos.backbone.convnext.{i}."
        W[p + "dwconv.weight"] = _uniform(rng, (vc.dim, 7, 1), 7)
        W[p + "dwconv.bias"] = _uniform(rng, (vc.dim,), 7)
        W[p + "norm.weight"] = _normal(rng, (vc.dim,), 0.1, 1.0)
        W[p + "norm.bias"] = _normal(rng, (vc.dim,), 0.1)
        W[p + "pwconv1.weight"] = _uniform(rng, (vc.intermediate_dim, vc.dim), vc.dim)
        W[p + "pwconv1.bias"] = _uniform(rng, (vc.intermediate_dim,), vc.dim)
        W[p + "pwconv2.weight"] = _uniform(rng, (vc.dim, vc.intermediate_dim), vc.intermediate_dim)
        W[p + "pwconv2.bias"] = _uniform(rng, (vc.dim,), vc.intermediate_dim)
        W[p + "gamma"] = _normal(rng, (vc.dim,), 0.1, 0.3)
    W["vocos.backbone.final_layer_norm.weight"] = _normal(rng, (vc.dim,), 0.1, 1.0)
    W["vocos.backbone.final_layer_norm.bias"] = _normal(rng, (vc.dim,), 0.1)
    W["vocos.head.out.weight"] = _uniform(rng, (vc.n_fft + 2, vc.dim), vc.dim)
    W["vocos.head.out.bias"] = _uniform(rng, (vc.n_fft + 2,), vc.dim)
    return W


def convert_upstream_keys(weights: Weights) -> Weights:
    """The key rename + conv-weight transpose of F5TTS.from_pretrained (cfm.py:477-508): upstream
    (PyTorch F5-TTS) checkpoint names/layouts -> the MLX names/layouts used everywhere here."""
    out: Weights = {}
    for k, v in weights.items():
        k = k.replace("ema_model.", "")
        if len(k) < 1 or "mel_spec." in k or k in ("initted", "step"):
            continue
        elif ".to_out" in k:
            k = k.replace(".to_out", ".to_out.layers")
        elif ".text_blocks" in k:
            k = k.replace(".text_blocks", ".text_blocks.layers")
        elif ".ff.ff.0.0" in k:
            k = k.replace(".ff.ff.0.0", ".ff.ff.layers.0.layers.0")
        elif ".ff.ff.2" in k:
            k = k.replace(".ff.ff.2", ".ff.ff.layers.2")
        elif ".time_mlp" in k:
            k = k.replace(".time_mlp", ".time_mlp.layers")
        elif ".conv1d" in k:
            k = k.replace(".conv1d", ".conv1d.layers")
        if ".dwconv.weight" in k or ".conv1d.layers.0.weight" in k or ".conv1d.layers.2.weight" in k:
            v = v.transpose(1, 2)
        out[k] = v
    return out


# ---------------------------------------------------------------------------------------------
# MLX affine quantisation (cfm.py:451-452, 510-515): `model_v1_{4,8}b.safetensors` store, for every nn.Linear whose
# input dim is a multiple of 64, `weight` (uint32, `32 // bits` codes per word, code j of a word in bits
# [j*bits, (j+1)*bits)), `scales` and `biases` (one per group of 64 consecutive input channels):
#     w[o, i] = scales[o, i // 64] * code[o, i] + biases[o, i // 64]        (mx.dequantize)
# The H100 path computes in bf16 anyway, so such files are dequantised once at load time (pack time).
# ---------------------------------------------------------------------------------------------
MLX_GROUP_SIZE = 64


def dequantize_mlx_affine(wq: torch.Tensor, scales: torch.Tensor, biases: torch.Tensor, bits: int,
                          group_size: int = MLX_GROUP_SIZE) -> torch.Tensor:
    if bits not in (2, 4, 8):
        raise ValueError(f"unsupported MLX quantisation width: {bits} bits")
    per_word = 32 // bits
    words = wq.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF          # uint32 payload, whatever the dtype tag
    out_f, n_words = words.shape
    shifts = torch.arange(per_word, dtype=torch.int64) * bits
    codes = ((words[:, :, None] >> shifts) & ((1 << bits) - 1)).reshape(out_f, n_words * per_word).float()
    in_f = codes.shape[1]
    if scales.shape != (out_f, in_f // group_size) or biases.shape != scales.shape:
        raise ValueError(f"quantised Linear {tuple(wq.shape)}: scales/biases {tuple(scales.shape)} do not match "
                         f"{out_f} x {in_f // group_size} groups of {group_size}")
    g = codes.view(out_f, in_f // group_size, group_size)
    return (g * scales.float()[:, :, None] + biases.float()[:, :, None]).reshape(out_f, in_f)


def quantize_mlx_affine(w: torch.Tensor, bits: int, group_size: int = MLX_GROUP_SIZE):
    """Min/max affine quantiser producing the MLX file layout (used by the tests and by tools that want a `--q`
    style checkpoint); returns (packed uint32-as-int32 weight, scales, biases)."""
    out_f, in_f = w.shape
    assert in_f % group_size == 0
    g = w.float().view(out_f, in_f // group_size, group_size)
    lo, hi = g.min(dim=-1).values, g.max(dim=-1).values
    n_bins = (1 << bits) - 1
    scales = ((hi - lo) / n_bins).clamp_min(1e-7)
    codes = torch.round((g - lo[:, :, None]) / scales[:, :, None]).clamp(0, n_bins).to(torch.int64).reshape(out_f, in_f)
    per_word = 32 // bits
    shifts = torch.arange(per_word, dtype=torch.int64) * bits
    words = (codes.view(out_f, in_f // per_word, per_word) << shifts).sum(dim=-1)
    words = torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)
    return words, scales, lo


def dequantize_mlx_checkpoint(weights: Weights, bits: int, group_size: int = MLX_GROUP_SIZE) -> Weights:
    """Replaces every (`X.weight` packed, `X.scales`, `X.biases`) triple by the dense fp32 `X.weight`."""
    out: Weights = {}
    for k, v in weights.items():
        if k.endswith(".scales") or k.endswith(".biases"):
            continue
        stem = k[: -len(".weight")] if k.endswith(".weight") else None
        if stem is not None and stem + ".scales" in weights:
            v = dequantize_mlx_affine(v, weights[stem + ".scales"], weights[stem + ".biases"], bits, group_size)
        out[k] = v
    return out


# ---------------------------------------------------------------------------------------------
# packing
# ---------------------------------------------------------------------------------------------
class ConvNextWeightsC(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in
                ("dw_w", "dw_b", "ln_w", "ln_b", "pw1_w", "pw1_b", "grn_gamma", "grn_beta", "pw2_w", "pw2_b")]


class DitBlockWeightsC(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in
                ("qkv_w", "qkv_b", "out_w", "out_b", "ff1_w", "ff1_b", "ff2_w", "ff2_b", "qkv_w8", "ff1_w8", "out_w8",
                 "ff2_w8")] + \
               [("qkv_s8", C.c_float), ("ff1_s8", C.c_float), ("out_s8", C.c_float), ("ff2_s8", C.c_float)] + \
               [(n, C.c_void_p) for n in ("qkv_ws", "ff1_ws", "out_ws", "ff2_ws")]


E4M3_MAX = 448.0


def quantize_e4m3(w: torch.Tensor):
    """Per-tensor e4m3 quantisation of a weight matrix: w ~= scale * q, q in float8_e4m3fn (round to nearest even,
    |q| <= 448).  Returns (bytes as uint8 tensor, scale)."""
    w = w.detach().float()
    scale = float(w.abs().max().item()) / E4M3_MAX
    if scale == 0.0:
        scale = 1.0
    q = (w / scale).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q.view(torch.uint8), scale


FP8_SCALINGS = ("tensor", "block")


def e4m3_block_scale(amax: torch.Tensor) -> torch.Tensor:
    """The scale rule of the block-scaled FP8 mode, element-wise on fp32 amax >= 0: the smallest power of two s >= 2^-126
    with amax <= 448 s, read off amax's exponent and mantissa bits exactly as the kernels do (ptx.cuh e4m3_block_scale);
    1 for amax == 0; a non-finite amax is its own scale.  (The floor 2^-126 keeps 1 / s finite.)"""
    a = amax.float().contiguous()
    b = a.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    e, m = (b >> 23) & 0xFF, b & 0x7FFFFF
    k = (e - 135 + (m > 0x600000).to(torch.int64)).clamp_min(-126)
    s = ((k + 127) << 23).to(torch.int32).view(torch.float32)
    s = torch.where(b == 0, torch.ones_like(s), s)
    return torch.where(e == 0xFF, a, s)


def quantize_e4m3_blocks(x: torch.Tensor, block: int = 64):
    """Block-scaled e4m3 of an fp32 matrix [rows, cols]: one power-of-two scale per (row, `block` columns) (a whole row
    with block = cols: the per-output-channel weight scale).  Returns (e4m3 codes as uint8 [rows, cols], scales fp32
    [rows, cols / block]) with x ~= codes * scale, quantised as x * (1 / s) rounded to nearest even."""
    x = x.detach().float()
    r, c = x.shape
    g = x.reshape(r, c // block, block)
    s = e4m3_block_scale(g.abs().amax(dim=-1))
    q = (g * (1.0 / s)[..., None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q.view(torch.uint8).reshape(r, c), s


def fp8_vt_key_order() -> torch.Tensor:
    """Key order of the FP8 attention's V^T (f5_qkv_quant_e4m3): position p of every 32-key group holds key
    order[p].  It makes the softmax's S accumulator fragment (keys {2l, 2l+1, 2l+8, 2l+9} and 16 + those, l = lane % 4)
    the e4m3 register A fragment of the P·V wgmma (k = 4l .. 4l+3 and 16 + those): position 16 h + 4 l + i holds key
    16 h + (2l, 2l+1, 2l+8, 2l+9)[i] (csrc/attention_fp8_sm90.cuh fp8_vt_key)."""
    p = torch.arange(32)
    return (p & 16) + 2 * ((p >> 2) & 3) + 8 * ((p >> 1) & 1) + (p & 1)


class DitWeightsC(C.Structure):
    _fields_ = [
        ("dim", C.c_int32), ("depth", C.c_int32), ("heads", C.c_int32), ("ff_inner", C.c_int32),
        ("mel_dim", C.c_int32), ("text_dim", C.c_int32), ("text_inner", C.c_int32), ("conv_layers", C.c_int32),
        ("text_rows", C.c_int32), ("text_max_pos", C.c_int32), ("ct_ld", C.c_int32), ("reserved", C.c_int32),
        ("time_w0", C.c_void_p), ("time_b0", C.c_void_p), ("time_w2", C.c_void_p), ("time_b2", C.c_void_p),
        ("text_emb", C.c_void_p), ("text_pos", C.c_void_p),
        ("text_blocks", C.POINTER(ConvNextWeightsC)),
        ("in_x_w", C.c_void_p), ("in_ct_w", C.c_void_p), ("in_b", C.c_void_p),
        ("conv_w", C.c_void_p * 2), ("conv_b", C.c_void_p * 2),
        ("mod_w", C.c_void_p), ("mod_b", C.c_void_p),
        ("blocks", C.POINTER(DitBlockWeightsC)),
        ("proj_w", C.c_void_p), ("proj_b", C.c_void_p),
        ("text_unmasked", C.c_int32), ("rope_heads", C.c_int32),
    ]


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def text_pos_table(dim: int, end: int = 4096, theta: float = 10000.0) -> torch.Tensor:
    """rope.py:63-73 precompute_freqs_cis — a constant of the model, built once at pack time."""
    freqs = 1.0 / (theta ** (torch.arange(0, dim, 2)[: dim // 2].float() / dim))
    t = torch.arange(end, dtype=torch.float32)
    freqs = torch.outer(t, freqs).float()
    return torch.cat([freqs.cos(), freqs.sin()], dim=-1)


def pack_grouped_conv(w_mlx: torch.Tensor, groups: int = 16) -> torch.Tensor:
    """MLX Conv1d weight (O, K, I/g) -> [O, K*64] tap-major, block-diagonal by 64 input channels:
    output channel o only reads the 64-channel block it lives in (block = o // 64); inside that
    block, channels of other groups get zero weight (only happens when I/g < 64)."""
    O, K, cg = w_mlx.shape
    out = torch.zeros(O, K, 64, dtype=torch.float32)
    o = torch.arange(O)
    g = o // cg                    # conv group of each output channel (O/groups == cg here)
    blk = o // 64
    base = g * cg - blk * 64       # offset of the group's first input channel inside the block
    for i in range(cg):
        out[o, :, base + i] = w_mlx[:, :, i].float()
    return out.reshape(O, K * 64)


@dataclass
class _Spec:
    name: str
    shape: tuple
    dtype: torch.dtype
    offset: int = 0


class PackedWeights:
    """A backbone's packed weights in one device buffer, so that the multi-GPU path is one broadcast.  Each tensor sits
    at an ALIGN-byte aligned offset in the order the subclass's `_layout()` yields (name, shape, dtype) triples; the
    layout depends on the config only, so every rank derives the same one.  Subclasses add `load` and `c_struct`."""

    ALIGN = 256

    def __init__(self, cfg, device: torch.device | str = "cuda"):
        self.cfg = cfg
        self.device = torch.device(device)
        self.ct_ld = _round_up(cfg.mel_dim + cfg.text_dim, 64)
        self.specs: Dict[str, _Spec] = {}
        off = 0
        for name, shape, dtype in self._layout():
            nbytes = int(np.prod(shape)) * self._esize(dtype)
            self.specs[name] = _Spec(name, tuple(shape), dtype, off)
            off = _round_up(off + nbytes, self.ALIGN)
        self.nbytes = off
        self.buffer = torch.zeros(self.nbytes, dtype=torch.uint8, device=self.device)
        self._c = None
        self._keep: list = []

    @staticmethod
    def _esize(dtype) -> int:
        return {torch.bfloat16: 2, torch.uint8: 1}.get(dtype, 4)

    def view(self, name: str) -> torch.Tensor:
        s = self.specs[name]
        n = int(np.prod(s.shape))
        nbytes = n * self._esize(s.dtype)
        return self.buffer[s.offset:s.offset + nbytes].view(s.dtype).view(s.shape)

    def _put(self, name: str, t: torch.Tensor) -> None:
        v = self.view(name)
        assert tuple(t.shape) == tuple(v.shape), (name, t.shape, v.shape)
        v.copy_(t.to(v.dtype))

    def broadcast(self, src: int = 0):
        """The ONE collective of the multi-GPU path: rank `src` holds the packed weights, every
        other rank receives them (NCCL over NVLink when the process group is nccl)."""
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            dist.broadcast(self.buffer, src=src)
        return self


class PackedDiT(PackedWeights):
    """Packed DiT weights living in one device buffer + the ctypes view libf5b200 takes."""

    def __init__(self, cfg: DiTConfig, device: torch.device | str = "cuda", fp8: bool = False,
                 fp8_scaling: str = "tensor"):
        self.fp8 = bool(fp8)           # also keep e4m3 copies of the QKV / FF1 weights (appended after the bf16 layout)
        if fp8_scaling not in FP8_SCALINGS:
            raise ValueError(f"fp8_scaling must be one of {FP8_SCALINGS}, not {fp8_scaling!r}")
        # "tensor": one scale per weight tensor; "block": one power-of-two scale per output channel (the block-scaled mode)
        self.fp8_scaling = fp8_scaling
        self.fp8_block = self.fp8 and fp8_scaling == "block"
        super().__init__(cfg, device)

    def _layout(self):
        c = self.cfg
        D, F, Ct, Ci = c.dim, c.ff_inner, c.text_dim, 2 * c.text_dim
        bf, f32 = torch.bfloat16, torch.float32
        yield "time_w0", (D, 256), f32
        yield "time_b0", (D,), f32
        yield "time_w2", (D, D), f32
        yield "time_b2", (D,), f32
        yield "text_emb", (c.text_num_embeds + 1, Ct), f32
        yield "text_pos", (4096, Ct), f32
        for i in range(c.conv_layers):
            yield f"tb{i}.dw_w", (7, Ct), f32
            yield f"tb{i}.dw_b", (Ct,), f32
            yield f"tb{i}.ln_w", (Ct,), f32
            yield f"tb{i}.ln_b", (Ct,), f32
            yield f"tb{i}.pw1_w", (Ci, Ct), bf
            yield f"tb{i}.pw1_b", (Ci,), f32
            yield f"tb{i}.grn_gamma", (Ci,), f32
            yield f"tb{i}.grn_beta", (Ci,), f32
            yield f"tb{i}.pw2_w", (Ct, Ci), bf
            yield f"tb{i}.pw2_b", (Ct,), f32
        yield "in_x_w", (D, 128), bf
        yield "in_ct_w", (D, self.ct_ld), bf
        yield "in_b", (D,), f32
        for j in range(2):
            yield f"conv_w{j}", (D, 31 * 64), bf
            yield f"conv_b{j}", (D,), f32
        yield "mod_w", (c.depth * 6 * D + 2 * D, D), bf
        yield "mod_b", (c.depth * 6 * D + 2 * D,), f32
        for i in range(c.depth):
            yield f"blk{i}.qkv_w", (3 * D, D), bf
            yield f"blk{i}.qkv_b", (3 * D,), f32
            yield f"blk{i}.out_w", (D, D), bf
            yield f"blk{i}.out_b", (D,), f32
            yield f"blk{i}.ff1_w", (F, D), bf
            yield f"blk{i}.ff1_b", (F,), f32
            yield f"blk{i}.ff2_w", (D, F), bf
            yield f"blk{i}.ff2_b", (D,), f32
        yield "proj_w", (c.mel_dim, D), bf
        yield "proj_b", (c.mel_dim,), f32
        if self.fp8_block:   # block-scaled FP8: per-channel e4m3 weights in the order a block reads them, + fp32 scales
            for i in range(c.depth):
                for n, (o, k) in (("qkv", (3 * D, D)), ("out", (D, D)), ("ff1", (F, D)), ("ff2", (D, F))):
                    yield f"blk{i}.{n}_w8c", (o, k), torch.uint8
                    yield f"blk{i}.{n}_s8c", (o,), f32
        elif self.fp8:       # FP8 mode: appended, so the bf16 prefix is the layout the C packer (f5_pack_weights) knows
            for i in range(c.depth):
                yield f"blk{i}.qkv_w8", (3 * D, D), torch.uint8
                yield f"blk{i}.ff1_w8", (F, D), torch.uint8
                yield f"blk{i}.out_w8", (D, D), torch.uint8
                yield f"blk{i}.ff2_w8", (D, F), torch.uint8
            yield "fp8_scales", (c.depth, 4), f32       # (qkv, ff1, out, ff2) per block: travels with the ONE broadcast

    def load(self, W: Weights) -> "PackedDiT":
        """Fill the buffer from an MLX-named parameter dict (fp32)."""
        c = self.cfg
        D = c.dim
        g = lambda k: W[k].detach().float()
        T = "transformer."
        self._put("time_w0", g(T + "time_embed.time_mlp.layers.0.weight"))
        self._put("time_b0", g(T + "time_embed.time_mlp.layers.0.bias"))
        self._put("time_w2", g(T + "time_embed.time_mlp.layers.2.weight"))
        self._put("time_b2", g(T + "time_embed.time_mlp.layers.2.bias"))
        self._put("text_emb", g(T + "text_embed.text_embed.weight"))
        self._put("text_pos", text_pos_table(c.text_dim))
        for i in range(c.conv_layers):
            p = T + f"text_embed.text_blocks.layers.{i}."
            self._put(f"tb{i}.dw_w", g(p + "dwconv.weight")[:, :, 0].t().contiguous())
            self._put(f"tb{i}.dw_b", g(p + "dwconv.bias"))
            self._put(f"tb{i}.ln_w", g(p + "norm.weight"))
            self._put(f"tb{i}.ln_b", g(p + "norm.bias"))
            self._put(f"tb{i}.pw1_w", g(p + "pwconv1.weight"))
            self._put(f"tb{i}.pw1_b", g(p + "pwconv1.bias"))
            self._put(f"tb{i}.grn_gamma", g(p + "grn.gamma").reshape(-1))
            self._put(f"tb{i}.grn_beta", g(p + "grn.beta").reshape(-1))
            self._put(f"tb{i}.pw2_w", g(p + "pwconv2.weight"))
            self._put(f"tb{i}.pw2_b", g(p + "pwconv2.bias"))
        pw = g(T + "input_embed.proj.weight")               # (D, mel + mel + text)
        wx = torch.zeros(D, 128); wx[:, :c.mel_dim] = pw[:, :c.mel_dim]
        wct = torch.zeros(D, self.ct_ld); wct[:, :c.mel_dim + c.text_dim] = pw[:, c.mel_dim:]
        self._put("in_x_w", wx)
        self._put("in_ct_w", wct)
        self._put("in_b", g(T + "input_embed.proj.bias"))
        for j, lj in enumerate((0, 2)):
            p = T + f"input_embed.conv_pos_embed.conv1d.layers.{lj}."
            self._put(f"conv_w{j}", pack_grouped_conv(g(p + "weight")))
            self._put(f"conv_b{j}", g(p + "bias"))
        mw = [g(T + f"transformer_blocks.{i}.attn_norm.linear.weight") for i in range(c.depth)]
        mb = [g(T + f"transformer_blocks.{i}.attn_norm.linear.bias") for i in range(c.depth)]
        mw.append(g(T + "norm_out.linear.weight")); mb.append(g(T + "norm_out.linear.bias"))
        self._put("mod_w", torch.cat(mw, 0)); self._put("mod_b", torch.cat(mb, 0))
        for i in range(c.depth):
            p = T + f"transformer_blocks.{i}."
            self._put(f"blk{i}.qkv_w", torch.cat([g(p + f"attn.to_{n}.weight") for n in "qkv"], 0))
            self._put(f"blk{i}.qkv_b", torch.cat([g(p + f"attn.to_{n}.bias") for n in "qkv"], 0))
            self._put(f"blk{i}.out_w", g(p + "attn.to_out.layers.0.weight"))
            self._put(f"blk{i}.out_b", g(p + "attn.to_out.layers.0.bias"))
            self._put(f"blk{i}.ff1_w", g(p + "ff.ff.layers.0.layers.0.weight"))
            self._put(f"blk{i}.ff1_b", g(p + "ff.ff.layers.0.layers.0.bias"))
            self._put(f"blk{i}.ff2_w", g(p + "ff.ff.layers.2.weight"))
            self._put(f"blk{i}.ff2_b", g(p + "ff.ff.layers.2.bias"))
            if self.fp8_block:
                for n, wt in (("qkv", torch.cat([g(p + f"attn.to_{n}.weight") for n in "qkv"], 0)),
                              ("out", g(p + "attn.to_out.layers.0.weight")),
                              ("ff1", g(p + "ff.ff.layers.0.layers.0.weight")),
                              ("ff2", g(p + "ff.ff.layers.2.weight"))):
                    q, sc = quantize_e4m3_blocks(wt, wt.shape[1])
                    self.view(f"blk{i}.{n}_w8c").copy_(q)
                    self._put(f"blk{i}.{n}_s8c", sc.reshape(-1))
            elif self.fp8:
                for j, (dst, wt) in enumerate(((f"blk{i}.qkv_w8", torch.cat([g(p + f"attn.to_{n}.weight") for n in "qkv"], 0)),
                                               (f"blk{i}.ff1_w8", g(p + "ff.ff.layers.0.layers.0.weight")),
                                               (f"blk{i}.out_w8", g(p + "attn.to_out.layers.0.weight")),
                                               (f"blk{i}.ff2_w8", g(p + "ff.ff.layers.2.weight")))):
                    q, sc = quantize_e4m3(wt)
                    self.view(dst).copy_(q)
                    self.view("fp8_scales")[i, j] = sc
        self._put("proj_w", g(T + "proj_out.weight"))
        self._put("proj_b", g(T + "proj_out.bias"))
        return self

    def c_struct(self) -> DitWeightsC:
        if self._c is not None:
            return self._c
        c = self.cfg
        ptr = lambda name: self.buffer.data_ptr() + self.specs[name].offset
        w = DitWeightsC()
        w.dim, w.depth, w.heads, w.ff_inner = c.dim, c.depth, c.heads, c.ff_inner
        w.mel_dim, w.text_dim, w.text_inner, w.conv_layers = c.mel_dim, c.text_dim, 2 * c.text_dim, c.conv_layers
        w.text_rows, w.text_max_pos, w.ct_ld = c.text_num_embeds + 1, 4096, self.ct_ld
        w.text_unmasked, w.rope_heads = int(not c.text_mask_padding), c.pe_attn_head or 0
        for n in ("time_w0", "time_b0", "time_w2", "time_b2", "text_emb", "text_pos", "in_x_w", "in_ct_w", "in_b",
                  "mod_w", "mod_b", "proj_w", "proj_b"):
            setattr(w, n, ptr(n))
        tbs = (ConvNextWeightsC * max(c.conv_layers, 1))()
        for i in range(c.conv_layers):
            for n, _ in ConvNextWeightsC._fields_:
                setattr(tbs[i], n, ptr(f"tb{i}.{n}"))
        blks = (DitBlockWeightsC * c.depth)()
        for i in range(c.depth):
            for n, _ in DitBlockWeightsC._fields_[:8]:
                setattr(blks[i], n, ptr(f"blk{i}.{n}"))
            if self.fp8_block:
                for n in ("qkv", "ff1", "out", "ff2"):
                    setattr(blks[i], f"{n}_w8", ptr(f"blk{i}.{n}_w8c"))
                    setattr(blks[i], f"{n}_ws", ptr(f"blk{i}.{n}_s8c"))
                    setattr(blks[i], f"{n}_s8", 1.0)
            elif self.fp8:
                sc = self.view("fp8_scales").cpu()
                blks[i].qkv_w8, blks[i].ff1_w8 = ptr(f"blk{i}.qkv_w8"), ptr(f"blk{i}.ff1_w8")
                blks[i].out_w8, blks[i].ff2_w8 = ptr(f"blk{i}.out_w8"), ptr(f"blk{i}.ff2_w8")
                blks[i].qkv_s8, blks[i].ff1_s8 = float(sc[i, 0]), float(sc[i, 1])
                blks[i].out_s8, blks[i].ff2_s8 = float(sc[i, 2]), float(sc[i, 3])
        w.text_blocks = tbs
        w.blocks = blks
        for j in range(2):
            w.conv_w[j] = ptr(f"conv_w{j}")
            w.conv_b[j] = ptr(f"conv_b{j}")
        self._keep = [tbs, blks]
        self._c = w
        return w
