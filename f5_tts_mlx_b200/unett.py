"""UNetT — the flat UNet-Transformer backbone of upstream F5-TTS's E2TTS_Base (f5_tts/model/backbones/unett.py).

Same constructor arguments as upstream's UNetT; the sessions, C entry points and `__call__` that `F5TTS` uses come from
`dit.Backbone`, shared with the DiT.  All arithmetic runs in libf5b200 (f5_unett_*, sm_90a).
Only the E2TTS_Base form is built: skip_connect_type "concat", no qk_norm, conv_layers 0 (no ConvNeXt, no position
table), text_mask_padding False, an even depth.  Forward of x, cond [b, n, mel]:

    t = TimestepEmbedding(time);  x = InputEmbedding(x, cond, Embedding(text + 1))        (the DiT's input embedding)
    x = [t | x]  (n + 1 rows, RoPE positions 0..n, rotation on the first pe_attn_head heads)
    layer i:  i < depth/2: push x;  else x = skip_proj([x | pop()])
              x = attn(RMSNorm(x)) + x;  x = ff(RMSNorm(x)) + x
    out = proj_out(RMSNorm(x)[:, 1:])

RMSNorm is x_transformers': x * sqrt(D) / max(||x||, 1e-12) * g.  Each g is folded into the Linear that consumes the
norm at pack time (W diag(g), then bf16), and the row scale is applied in that GEMM's epilogue (f5_gemm_args.ln_rms).

Weights use upstream's state-dict names with the `ema_model.` prefix stripped (`checkpoint_state`): no E2 checkpoint was
ever converted to the MLX layout, so there is no other naming to follow.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from .dit import Backbone, rope_table
from .weights import DitBlockWeightsC, PackedWeights, Weights, _normal, _uniform, pack_grouped_conv


@dataclass(frozen=True)
class UNetTConfig:
    """Constructor arguments of upstream's UNetT that this backbone honours; defaults = E2TTS_Base."""
    dim: int = 1024
    depth: int = 24
    heads: int = 16
    dim_head: int = 64
    ff_mult: int = 4
    mel_dim: int = 100
    text_num_embeds: int = 2545
    text_dim: int = 100
    pe_attn_head: Optional[int] = 1

    @property
    def ff_inner(self) -> int:
        return int(self.dim * self.ff_mult)


E2_BASE_CONFIG = UNetTConfig()
ROPE_INV_FREQ_KEY = "transformer.rotary_embed.inv_freq"


def checkpoint_keys(cfg: UNetTConfig) -> set:
    """The parameter names of an E2TTS_Base-form UNetT checkpoint, `ema_model.` stripped."""
    T = "transformer."
    keys = {T + f"time_embed.time_mlp.{j}.{p}" for j in (0, 2) for p in ("weight", "bias")}
    keys.add(T + "text_embed.text_embed.weight")
    keys |= {T + f"input_embed.proj.{p}" for p in ("weight", "bias")}
    keys |= {T + f"input_embed.conv_pos_embed.conv1d.{j}.{p}" for j in (0, 2) for p in ("weight", "bias")}
    for i in range(cfg.depth):
        p = T + f"layers.{i}."
        if i >= cfg.depth // 2:
            keys.add(p + "0.weight")
        keys |= {p + "1.g", p + "3.g"}
        keys |= {p + f"2.{n}.{q}" for n in ("to_q", "to_k", "to_v", "to_out.0") for q in ("weight", "bias")}
        keys |= {p + f"4.ff.{n}.{q}" for n in ("0.0", "2") for q in ("weight", "bias")}
    keys |= {T + "norm_out.g", T + "proj_out.weight", T + "proj_out.bias"}
    return keys


def _rope_inv_freq(dim_head: int = 64) -> torch.Tensor:
    return 1.0 / (10000.0 ** (torch.arange(0, dim_head, 2, dtype=torch.float32) / dim_head))


def checkpoint_state(sd: Weights, cfg: UNetTConfig) -> Weights:
    """An upstream state dict (`ema_model.` prefix or not) -> the weights UNetT.load_weights takes: the prefix stripped,
    `mel_spec.*`, `initted` and `step` dropped.  Any missing or unexpected key is a ValueError naming it: the key list
    is restated from upstream's module structure, so a file that differs must not load as a partial model.  The
    rotary table `transformer.rotary_embed.inv_freq` (a buffer, not a parameter) may be present; it must then hold the
    fixed base-10000 frequencies the kernels use."""
    out: Weights = {}
    for k, v in sd.items():
        if k.startswith("ema_model."):
            k = k[len("ema_model."):]
        if k.startswith("mel_spec.") or k in ("initted", "step"):
            continue
        out[k] = v
    inv = out.pop(ROPE_INV_FREQ_KEY, None)
    if inv is not None and not torch.allclose(inv.float().cpu(), _rope_inv_freq(cfg.dim_head), rtol=1e-6, atol=0):
        raise ValueError(f"{ROPE_INV_FREQ_KEY} is not the base-10000 rotary table this backbone computes")
    want = checkpoint_keys(cfg)
    missing, extra = sorted(want - out.keys()), sorted(out.keys() - want)
    if missing or extra:
        raise ValueError("not an E2TTS_Base-form UNetT checkpoint: " +
                         "; ".join(s for s in (f"missing keys {missing}" if missing else "",
                                               f"unexpected keys {extra}" if extra else "") if s))
    return out


def random_unett_weights(cfg: UNetTConfig = E2_BASE_CONFIG, seed: int = 1234) -> Weights:
    """Seeded random UNetT weights with upstream's names.  Linear: U(-1/sqrt(fan_in), 1/sqrt(fan_in)) weight and bias;
    RMSNorm gains 1 + 0.1 N(0, 1), so that a mis-folded gain shows; embedding N(0, 1/text_dim)."""
    rng = np.random.default_rng(seed)
    D, F = cfg.dim, cfg.ff_inner
    T = "transformer."
    W: Weights = {}

    def lin(name, out_f, in_f, bias=True):
        W[name + ".weight"] = _uniform(rng, (out_f, in_f), in_f)
        if bias:
            W[name + ".bias"] = _uniform(rng, (out_f,), in_f)

    lin(T + "time_embed.time_mlp.0", D, 256)
    lin(T + "time_embed.time_mlp.2", D, D)
    W[T + "text_embed.text_embed.weight"] = _normal(rng, (cfg.text_num_embeds + 1, cfg.text_dim), math.sqrt(1.0 / cfg.text_dim))
    lin(T + "input_embed.proj", D, 2 * cfg.mel_dim + cfg.text_dim)
    for j in (0, 2):   # PyTorch Conv1d layout (out, in / groups, k)
        W[T + f"input_embed.conv_pos_embed.conv1d.{j}.weight"] = _uniform(rng, (D, D // 16, 31), 31 * (D // 16))
        W[T + f"input_embed.conv_pos_embed.conv1d.{j}.bias"] = _uniform(rng, (D,), 31 * (D // 16))
    for i in range(cfg.depth):
        p = T + f"layers.{i}."
        if i >= cfg.depth // 2:
            lin(p + "0", D, 2 * D, bias=False)
        W[p + "1.g"] = _normal(rng, (D,), 0.1, 1.0)
        for n in ("to_q", "to_k", "to_v", "to_out.0"):
            lin(p + "2." + n, D, D)
        W[p + "3.g"] = _normal(rng, (D,), 0.1, 1.0)
        lin(p + "4.ff.0.0", F, D)
        lin(p + "4.ff.2", D, F)
    W[T + "norm_out.g"] = _normal(rng, (D,), 0.1, 1.0)
    lin(T + "proj_out", cfg.mel_dim, D)
    return W


class UNetTWeightsC(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("dim", "depth", "heads", "ff_inner", "mel_dim", "text_dim", "text_rows",
                                         "ct_ld", "rope_heads", "reserved")] + \
               [(n, C.c_void_p) for n in ("time_w0", "time_b0", "time_w2", "time_b2", "text_emb", "in_x_w", "in_ct_w",
                                          "in_b")] + \
               [("conv_w", C.c_void_p * 2), ("conv_b", C.c_void_p * 2), ("blocks", C.POINTER(DitBlockWeightsC)),
                ("skip_w", C.c_void_p), ("proj_w", C.c_void_p), ("proj_b", C.c_void_p)]


class UNetTBuffersC(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("batch", "frames", "cfg", "n_times", "text_len_max", "drop_flags")] + \
               [(n, C.c_void_p) for n in ("text", "seq_len1", "valid_len", "valid_len1", "cond", "tvals", "rope",
                                          "hoist", "t_emb", "text_x", "ct_bf16", "silu_t", "y_bf16", "h", "x", "a_bf16",
                                          "c_bf16", "qkv_bf16", "ff_bf16", "ln_stats", "skip", "v")]


class PackedUNetT(PackedWeights):
    """Packed UNetT weights in one device buffer + the ctypes view libf5b200 takes."""

    def _layout(self):
        c = self.cfg
        D, F = c.dim, c.ff_inner
        bf, f32 = torch.bfloat16, torch.float32
        yield "time_w0", (D, 256), f32
        yield "time_b0", (D,), f32
        yield "time_w2", (D, D), f32
        yield "time_b2", (D,), f32
        yield "text_emb", (c.text_num_embeds + 1, c.text_dim), f32
        yield "in_x_w", (D, 128), bf
        yield "in_ct_w", (D, self.ct_ld), bf
        yield "in_b", (D,), f32
        for j in range(2):
            yield f"conv_w{j}", (D, 31 * 64), bf
            yield f"conv_b{j}", (D,), f32
        for i in range(c.depth):
            yield f"blk{i}.qkv_w", (3 * D, D), bf
            yield f"blk{i}.qkv_b", (3 * D,), f32
            yield f"blk{i}.out_w", (D, D), bf
            yield f"blk{i}.out_b", (D,), f32
            yield f"blk{i}.ff1_w", (F, D), bf
            yield f"blk{i}.ff1_b", (F,), f32
            yield f"blk{i}.ff2_w", (D, F), bf
            yield f"blk{i}.ff2_b", (D,), f32
        yield "skip_w", (c.depth // 2, D, 2 * D), bf
        yield "proj_w", (c.mel_dim, D), bf
        yield "proj_b", (c.mel_dim,), f32

    def load(self, W: Weights) -> "PackedUNetT":
        """Fill the buffer from checkpoint_state() weights (fp32), folding each RMSNorm gain into its consumer."""
        c = self.cfg
        D = c.dim
        g = lambda k: W[k].detach().float().cpu()
        T = "transformer."
        self._put("time_w0", g(T + "time_embed.time_mlp.0.weight"))
        self._put("time_b0", g(T + "time_embed.time_mlp.0.bias"))
        self._put("time_w2", g(T + "time_embed.time_mlp.2.weight"))
        self._put("time_b2", g(T + "time_embed.time_mlp.2.bias"))
        self._put("text_emb", g(T + "text_embed.text_embed.weight"))
        pw = g(T + "input_embed.proj.weight")               # (D, mel + mel + text)
        wx = torch.zeros(D, 128); wx[:, :c.mel_dim] = pw[:, :c.mel_dim]
        wct = torch.zeros(D, self.ct_ld); wct[:, :c.mel_dim + c.text_dim] = pw[:, c.mel_dim:]
        self._put("in_x_w", wx)
        self._put("in_ct_w", wct)
        self._put("in_b", g(T + "input_embed.proj.bias"))
        for j, lj in enumerate((0, 2)):
            p = T + f"input_embed.conv_pos_embed.conv1d.{lj}."
            self._put(f"conv_w{j}", pack_grouped_conv(g(p + "weight").transpose(1, 2)))
            self._put(f"conv_b{j}", g(p + "bias"))
        skip = torch.zeros(c.depth // 2, D, 2 * D)
        for i in range(c.depth):
            p = T + f"layers.{i}."
            wqkv = torch.cat([g(p + f"2.to_{n}.weight") for n in "qkv"], 0)
            self._put(f"blk{i}.qkv_w", wqkv * g(p + "1.g")[None, :])
            self._put(f"blk{i}.qkv_b", torch.cat([g(p + f"2.to_{n}.bias") for n in "qkv"], 0))
            self._put(f"blk{i}.out_w", g(p + "2.to_out.0.weight"))
            self._put(f"blk{i}.out_b", g(p + "2.to_out.0.bias"))
            self._put(f"blk{i}.ff1_w", g(p + "4.ff.0.0.weight") * g(p + "3.g")[None, :])
            self._put(f"blk{i}.ff1_b", g(p + "4.ff.0.0.bias"))
            self._put(f"blk{i}.ff2_w", g(p + "4.ff.2.weight"))
            self._put(f"blk{i}.ff2_b", g(p + "4.ff.2.bias"))
            if i >= c.depth // 2:
                skip[i - c.depth // 2] = g(p + "0.weight")
        self._put("skip_w", skip)
        self._put("proj_w", g(T + "proj_out.weight") * g(T + "norm_out.g")[None, :])
        self._put("proj_b", g(T + "proj_out.bias"))
        return self

    def c_struct(self) -> UNetTWeightsC:
        if self._c is not None:
            return self._c
        c = self.cfg
        ptr = lambda name: self.buffer.data_ptr() + self.specs[name].offset
        w = UNetTWeightsC()
        w.dim, w.depth, w.heads, w.ff_inner = c.dim, c.depth, c.heads, c.ff_inner
        w.mel_dim, w.text_dim, w.text_rows, w.ct_ld = c.mel_dim, c.text_dim, c.text_num_embeds + 1, self.ct_ld
        w.rope_heads = c.pe_attn_head or 0
        for n in ("time_w0", "time_b0", "time_w2", "time_b2", "text_emb", "in_x_w", "in_ct_w", "in_b", "skip_w",
                  "proj_w", "proj_b"):
            setattr(w, n, ptr(n))
        blks = (DitBlockWeightsC * c.depth)()
        for i in range(c.depth):
            for n, _ in DitBlockWeightsC._fields_[:8]:
                setattr(blks[i], n, ptr(f"blk{i}.{n}"))
        w.blocks = blks
        for j in range(2):
            w.conv_w[j] = ptr(f"conv_w{j}")
            w.conv_b[j] = ptr(f"conv_b{j}")
        self._keep = [blks]
        self._c = w
        return w


class UNetTSession:
    """Device buffers (f5_unett_buffers) for `batch` utterances padded to `frames`, `n_times` evaluation times, with or
    without the CFG batch doubling.  The skip slots take depth/2 * rows1 * 2 * dim * 2 bytes."""

    def __init__(self, cfg: UNetTConfig, ct_ld: int, batch: int, frames: int, n_times: int, use_cfg: bool,
                 text_cols: int, device: torch.device, masked: bool):
        self.cfg, self.batch, self.frames, self.n_times, self.use_cfg = cfg, batch, frames, n_times, use_cfg
        self.device = device
        D, F = cfg.dim, cfg.ff_inner
        BU = (2 if use_cfg else 1) * batch
        R, R1 = BU * frames, BU * (frames + 1)
        self.rows, self.rows1, self.row_utts = R, R1, BU
        f32, bf16, i32 = torch.float32, torch.bfloat16, torch.int32
        z = lambda *s, dt=f32: torch.zeros(*s, dtype=dt, device=device)
        self.text = z(batch, max(text_cols, 1), dt=i32)
        self.seq_len = z(BU, dt=i32) if masked else None        # valid frames (what callers read back)
        self.seq_len1 = z(BU, dt=i32) if masked else None       # + the time row: the attention and row masks
        self.valid_len_buf = torch.full((BU,), frames, dtype=i32, device=device)
        self.valid_len1_buf = torch.full((BU,), frames + 1, dtype=i32, device=device)
        self.valid_len = self.valid_len1 = None
        self.cond = z(batch, frames, cfg.mel_dim)
        self.tvals = z(n_times)
        self.rope = rope_table(frames + 1, cfg.dim_head).to(device)
        self.hoist = z(R, D)
        self.t_emb = z(n_times, D)
        self.text_x = z(R, cfg.text_dim)
        self.ct_bf16 = z(R, ct_ld, dt=bf16)
        self.silu_t = z(n_times, D, dt=bf16)
        self.y_bf16 = z(R, 128, dt=bf16)
        self.h = z(R, D)
        self.x = z(R1, D)
        self.a_bf16 = z(R1, D, dt=bf16)
        self.c_bf16 = z(R1, D, dt=bf16)
        self.qkv_bf16 = z(R1, 3 * D, dt=bf16)
        self.ff_bf16 = z(R1, F, dt=bf16)
        self.ln_stats = z(R1, D // 64, 2)
        self.skip = z(cfg.depth // 2, R1, 2 * D, dt=bf16)
        self.v = z(R1, cfg.mel_dim)
        c = UNetTBuffersC()
        c.batch, c.frames, c.cfg, c.n_times = batch, frames, int(use_cfg), n_times
        c.text_len_max, c.drop_flags = self.text.shape[1], 0
        for name, _ in UNetTBuffersC._fields_[6:]:
            t = getattr(self, name)
            setattr(c, name, t.data_ptr() if t is not None else None)
        self.c = c

    def use_bucketing(self) -> None:
        """Bind the valid-length buffers: `frames` is a bucket size from now on (before the plan's graph is captured)."""
        self.valid_len, self.valid_len1 = self.valid_len_buf, self.valid_len1_buf
        self.c.valid_len = self.valid_len_buf.data_ptr()
        self.c.valid_len1 = self.valid_len1_buf.data_ptr()

    def set_inputs(self, text: torch.Tensor, cond: torch.Tensor, tvals: torch.Tensor,
                   seq_len: Optional[torch.Tensor], frames_valid: Optional[int] = None) -> None:
        """As DitSession.set_inputs."""
        B = self.batch
        assert text.shape == self.text.shape, (text.shape, self.text.shape)
        nv = self.frames if frames_valid is None else int(frames_valid)
        assert 0 < nv <= self.frames and (nv == self.frames or self.valid_len is not None)
        self.valid_len_buf.fill_(nv)
        self.valid_len1_buf.fill_(nv + 1)
        self.text.copy_(text.to(torch.int32))
        self.cond.copy_(cond)
        self.tvals.copy_(tvals)
        if self.seq_len is not None:
            assert seq_len is not None
            sl = seq_len.to(device=self.device, dtype=torch.int32)
            for half in range(2 if self.use_cfg else 1):
                self.seq_len[half * B:(half + 1) * B].copy_(sl)
            self.seq_len1.copy_(self.seq_len + 1)


class UNetT(Backbone):
    """Drop-in for upstream F5-TTS's UNetT (inference only) in its E2TTS_Base form."""

    _precompute, _forward, _ode_sample = "f5_unett_precompute", "f5_unett_forward", "f5_unett_ode_sample"
    _session_cls = UNetTSession

    def __init__(self, *, dim, depth=8, heads=8, dim_head=64, dropout=0.0, ff_mult=4, mel_dim=100,
                 text_num_embeds=256, text_dim=None, text_mask_padding=False, qk_norm=None, conv_layers=0,
                 pe_attn_head: Optional[int] = None, skip_connect_type="concat", device: str | torch.device = "cuda"):
        if text_dim is None:
            text_dim = mel_dim
        if skip_connect_type != "concat":
            raise ValueError(f'skip_connect_type {skip_connect_type!r} is not built: only "concat" (E2TTS_Base)')
        if qk_norm is not None:
            raise ValueError(f"qk_norm {qk_norm!r} is not built: only None (E2TTS_Base)")
        if conv_layers != 0:
            raise ValueError(f"conv_layers {conv_layers} is not built: only 0 (E2TTS_Base has no ConvNeXt text blocks)")
        if text_mask_padding:
            raise ValueError("text_mask_padding=True is not built: E2TTS_Base keeps filler tokens unmasked")
        if not isinstance(depth, int) or depth <= 0 or depth % 2:
            raise ValueError(f"depth must be a positive even number (the skips pair layer i with depth - 1 - i), not {depth!r}")
        if text_dim % 4:
            raise ValueError(f"text_dim must be a multiple of 4, not {text_dim}")
        super().__init__(dim=dim, depth=depth, heads=heads, dim_head=dim_head, dropout=dropout,
                         pe_attn_head=pe_attn_head, device=device)
        self.config = UNetTConfig(dim=dim, depth=depth, heads=heads, dim_head=dim_head, ff_mult=ff_mult,
                                  mel_dim=mel_dim, text_num_embeds=text_num_embeds, text_dim=text_dim,
                                  pe_attn_head=pe_attn_head)

    def load_weights(self, weights: Weights) -> "UNetT":
        """Upstream-named weights (an upstream state dict: see checkpoint_state, which this applies)."""
        self.packed = self._new_packed().load(checkpoint_state(dict(weights), self.config))
        return self

    def _new_packed(self) -> PackedUNetT:
        return PackedUNetT(self.config, self.device)
