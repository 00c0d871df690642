"""DurationPredictor — host-side mirror of f5_tts_mlx/duration.py:97-253 (inference branch).

Same constructor shapes as the reference (`DurationPredictor(transformer=DurationTransformer(dim=512,
depth=8, heads=8, text_dim=512, ff_mult=2, conv_layers=2, text_num_embeds=...), vocab_char_map=...)`,
cfm.py:428-440) and the same call `predictor(mel_or_wave, text, lens=None) -> seconds (b,)`.
Arithmetic: libf5b200 `f5_duration_forward` (the DiT's kernels + an RMSNorm/masked-mean/Softplus
head).  Training (`return_loss=True`) is out of scope.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch

from . import _lib
from .audio import MelSpec
from .dit import _check_prefix_padding, rope_table
from .utils import list_str_to_idx, list_str_to_tensor
from .weights import (ConvNextWeightsC, DitBlockWeightsC, Weights, _round_up, pack_grouped_conv, text_pos_table)


class DurationWeightsC(C.Structure):
    _fields_ = [
        ("dim", C.c_int32), ("depth", C.c_int32), ("heads", C.c_int32), ("ff_inner", C.c_int32),
        ("mel_dim", C.c_int32), ("text_dim", C.c_int32), ("text_inner", C.c_int32), ("conv_layers", C.c_int32),
        ("text_rows", C.c_int32), ("text_max_pos", C.c_int32), ("ct_ld", C.c_int32), ("reserved", C.c_int32),
        ("text_emb", C.c_void_p), ("text_pos", C.c_void_p),
        ("text_blocks", C.POINTER(ConvNextWeightsC)),
        ("in_w", C.c_void_p), ("in_b", C.c_void_p),
        ("conv_w", C.c_void_p * 2), ("conv_b", C.c_void_p * 2),
        ("blocks", C.POINTER(DitBlockWeightsC)),
        ("zeros", C.c_void_p), ("norm_w", C.c_void_p), ("pred_w", C.c_void_p),
    ]


class DurationBuffersC(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("frames", C.c_int32), ("text_len_max", C.c_int32), ("reserved", C.c_int32),
        ("text", C.c_void_p), ("lens", C.c_void_p), ("inp", C.c_void_p), ("rope", C.c_void_p),
        ("text_x", C.c_void_p), ("text_a", C.c_void_p), ("text_h", C.c_void_p), ("text_g", C.c_void_p),
        ("grn_nx", C.c_void_p), ("ct_bf16", C.c_void_p),
        ("x", C.c_void_p), ("h", C.c_void_p), ("a_bf16", C.c_void_p), ("c_bf16", C.c_void_p),
        ("qkv_bf16", C.c_void_p), ("ff_bf16", C.c_void_p), ("out", C.c_void_p),
    ]


class DurationTransformer:
    """duration.py:97-131 — configuration holder (the compute lives in DurationPredictor)."""

    def __init__(self, *, dim, depth=8, heads=8, dim_head=64, dropout=0.0, ff_mult=4, mel_dim=100,
                 text_num_embeds=256, text_dim=None, conv_layers=0):
        if text_dim is None:
            text_dim = mel_dim
        if dim_head != 64 or dim != heads * dim_head:
            raise ValueError("libf5b200 supports dim_head == 64 and dim == heads * 64")
        if dim % 128 != 0 or 64 % (dim // 16) != 0:
            raise ValueError(f"libf5b200 supports dim 128, 256, 512 or 1024, not {dim}: the conv position embedding's "
                             "dim/16-channel groups must tile 64-channel blocks")
        if conv_layers <= 0:
            raise NotImplementedError("conv_layers == 0 (no positional table) is not on the accelerated path")
        self.dim, self.depth, self.heads, self.ff_mult = dim, depth, heads, ff_mult
        self.mel_dim, self.text_num_embeds, self.text_dim, self.conv_layers = mel_dim, text_num_embeds, text_dim, conv_layers

    @property
    def ff_inner(self) -> int:
        return int(self.dim * self.ff_mult)


class DurationPredictor:
    def __init__(self, transformer: DurationTransformer, num_channels=None, mel_spec_kwargs: dict = dict(),
                 vocab_char_map: Optional[Dict[str, int]] = None, device: str | torch.device = "cuda"):
        self._mel_spec = MelSpec(**mel_spec_kwargs)
        self.num_channels = num_channels if num_channels is not None else self._mel_spec.n_mels
        self.transformer = transformer
        self.dim = transformer.dim
        self._vocab_char_map = vocab_char_map
        self.device = torch.device(device)
        self._t: Dict[str, torch.Tensor] = {}
        self._c: Optional[DurationWeightsC] = None
        self._bufs: Dict[tuple, tuple] = {}

    def load_weights(self, weights: Weights | list) -> "DurationPredictor":
        """MLX-named parameters of duration_v2.safetensors: `transformer.…`, `to_pred.layers.0.weight`."""
        W = dict(weights)
        tr, dev = self.transformer, self.device
        D, Ct = tr.dim, tr.text_dim
        f32 = lambda t: t.detach().float().contiguous().to(dev)
        bf = lambda t: t.detach().float().to(dev).bfloat16().contiguous()
        T = self._t
        P = "transformer."
        T["text_emb"] = f32(W[P + "text_embed.text_embed.weight"])
        T["text_pos"] = text_pos_table(Ct).to(dev)
        for i in range(tr.conv_layers):
            p = P + f"text_embed.text_blocks.layers.{i}."
            T[f"tb{i}.dw_w"] = f32(W[p + "dwconv.weight"][:, :, 0].t()); T[f"tb{i}.dw_b"] = f32(W[p + "dwconv.bias"])
            T[f"tb{i}.ln_w"] = f32(W[p + "norm.weight"]); T[f"tb{i}.ln_b"] = f32(W[p + "norm.bias"])
            T[f"tb{i}.pw1_w"] = bf(W[p + "pwconv1.weight"]); T[f"tb{i}.pw1_b"] = f32(W[p + "pwconv1.bias"])
            T[f"tb{i}.grn_gamma"] = f32(W[p + "grn.gamma"].reshape(-1)); T[f"tb{i}.grn_beta"] = f32(W[p + "grn.beta"].reshape(-1))
            T[f"tb{i}.pw2_w"] = bf(W[p + "pwconv2.weight"]); T[f"tb{i}.pw2_b"] = f32(W[p + "pwconv2.bias"])
        self.ct_ld = _round_up(tr.mel_dim + Ct, 64)
        pw = W[P + "input_embed.proj.weight"].float()
        wp = torch.zeros(D, self.ct_ld); wp[:, : tr.mel_dim + Ct] = pw
        T["in_w"] = bf(wp); T["in_b"] = f32(W[P + "input_embed.proj.bias"])
        for j, lj in enumerate((0, 2)):
            p = P + f"input_embed.conv_pos_embed.conv1d.layers.{lj}."
            T[f"conv_w{j}"] = bf(pack_grouped_conv(W[p + "weight"].float())); T[f"conv_b{j}"] = f32(W[p + "bias"])
        for i in range(tr.depth):
            p = P + f"transformer_blocks.{i}."
            T[f"blk{i}.qkv_w"] = bf(torch.cat([W[p + f"attn.to_{n}.weight"].float() for n in "qkv"], 0))
            T[f"blk{i}.qkv_b"] = f32(torch.cat([W[p + f"attn.to_{n}.bias"].float() for n in "qkv"], 0))
            T[f"blk{i}.out_w"] = bf(W[p + "attn.to_out.layers.0.weight"]); T[f"blk{i}.out_b"] = f32(W[p + "attn.to_out.layers.0.bias"])
            T[f"blk{i}.ff1_w"] = bf(W[p + "ff.ff.layers.0.layers.0.weight"]); T[f"blk{i}.ff1_b"] = f32(W[p + "ff.ff.layers.0.layers.0.bias"])
            T[f"blk{i}.ff2_w"] = bf(W[p + "ff.ff.layers.2.weight"]); T[f"blk{i}.ff2_b"] = f32(W[p + "ff.ff.layers.2.bias"])
        T["zeros"] = torch.zeros(D, device=dev)
        T["norm_w"] = f32(W[P + "norm_out.weight"])
        T["pred_w"] = f32(W["to_pred.layers.0.weight"].reshape(-1))
        c = DurationWeightsC()
        c.dim, c.depth, c.heads, c.ff_inner = D, tr.depth, tr.heads, tr.ff_inner
        c.mel_dim, c.text_dim, c.text_inner, c.conv_layers = tr.mel_dim, Ct, 2 * Ct, tr.conv_layers
        c.text_rows, c.text_max_pos, c.ct_ld = tr.text_num_embeds + 1, 4096, self.ct_ld
        for n in ("text_emb", "text_pos", "in_w", "in_b", "zeros", "norm_w", "pred_w"):
            setattr(c, n, T[n].data_ptr())
        tbs = (ConvNextWeightsC * tr.conv_layers)()
        for i in range(tr.conv_layers):
            for n, _ in ConvNextWeightsC._fields_:
                setattr(tbs[i], n, T[f"tb{i}.{n}"].data_ptr())
        blks = (DitBlockWeightsC * tr.depth)()
        for i in range(tr.depth):
            for n, _ in DitBlockWeightsC._fields_[:8]:          # the FP8 fields stay NULL: the duration model runs in bf16
                setattr(blks[i], n, T[f"blk{i}.{n}"].data_ptr())
        c.text_blocks, c.blocks = tbs, blks
        for j in range(2):
            c.conv_w[j] = T[f"conv_w{j}"].data_ptr(); c.conv_b[j] = T[f"conv_b{j}"].data_ptr()
        self._keep = (tbs, blks)
        self._c = c
        return self

    def _buffers(self, batch: int, frames: int, text_cols: int):
        key = (batch, frames, text_cols)
        if key not in self._bufs:
            if len(self._bufs) >= 4:
                self._bufs.pop(next(iter(self._bufs)))
            tr, dev = self.transformer, self.device
            D, F, Ct, R = tr.dim, tr.ff_inner, tr.text_dim, batch * frames
            z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=dev)
            bf16 = torch.bfloat16
            t = dict(text=z(batch, text_cols, dt=torch.int32), lens=z(batch, dt=torch.int32), inp=z(batch, frames, tr.mel_dim),
                     rope=rope_table(frames).to(dev), text_x=z(R, Ct), text_a=z(R, Ct, dt=bf16), text_h=z(R, 2 * Ct, dt=bf16),
                     text_g=z(R, 2 * Ct, dt=bf16), grn_nx=z(batch, 1 + (frames + 31) // 32, 2 * Ct),
                     ct_bf16=z(R, self.ct_ld, dt=bf16), x=z(R, D), h=z(R, D), a_bf16=z(R, D, dt=bf16), c_bf16=z(R, D, dt=bf16),
                     qkv_bf16=z(R, 3 * D, dt=bf16), ff_bf16=z(R, F, dt=bf16), out=z(batch))
            c = DurationBuffersC()
            c.batch, c.frames, c.text_len_max = batch, frames, text_cols
            for n, v in t.items():
                setattr(c, n, v.data_ptr())
            self._bufs[key] = (t, c)
        return self._bufs[key]

    @torch.no_grad()
    def __call__(self, inp: torch.Tensor, text, *, lens: Optional[torch.Tensor] = None, return_loss: bool = False):
        if return_loss:
            raise NotImplementedError("training loss (duration.py:233-253) is out of scope")
        if self._c is None:
            raise RuntimeError("DurationPredictor has no weights: call load_weights() first")
        if not inp.is_cuda:
            raise _lib.F5Error("DurationPredictor needs CUDA tensors: there is no CPU path")
        if inp.ndim == 2:                                        # raw wave (duration.py:206-209)
            inp = self._mel_spec(inp)
        inp = inp.float()
        batch, seq_len = inp.shape[:2]
        if isinstance(text, list):                               # duration.py:213-218
            text = list_str_to_idx(text, self._vocab_char_map) if self._vocab_char_map is not None else list_str_to_tensor(text)
            assert text.shape[0] == batch
        text = text.detach().cpu().to(torch.int32)
        _check_prefix_padding(text)
        if seq_len < text.shape[1]:                              # duration.py:220-222
            seq_len = text.shape[1]
            inp = torch.nn.functional.pad(inp, (0, 0, 0, seq_len - inp.shape[1]))
        if lens is None:
            lens = torch.full((batch,), seq_len)                 # duration.py:226-227
        t, c = self._buffers(batch, seq_len, text.shape[1])
        t["text"].copy_(text); t["lens"].copy_(lens.to(torch.int32)); t["inp"].copy_(inp)
        _lib.check(_lib.load().f5_duration_forward(C.byref(self._c), C.byref(c),
                                                   C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        return t["out"].clone()
