"""Vocos vocoder — host-side stand-in for `vocos_mlx.Vocos` as the reference uses it
(cfm.py:19,446,471: `vocoder=vocos.decode`, called as `vocoder(out)` on a (b, n, 100) mel at
cfm.py:399-400).  Arithmetic: libf5b200 `f5_vocos_decode` (wgmma GEMMs, dwconv+LN kernel,
warp-shuffle inverse FFT + overlap-add).

vocos-mlx is a third-party package that is not vendored in the reference tree; the architecture
here is the public Vocos "mel-24khz" design, and the ISTFT
normalisation/trim convention is an explicit switch (VocosConfig.istft_norm / istft_trim).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch

from . import _lib
from .audio import hanning
from .weights import VocosConfig, Weights, _round_up


class VocosBlockWeightsC(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in
                ("dw_w", "dw_b", "ln_w", "ln_b", "pw1_w", "pw1_b", "pw2_w", "pw2_b", "gamma")]


class VocosWeightsC(C.Structure):
    _fields_ = [
        ("n_mels", C.c_int32), ("dim", C.c_int32), ("inner", C.c_int32), ("num_layers", C.c_int32),
        ("head_ld", C.c_int32), ("hop", C.c_int32), ("istft_norm_sq", C.c_int32), ("istft_trim", C.c_int32),
        ("embed_w", C.c_void_p), ("embed_b", C.c_void_p), ("norm_w", C.c_void_p), ("norm_b", C.c_void_p),
        ("blocks", C.POINTER(VocosBlockWeightsC)),
        ("final_w", C.c_void_p), ("final_b", C.c_void_p), ("head_w", C.c_void_p), ("head_b", C.c_void_p),
        ("window", C.c_void_p),
    ]


class VocosBuffersC(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("frames", C.c_int32), ("out_len", C.c_int32), ("reserved", C.c_int32),
        ("mel_bf16", C.c_void_p), ("h", C.c_void_p), ("x", C.c_void_p), ("a_bf16", C.c_void_p),
        ("i_bf16", C.c_void_p), ("head", C.c_void_p), ("frames_f32", C.c_void_p),
    ]


class Vocos:
    def __init__(self, config: VocosConfig = VocosConfig(), device: str | torch.device = "cuda"):
        self.config = config
        self.device = torch.device(device)
        self.head_ld = _round_up(config.n_fft + 2, 4)
        self._t: Dict[str, torch.Tensor] = {}
        self._c: Optional[VocosWeightsC] = None
        self._bufs: Dict[tuple, tuple] = {}

    def load_weights(self, W: Weights) -> "Vocos":
        vc, dev = self.config, self.device
        f32 = lambda t: t.detach().float().contiguous().to(dev)
        bf = lambda t: t.detach().float().to(dev).bfloat16().contiguous()
        T = self._t
        ew = W["vocos.backbone.embed.weight"].float()                  # (D, 7, n_mels) MLX layout
        ewp = torch.zeros(vc.dim, 7, 128); ewp[:, :, :vc.n_mels] = ew
        T["embed_w"] = bf(ewp.reshape(vc.dim, 7 * 128)); T["embed_b"] = f32(W["vocos.backbone.embed.bias"])
        T["norm_w"] = f32(W["vocos.backbone.norm.weight"]); T["norm_b"] = f32(W["vocos.backbone.norm.bias"])
        for i in range(vc.num_layers):
            p = f"vocos.backbone.convnext.{i}."
            T[f"b{i}.dw_w"] = f32(W[p + "dwconv.weight"][:, :, 0].t())
            T[f"b{i}.dw_b"] = f32(W[p + "dwconv.bias"])
            T[f"b{i}.ln_w"] = f32(W[p + "norm.weight"]); T[f"b{i}.ln_b"] = f32(W[p + "norm.bias"])
            T[f"b{i}.pw1_w"] = bf(W[p + "pwconv1.weight"]); T[f"b{i}.pw1_b"] = f32(W[p + "pwconv1.bias"])
            T[f"b{i}.pw2_w"] = bf(W[p + "pwconv2.weight"]); T[f"b{i}.pw2_b"] = f32(W[p + "pwconv2.bias"])
            T[f"b{i}.gamma"] = f32(W[p + "gamma"].reshape(-1))
        T["final_w"] = f32(W["vocos.backbone.final_layer_norm.weight"])
        T["final_b"] = f32(W["vocos.backbone.final_layer_norm.bias"])
        hw = torch.zeros(self.head_ld, vc.dim); hw[: vc.n_fft + 2] = W["vocos.head.out.weight"].float()
        hb = torch.zeros(self.head_ld); hb[: vc.n_fft + 2] = W["vocos.head.out.bias"].float()
        T["head_w"] = bf(hw); T["head_b"] = f32(hb)
        T["window"] = hanning(vc.n_fft).to(dev)
        c = VocosWeightsC()
        c.n_mels, c.dim, c.inner, c.num_layers = vc.n_mels, vc.dim, vc.intermediate_dim, vc.num_layers
        c.head_ld, c.hop = self.head_ld, vc.hop_length
        c.istft_norm_sq = int(vc.istft_norm == "window_sq")
        c.istft_trim = vc.n_fft // 2 if vc.istft_trim else 0
        for n in ("embed_w", "embed_b", "norm_w", "norm_b", "final_w", "final_b", "head_w", "head_b", "window"):
            setattr(c, n, T[n].data_ptr())
        blks = (VocosBlockWeightsC * vc.num_layers)()
        for i in range(vc.num_layers):
            for n, _ in VocosBlockWeightsC._fields_:
                setattr(blks[i], n, T[f"b{i}.{n}"].data_ptr())
        c.blocks = blks
        self._blks = blks
        self._c = c
        return self

    def out_len(self, frames: int) -> int:
        vc = self.config
        full = (frames - 1) * vc.hop_length + vc.n_fft
        return full - vc.n_fft if vc.istft_trim else full

    def _buffers(self, batch: int, frames: int):
        key = (batch, frames)
        if key not in self._bufs:
            if len(self._bufs) >= 4:
                self._bufs.pop(next(iter(self._bufs)))
            vc, dev = self.config, self.device
            R = batch * frames
            t = dict(
                mel_bf16=torch.zeros(R, 128, dtype=torch.bfloat16, device=dev),
                h=torch.zeros(R, vc.dim, device=dev), x=torch.zeros(R, vc.dim, device=dev),
                a_bf16=torch.zeros(R, vc.dim, dtype=torch.bfloat16, device=dev),
                i_bf16=torch.zeros(R, vc.intermediate_dim, dtype=torch.bfloat16, device=dev),
                head=torch.zeros(R, self.head_ld, device=dev),
                frames_f32=torch.zeros(R, vc.n_fft, device=dev),
            )
            c = VocosBuffersC()
            c.batch, c.frames, c.out_len = batch, frames, self.out_len(frames)
            for n, v in t.items():
                setattr(c, n, v.data_ptr())
            self._bufs[key] = (t, c)
        return self._bufs[key]

    def decode(self, mel: torch.Tensor) -> torch.Tensor:
        """(b, n, n_mels) log-mel -> waveform; batch 1 returns a 1-D tensor like vocos-mlx (the
        reference slices `wave[audio.shape[0]:]`, generate.py:183), batch > 1 returns (b, samples)."""
        if self._c is None:
            raise RuntimeError("Vocos has no weights: call load_weights() first")
        if not mel.is_cuda:
            raise _lib.F5Error("Vocos.decode needs a CUDA tensor: there is no CPU path")
        b, n, _ = mel.shape
        _, c = self._buffers(b, n)
        mel = mel.float().contiguous()
        wave = torch.empty(b, max(c.out_len, 0), device=mel.device, dtype=torch.float32)
        if c.out_len <= 0:          # a single frame with centre trimming leaves no samples
            return wave[0] if b == 1 else wave
        _lib.check(_lib.load().f5_vocos_decode(C.byref(self._c), C.byref(c), C.c_void_p(mel.data_ptr()),
                                               C.c_void_p(wave.data_ptr()),
                                               C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        return wave[0] if b == 1 else wave

    __call__ = decode
