"""Thin torch-tensor wrappers over the C ABI (pointer + shape marshalling only; no arithmetic).

torch is used for device memory and streams.  Every function launches on the current torch CUDA
stream and returns its output tensor; nothing here falls back to a torch kernel.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib

ACT_NONE, ACT_GELU_TANH, ACT_GELU_ERF, ACT_MISH = 0, 1, 2, 3


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t: torch.Tensor | None) -> C.c_void_p | None:
    if t is None:
        return None
    return C.c_void_p(t.data_ptr())


def _need_cuda(*ts: torch.Tensor | None) -> None:
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.F5Error("f5_tts_mlx_b200 ops need CUDA tensors (no CPU fallback exists)")


def gemm(
    a: torch.Tensor,            # bf16 [rows, >=k] (row stride = a.stride(0))
    w: torch.Tensor,            # bf16 [n, taps*k_pad]
    out: torch.Tensor,          # bf16 / f32 [rows, >=n]
    *,
    n: int | None = None,
    k: int | None = None,
    bias: torch.Tensor | None = None,
    act: int = ACT_NONE,
    resid: torch.Tensor | None = None,
    gate: torch.Tensor | None = None,      # f32 [n], shared by all utterances: out = v * gate + resid
    row_len: torch.Tensor | None = None,   # i32 [num_batches]
    rope: torch.Tensor | None = None,      # f32 [rows_per_batch, 32, 2]
    rope_cols: int = 0,
    rope_col2: int = 0,                    # nonzero: [rope_col2, rope_col2 + rope_cols) is rotated too
    q_scale: float = 1.0,
    q_cols: int = 0,
    rows_per_batch: int = 0,
    num_batches: int = 1,
    batched_tiles: bool = False,
    conv_taps: int = 1,
    conv_pad: int = 0,
    conv_grouped: bool = False,
    conv_dilation: int = 0,                # frames between taps (0 or 1: adjacent frames)
    tile_n: int = 0,                       # 0 (auto), 64 or 128
    out2: torch.Tensor | None = None,          # bf16 [rows, >=n] second copy (or the fused-LN operand, see ln_scale)
    ln_scale: torch.Tensor | None = None,      # f32 [n]: producer mode — out2 = bf16(out * (1 + ln_scale)), ln_stats filled
    ln_stats: torch.Tensor | None = None,      # f32 [rows, n/64, 2] (sum, sum of squares) per 64 columns (with or
                                               # without ln_scale: the statistics of out)
    ln_in_stats: torch.Tensor | None = None,   # f32 [rows, k/64, 2]: consumer mode
    ln_tab: torch.Tensor | None = None,        # f32 [4, >=n] rows c1_hi, c1_lo, c2_hi, c2_lo
    ln_rms: bool = False,                      # RMSNorm consumer: ln_in_stats without ln_tab, the norm's gain in w
    ab_fp8: bool = False,                      # a and w are e4m3 bytes (uint8 / float8_e4m3fn tensors), k % 128 == 0
    acc_scale: float = 1.0,                    # multiplies the accumulator in FP8 mode (weight tensor scale)
    out2_fp8: bool = False,                    # out2 is written as e4m3 bytes (uint8 tensor)
    out_fp8: bool = False,                     # out (a uint8 tensor) is written as e4m3 bytes
    w_static: bool = False,                    # w is not written by the preceding kernel: its first tiles load before the PDL wait
    prefetch: torch.Tensor | None = None,      # weights of a later GEMM to pull into L2 while this one runs
    prefetch_bytes: int = 0,
    a_scale: torch.Tensor | None = None,      # f32 [k/64, >=rows] block scales of a (row stride = a_scale_ld)
    w_scale: torch.Tensor | None = None,      # f32 [n] per-output-channel weight scales
    out_scale: torch.Tensor | None = None,    # f32 [n/64, rows] written with a block-scaled e4m3 out (out_fp8)
    out2_scale: torch.Tensor | None = None,   # f32 [n/64, rows] written with a block-scaled e4m3 out2 (out2_fp8)
) -> torch.Tensor:
    _need_cuda(a, w, out, bias, resid, gate, row_len, rope, out2, ln_scale, ln_stats, ln_in_stats, ln_tab, prefetch,
               a_scale, w_scale, out_scale, out2_scale)
    if ab_fp8:
        a = a.view(torch.uint8) if a.dtype != torch.uint8 else a
        w = w.view(torch.uint8) if w.dtype != torch.uint8 else w
    else:
        assert a.dtype == torch.bfloat16 and w.dtype == torch.bfloat16
    assert a.stride(-1) == 1 and w.stride(-1) == 1 and out.stride(-1) == 1
    m = a.shape[0]
    g = _lib.GemmArgsDilated()
    g.a, g.lda = a.data_ptr(), a.stride(0)
    g.w, g.ldw = w.data_ptr(), w.stride(0)
    g.m = m
    g.n = n if n is not None else w.shape[0]
    g.k = k if k is not None else (64 if conv_grouped else a.shape[1])
    g.rows_per_batch = rows_per_batch
    g.num_batches = num_batches
    g.batched_tiles = int(batched_tiles)
    g.conv_taps, g.conv_pad, g.conv_grouped, g.conv_dilation = conv_taps, conv_pad, int(conv_grouped), conv_dilation
    g.act = act
    g.out_bf16 = int(out.dtype == torch.bfloat16 or out_fp8)
    g.out_fp8 = int(out_fp8)
    assert out.dtype in (torch.bfloat16, torch.float32) or (out_fp8 and out.dtype == torch.uint8)
    g.bias = bias.data_ptr() if bias is not None else None
    g.out, g.ldo = out.data_ptr(), out.stride(0)
    if resid is not None:
        assert resid.dtype == torch.float32
        g.resid, g.ldr = resid.data_ptr(), resid.stride(0)
    if gate is not None:
        assert gate.dtype == torch.float32 and gate.dim() == 1 and gate.stride(-1) == 1
        g.gate = gate.data_ptr()
    if row_len is not None:
        assert row_len.dtype == torch.int32
        g.row_len = row_len.data_ptr()
    if rope is not None:
        assert rope.dtype == torch.float32 and rope.is_contiguous()
        g.rope = rope.data_ptr()
    g.rope_cols, g.rope_col2, g.q_scale, g.q_cols = rope_cols, rope_col2, q_scale, q_cols
    g.tile_n = tile_n
    g.ab_fp8, g.acc_scale, g.out2_fp8 = int(ab_fp8), float(acc_scale), int(out2_fp8)
    g.w_static = int(w_static)
    if prefetch is not None:
        assert prefetch_bytes <= prefetch.numel() * prefetch.element_size()
        g.prefetch, g.prefetch_bytes = prefetch.data_ptr(), prefetch_bytes
    if out2 is not None:
        assert out2.dtype == (torch.uint8 if out2_fp8 else torch.bfloat16) and out2.stride(-1) == 1
        g.out2_bf16, g.ldo2 = out2.data_ptr(), out2.stride(0)
    if ln_scale is not None:
        assert ln_scale.dtype == torch.float32 and ln_stats is not None
        g.ln_scale = ln_scale.data_ptr()
    if ln_stats is not None:
        assert ln_stats.dtype == torch.float32 and out2 is not None
        g.ln_stats = ln_stats.data_ptr()
    if ln_rms:
        assert ln_in_stats is not None and ln_in_stats.dtype == torch.float32 and ln_tab is None
        g.ln_rms, g.ln_in_stats = 1, ln_in_stats.data_ptr()
    elif ln_in_stats is not None:
        assert ln_in_stats.dtype == torch.float32 and ln_tab is not None and ln_tab.dtype == torch.float32
        g.ln_in_stats, g.ln_tab, g.ln_tab_ld = ln_in_stats.data_ptr(), ln_tab.data_ptr(), ln_tab.stride(0)
    for t in (a_scale, w_scale, out_scale, out2_scale):
        assert t is None or (t.dtype == torch.float32 and t.stride(-1) == 1)
    if a_scale is not None:
        g.a_scale, g.a_scale_ld = a_scale.data_ptr(), a_scale.stride(0)
    if w_scale is not None:
        g.w_scale = w_scale.data_ptr()
    if out_scale is not None:
        assert out_scale.is_contiguous() and out_scale.shape[-1] == m
        g.out_scale = out_scale.data_ptr()
    if out2_scale is not None:
        assert out2_scale.is_contiguous() and out2_scale.shape[-1] == m
        g.out2_scale = out2_scale.data_ptr()
    _lib.check(_lib.load().f5_gemm_bf16(C.cast(C.pointer(g), C.POINTER(_lib.GemmArgs)), _stream()))
    return out
