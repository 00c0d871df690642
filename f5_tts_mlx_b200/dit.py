"""DiT — host-side mirror of the reference's `f5_tts_mlx.dit.DiT` (dit.py:331-401).

Same constructor arguments and `__call__(x, cond, text, time, drop_audio_cond, drop_text, mask)`
signature, torch CUDA tensors instead of mx.arrays.  All arithmetic runs in libf5b200 (sm_90a
kernels); this module only owns device buffers and fills the C structs.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch

from . import _lib
from .weights import DiTConfig, PackedDiT, Weights


class DitBuffersC(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("frames", C.c_int32), ("cfg", C.c_int32), ("n_times", C.c_int32),
        ("text_len_max", C.c_int32), ("drop_flags", C.c_int32),
        ("text", C.c_void_p), ("text_len", C.c_void_p), ("seq_len", C.c_void_p), ("cond", C.c_void_p),
        ("tvals", C.c_void_p), ("rope", C.c_void_p),
        ("hoist", C.c_void_p), ("mod_table", C.c_void_p),
        ("text_x", C.c_void_p), ("text_a", C.c_void_p), ("text_h", C.c_void_p), ("text_g", C.c_void_p),
        ("grn_nx", C.c_void_p), ("ct_bf16", C.c_void_p), ("silu_t", C.c_void_p),
        ("y_bf16", C.c_void_p), ("x", C.c_void_p), ("h", C.c_void_p), ("a_bf16", C.c_void_p),
        ("c_bf16", C.c_void_p), ("qkv_bf16", C.c_void_p), ("ff_bf16", C.c_void_p), ("v", C.c_void_p),
        ("ln_stats", C.c_void_p), ("ln_tab", C.c_void_p), ("ln_prep", C.c_void_p),
        ("valid_len", C.c_void_p), ("a_fp8", C.c_void_p),
    ]


def rope_table(frames: int, dim_head: int = 64, base: float = 10000.0) -> torch.Tensor:
    """(cos, sin) of n * theta_i, [frames, dim_head/2, 2] fp32 — RotaryEmbedding.forward_from_seq_len
    (rope.py:38-53): theta_i = base^(-2i/dim); freqs are duplicated per adjacent pair there, which is
    why one (cos, sin) per pair suffices here.  Host fp32 math, uploaded once per session."""
    inv_freq = 1.0 / (base ** (torch.arange(0, dim_head, 2, dtype=torch.float32) / dim_head))
    t = torch.arange(frames, dtype=torch.float32)
    freqs = torch.einsum("i,j->ij", t, inv_freq)
    return torch.stack([freqs.cos(), freqs.sin()], dim=-1).contiguous()


class DitSession:
    """Device buffers (f5_dit_buffers) for `batch` utterances padded to `frames`, `n_times` DiT
    evaluation times, with or without the CFG batch doubling."""

    def __init__(self, cfg: DiTConfig, ct_ld: int, batch: int, frames: int, n_times: int, use_cfg: bool,
                 text_cols: int, device: torch.device, masked: bool, fused_adaln: bool = True, fp8: bool = False):
        self.cfg, self.batch, self.frames, self.n_times, self.use_cfg = cfg, batch, frames, n_times, use_cfg
        self.device = device
        D, F, Ct = cfg.dim, cfg.ff_inner, cfg.text_dim
        BU = (2 if use_cfg else 1) * batch
        R = BU * frames
        self.rows, self.row_utts = R, BU
        f32, bf16, i32 = torch.float32, torch.bfloat16, torch.int32
        z = lambda *s, dt=f32: torch.zeros(*s, dtype=dt, device=device)
        self.text = z(batch, max(text_cols, 1), dt=i32)
        self.text_len = z(BU, dt=i32)
        self.seq_len = z(BU, dt=i32) if masked else None
        self.valid_len_buf = torch.full((BU,), frames, dtype=i32, device=device)   # frame bucketing (f5_dit_buffers.valid_len)
        self.valid_len = None
        self.cond = z(batch, frames, cfg.mel_dim)
        self.tvals = z(n_times)
        self.rope = rope_table(frames, cfg.dim_head).to(device)
        NM = cfg.depth * 6 * D + 2 * D
        self.hoist = z(R, D)
        self.mod_table = z(n_times, NM)
        self.text_x = z(R, Ct)
        self.text_a = z(R, Ct, dt=bf16)
        self.text_h = z(R, 2 * Ct, dt=bf16)
        self.text_g = z(R, 2 * Ct, dt=bf16)
        self.grn_nx = z(BU, 1 + (frames + 31) // 32, 2 * Ct)
        self.ct_bf16 = z(R, ct_ld, dt=bf16)
        self.silu_t = z(n_times, D, dt=bf16)
        self.y_bf16 = z(R, 128, dt=bf16)
        self.x = z(R, D)
        self.h = z(R, D)
        self.a_bf16 = z(R, D, dt=bf16)
        self.c_bf16 = z(R, D, dt=bf16)
        self.qkv_bf16 = z(R, 3 * D, dt=bf16)
        self.ff_bf16 = z(R, F, dt=bf16)
        self.v = z(R, cfg.mel_dim)
        # fused AdaLN (f5_gemm_args.ln_*): per-row chunk statistics, the c1/c2 operand tables of every consuming
        # Linear for every evaluation time, and the bf16 operand rows of the table GEMMs
        self.ln_tab_ld = cfg.depth * (3 * D + F) + 128
        self.ln_stats = z(R, D // 64, 2) if fused_adaln else None
        self.ln_tab = z(4 * n_times, self.ln_tab_ld) if fused_adaln else None
        self.ln_prep = z(2 * cfg.depth + 1, 4 * n_times, D, dt=bf16) if fused_adaln else None
        self.a_fp8 = z(R, D, dt=torch.uint8) if (fp8 and fused_adaln) else None   # e4m3 operand of the QKV / FF1 GEMMs
        c = DitBuffersC()
        c.batch, c.frames, c.cfg, c.n_times = batch, frames, int(use_cfg), n_times
        c.text_len_max, c.drop_flags = self.text.shape[1], 0
        for name, _ in DitBuffersC._fields_[6:]:
            t = getattr(self, name)
            setattr(c, name, t.data_ptr() if t is not None else None)
        self.c = c

    def use_bucketing(self) -> None:
        """Bind the valid-length buffer: from now on `frames` is a bucket size and set_inputs(frames_valid=N) says
        how many rows are real (must be called before the plan's graph is captured)."""
        self.valid_len = self.valid_len_buf
        self.c.valid_len = self.valid_len_buf.data_ptr()

    def set_inputs(self, text: torch.Tensor, cond: torch.Tensor, tvals: torch.Tensor,
                   seq_len: Optional[torch.Tensor], frames_valid: Optional[int] = None) -> None:
        """text int [batch, nt] (pad -1), cond fp32 [batch, frames, mel], tvals fp32 [n_times],
        seq_len int [batch] or None; frames_valid: real frames per utterance when `frames` is a bucket."""
        B = self.batch
        assert text.shape == self.text.shape, (text.shape, self.text.shape)
        nv = self.frames if frames_valid is None else int(frames_valid)
        assert 0 < nv <= self.frames and (nv == self.frames or self.valid_len is not None)
        self.valid_len_buf.fill_(nv)
        self.text.copy_(text.to(torch.int32))
        tl = (text != -1).sum(dim=-1).clamp(max=nv).to(torch.int32)
        self.text_len[:B].copy_(tl)
        if self.use_cfg:
            self.text_len[B:].copy_(tl)
        self.cond.copy_(cond)
        self.tvals.copy_(tvals)
        if self.seq_len is not None:
            assert seq_len is not None
            sl = seq_len.to(torch.int32)
            self.seq_len[:B].copy_(sl)
            if self.use_cfg:
                self.seq_len[B:].copy_(sl)


def _check_prefix_padding(text: torch.Tensor) -> None:
    """The kernels treat the text mask (dit.py:207, `text == 0` after the +1 shift) as a prefix
    mask, which is what pad_sequence(-1) produces; reject anything else loudly."""
    valid = (text != -1)
    n = valid.sum(dim=-1, keepdim=True)
    expect = torch.arange(text.shape[1], device=text.device)[None, :] < n
    if not torch.equal(valid, expect):
        raise ValueError("text ids must be right-padded with -1 (interior -1 is not supported)")


class DiT:
    """Drop-in for f5_tts_mlx.dit.DiT (inference only)."""

    def __init__(self, *, dim, depth=8, heads=8, dim_head=64, dropout=0.0, ff_mult=4, mel_dim=100,
                 text_num_embeds=256, text_dim=None, text_mask_padding=True, conv_layers=0,
                 device: str | torch.device = "cuda", fused_adaln: bool = True, fp8: bool = False):
        if text_dim is None:
            text_dim = mel_dim
        if dim_head != 64 or dim != heads * dim_head:
            raise ValueError("libf5b200 supports dim_head == 64 and dim == heads * 64")
        if dim % 128 != 0 or not (256 <= dim <= 1024):
            raise ValueError("libf5b200 supports 256 <= dim <= 1024, dim a multiple of 128 (see check_common in csrc/dit.cu)")
        if not text_mask_padding:
            raise NotImplementedError("text_mask_padding=False is not on the accelerated path")
        if dropout != 0.0:
            raise NotImplementedError("inference path: dropout must be 0")
        self.config = DiTConfig(dim=dim, depth=depth, heads=heads, dim_head=dim_head, ff_mult=ff_mult,
                                mel_dim=mel_dim, text_num_embeds=text_num_embeds, text_dim=text_dim,
                                conv_layers=conv_layers, text_mask_padding=text_mask_padding)
        self.dim, self.depth = dim, depth
        # AdaLN LayerNorm+modulate folded into the neighbouring GEMM epilogues (default); False keeps the separate
        # f5_ln_modulate launches (kept for A/B measurements and as a cross-check in the tests)
        self.fused_adaln = bool(fused_adaln)
        # FP8 mode — the H100 analogue of the reference's quantised `--q` checkpoints (cfm.py:451-452,510-515): the
        # QKV and FF1 GEMMs (63 % of a block's FLOPs) run on e4m3 operands (e4m3 wgmma): weights quantised per
        # tensor at pack time, activations written as e4m3 by the producing GEMM's epilogue.  Lossy like `--q`; gated
        # by the same derived-drift rule against the oracle's e4m3 emulation (tests/test_gpu_parity.py).
        self.fp8 = bool(fp8)
        if self.fp8 and not self.fused_adaln:
            raise ValueError("fp8=True needs fused_adaln=True (the e4m3 operand is written by the GEMM epilogues)")
        self.device = torch.device(device)
        self.packed: Optional[PackedDiT] = None
        self._sessions: Dict[tuple, DitSession] = {}
        self.session_cache_size = 12

    # -- weights --
    def load_weights(self, weights: Weights | list) -> "DiT":
        """Accepts the MLX-named parameter dict (or list of pairs, like mlx `load_weights`); names may
        carry or omit the leading 'transformer.' (the reference loads them through F5TTS)."""
        W = dict(weights)
        if not any(k.startswith("transformer.") for k in W):
            W = {"transformer." + k: v for k, v in W.items()}
        self.packed = PackedDiT(self.config, self.device, fp8=self.fp8).load(W)
        return self

    def allocate_weights(self) -> "DiT":
        """Allocate the packed buffer without filling it (non-source ranks before the broadcast)."""
        self.packed = PackedDiT(self.config, self.device, fp8=self.fp8)
        return self

    def _require_weights(self) -> PackedDiT:
        if self.packed is None:
            raise RuntimeError("DiT has no weights: call load_weights() first")
        return self.packed

    # -- sessions --
    def session(self, batch: int, frames: int, n_times: int, use_cfg: bool, text_cols: int,
                masked: bool, bucketed: bool = False) -> DitSession:
        key = (batch, frames, n_times, use_cfg, text_cols, masked, self.fused_adaln, bucketed, self.fp8)
        s = self._sessions.pop(key, None)
        if s is None:
            while len(self._sessions) >= self.session_cache_size:
                self._sessions.pop(next(iter(self._sessions)))
            s = DitSession(self.config, self._require_weights().ct_ld, batch, frames, n_times, use_cfg,
                           text_cols, self.device, masked, self.fused_adaln, self.fp8)
            if bucketed:
                s.use_bucketing()
        self._sessions[key] = s          # LRU order: most recently used last
        return s

    def release_session(self, s: DitSession) -> None:
        for k, v in list(self._sessions.items()):
            if v is s:
                del self._sessions[k]

    def precompute(self, s: DitSession) -> None:
        lib = _lib.load()
        _lib.check(lib.f5_dit_precompute(C.byref(self._require_weights().c_struct()), C.byref(s.c),
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream)))

    def forward_session(self, s: DitSession, time_index: int) -> torch.Tensor:
        lib = _lib.load()
        _lib.check(lib.f5_dit_forward(C.byref(self._require_weights().c_struct()), C.byref(s.c),
                                      int(time_index), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        return s.v

    def __call__(self, x: torch.Tensor, cond: torch.Tensor, text: torch.Tensor, time: torch.Tensor,
                 drop_audio_cond: bool = False, drop_text: bool = False,
                 mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """One flow-field evaluation, dit.py:374-401.  x, cond: (b, n, mel) fp32; text: (b, nt) int,
        pad -1; time: scalar or (b,) with equal entries; mask: (b, n) bool or None."""
        if not x.is_cuda:
            raise _lib.F5Error("DiT needs CUDA tensors: there is no CPU path")
        b, n, d = x.shape
        time = torch.as_tensor(time, dtype=torch.float32).reshape(-1)
        if time.numel() > 1 and not torch.all(time == time[0]):
            raise NotImplementedError("per-utterance time values are not on the inference path")
        text = text.to(self.device)
        _check_prefix_padding(text)
        s = self.session(b, n, 1, False, text.shape[1], mask is not None)
        seq_len = None
        if mask is not None:
            seq_len = mask.sum(dim=-1)
            expect = torch.arange(n, device=mask.device)[None, :] < seq_len[:, None]
            if not torch.equal(mask.bool(), expect):
                raise ValueError("mask must be a prefix (lens_to_mask) mask")
        s.set_inputs(text, cond.float(), time[:1].to(self.device), seq_len)
        s.c.drop_flags = (1 if drop_audio_cond else 0) | (2 if drop_text else 0)
        s.y_bf16.zero_()
        s.y_bf16[:, :d].copy_(x.reshape(b * n, d))
        self.precompute(s)
        v = self.forward_session(s, 0)
        return v.view(b, n, d).clone()
