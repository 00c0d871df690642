"""F5TTS / CFM — host-side mirror of `f5_tts_mlx.cfm.F5TTS` (cfm.py:128-402), inference only.

`sample()` keeps the reference's signature, defaults, return value `(out, trajectory)` and error
behaviour.  Host code here is bookkeeping only (the mask/duration prologue of cfm.py:279-336 on a
handful of integers, buffer management, CUDA-graph capture); every tensor operation of the hot
path is an sm_90a kernel in libf5b200 reached through the C ABI (f5_dit_precompute,
f5_ode_sample, f5_mel_forward, f5_vocos_decode).
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Callable, Dict, Literal, Optional, Tuple

import torch
import torch.nn.functional as F

from . import _lib
from .audio import MelSpec, resample
from .dit import DiT, DitSession, _check_prefix_padding
from .utils import default, exists, lens_to_mask, list_str_to_idx, list_str_to_tensor, pad_sequence

METHODS = {"euler": 0, "midpoint": 1, "rk4": 2}


def time_grid(steps: int, sway_sampling_coef: Optional[float]) -> torch.Tensor:
    """cfm.py:377-381 — fp32 grid of `steps` POINTS (steps-1 intervals) with sway warping."""
    t = torch.linspace(0, 1, steps, dtype=torch.float32)
    if exists(sway_sampling_coef):
        t = t + sway_sampling_coef * (torch.cos(math.pi / 2 * t) - 1 + t)
    return t


def ode_eval_times(t_grid: torch.Tensor, method: str) -> torch.Tensor:
    """Times at which the solver evaluates the DiT, in call order (f5_ode_eval_times)."""
    lib = _lib.load()
    tg = t_grid.contiguous().float().cpu()
    tp = tg.numpy().ctypes.data_as(C.POINTER(C.c_float))
    n = lib.f5_ode_eval_times(tp, tg.numel(), METHODS[method], None, 0)
    if n < 0:
        _lib.check(n)
    out = torch.empty(n, dtype=torch.float32)
    r = lib.f5_ode_eval_times(tp, tg.numel(), METHODS[method], out.numpy().ctypes.data_as(C.POINTER(C.c_float)), n)
    if r < 0:
        _lib.check(r)
    return out


def _odeint(func: Callable, y0: torch.Tensor, t: torch.Tensor, method: str) -> torch.Tensor:
    """Generic fixed-grid solvers with the reference's call pattern, for arbitrary `func` given as a
    Python callable (cfm.py:38-122).  The accelerated sample() does NOT go through these: its loop
    is f5_ode_sample.  The only tensor ops are the axpy updates of the solver itself."""
    ys = [y0]
    y = y0
    for i in range(len(t) - 1):
        tc = t[i]
        dt = t[i + 1] - tc
        if method == "euler":
            y = y + dt * func(tc, y)
        elif method == "midpoint":
            k1 = func(tc, y)
            k2 = func(tc + 0.5 * dt, y + 0.5 * dt * k1)
            y = y + dt * k2
        else:
            k1 = func(tc, y)
            k2 = func(tc + 0.5 * dt, y + 0.5 * dt * k1)
            k3 = func(tc + 0.5 * dt, y + 0.5 * dt * k2)
            k4 = func(tc + dt, y + dt * k3)
            y = y + (dt / 6) * (k1 + 2 * k2 + 2 * k3 + k4)
        ys.append(y)
    return torch.stack(ys)


def odeint_euler(func, y0, t):
    """cfm.py:38-61."""
    return _odeint(func, y0, t, "euler")


def odeint_midpoint(func, y0, t):
    """cfm.py:64-91."""
    return _odeint(func, y0, t, "midpoint")


def odeint_rk4(func, y0, t):
    """cfm.py:94-122."""
    return _odeint(func, y0, t, "rk4")


class _Plan:
    """Everything that is fixed for one (batch, frames, steps, method, sway, cfg) combination: the
    backbone's (DiT or UNetT) session buffers, ODE state buffers and the captured CUDA graph of precompute + ODE loop."""

    def __init__(self, model: "F5TTS", batch: int, frames: int, text_cols: int, steps: int, method: str,
                 sway: Optional[float], cfg_strength: float, masked: bool, keep_trajectory: bool, bucketed: bool = False):
        tr = model.transformer
        self.t_grid = time_grid(steps, sway)
        self.tvals = ode_eval_times(self.t_grid, method)
        self.use_cfg = cfg_strength >= 1e-5
        self.session: DitSession = tr.session(batch, frames, self.tvals.numel(), self.use_cfg, text_cols, masked, bucketed)
        dev, d = tr.device, model.num_channels
        self.steps, self.method, self.cfg_strength = steps, method, float(cfg_strength)
        self.keep_trajectory = keep_trajectory
        if keep_trajectory:
            self.trajectory = torch.zeros(steps, batch, frames, d, device=dev)
            self.y = self.trajectory[0]
        else:
            self.trajectory = None
            self.y = torch.zeros(batch, frames, d, device=dev)
        self.scratch = torch.zeros(2, batch, frames, d, device=dev) if method != "euler" else None
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.launches = 0

    def run_eager(self, model: "F5TTS") -> None:
        tr = model.transformer
        self.session.c.drop_flags = 0      # DiT.__call__ may have used this cached session with drop flags set
        tr.precompute(self.session)
        tr.ode_sample(self.session, self.t_grid, self.steps, METHODS[self.method], self.cfg_strength, self.y,
                      self.trajectory, self.scratch)

    def capture(self, model: "F5TTS") -> None:
        """Capture precompute + ODE loop into a CUDA graph (an eager pass must have run on this process before:
        it sets per-kernel attributes and validates the arguments).  Leaves the state buffer unchanged."""
        y0 = self.y.clone()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self.run_eager(model)
        self.graph = g
        self.y.copy_(y0)

    def run(self, model: "F5TTS", use_graph: bool) -> None:
        if not use_graph:
            self.run_eager(model)
            return
        if self.graph is None:
            y0 = self.y.clone()
            self.run_eager(model)
            torch.cuda.synchronize()
            self.y.copy_(y0)
            self.capture(model)
        self.graph.replay()


class F5TTS:
    """Drop-in for f5_tts_mlx.cfm.F5TTS (alias CFM); constructor per cfm.py:128-167."""

    def __init__(
        self,
        transformer: DiT,
        audio_drop_prob=0.3,
        cond_drop_prob=0.2,
        num_channels=None,
        mel_spec_module=None,
        mel_spec_kwargs: dict = dict(),
        frac_lengths_mask: Tuple[float, float] = (0.7, 1.0),
        vocab_char_map: Optional[Dict[str, int]] = None,
        vocoder: Optional[Callable] = None,
        duration_predictor=None,
    ):
        self.frac_lengths_mask = frac_lengths_mask
        self._mel_spec = default(mel_spec_module, MelSpec(**mel_spec_kwargs))
        self.num_channels = default(num_channels, self._mel_spec.n_mels)
        self.audio_drop_prob = audio_drop_prob
        self.cond_drop_prob = cond_drop_prob
        self.transformer = transformer
        self.dim = transformer.dim
        self._vocab_char_map = vocab_char_map
        self._vocoder = vocoder
        self._duration_predictor = duration_predictor
        self._plans: Dict[tuple, _Plan] = {}      # LRU, most recently used last
        self.plan_cache_size = 8
        # Plan reuse across utterances of different length (generate()'s sentence loop): 0 = every distinct
        # (frames, text columns) gets its own buffers + CUDA graph (the reference's exact shapes); k > 0 rounds the frame
        # count up to a multiple of k and the text columns to a multiple of text_bucket, the real length travelling
        # in a device-side scalar (f5_dit_buffers.valid_len) so one captured graph serves the whole bucket.
        self.frame_bucket = 0
        self.text_bucket = 32
        self.use_cuda_graph = True
        self.last_plan: Optional[_Plan] = None

    def eval(self):
        return self

    def __call__(self, *a, **k):
        raise NotImplementedError("training loss (cfm.py:169-251) is out of scope: inference path only")

    def predict_duration(self, cond, text, speed: float = 1.0):
        """cfm.py:253-262 (integer frame_rate = 24000 // 256 = 93, as the reference)."""
        if self._duration_predictor is None:
            raise ValueError("no duration predictor set")
        duration_in_sec = self._duration_predictor(cond, text)
        frame_rate = self._mel_spec.sample_rate // self._mel_spec.hop_length
        return (duration_in_sec * frame_rate / speed).to(torch.int32)

    def _plan(self, batch, frames, text_cols, steps, method, sway, cfg_strength, masked, keep_traj, bucketed=False) -> _Plan:
        key = (batch, frames, text_cols, steps, method, sway, float(cfg_strength), masked, keep_traj, bucketed)
        p = self._plans.pop(key, None)
        if p is None:
            while len(self._plans) >= max(1, self.plan_cache_size):
                old = self._plans.pop(next(iter(self._plans)))
                self.transformer.release_session(old.session)
            p = _Plan(self, batch, frames, text_cols, steps, method, sway, cfg_strength, masked, keep_traj, bucketed)
        self._plans[key] = p
        return p

    @torch.no_grad()
    def sample(
        self,
        cond: torch.Tensor,
        text,
        duration=None,
        *,
        lens: Optional[torch.Tensor] = None,
        steps=8,
        method: Literal["euler", "midpoint", "rk4"] = "rk4",
        cfg_strength=2.0,
        speed=1.0,
        sway_sampling_coef=-1.0,
        seed: Optional[int] = None,
        max_duration=4096,
        y0: Optional[torch.Tensor] = None,
        return_trajectory: bool = True,
        pad_frames: Optional[int] = None,
        frame_bucket: Optional[int] = None,
        cond_sample_rate: Optional[int] = None,
        edit_mask: Optional[torch.Tensor] = None,
    ) -> Tuple[torch.Tensor, torch.Tensor]:
        """cfm.py:264-402.  Extensions (default-compatible): `y0` injects the initial noise
        (b, n, mel) — MLX's RNG stream cannot be reproduced, so seeded parity is defined on injected
        noise; `return_trajectory=False` skips keeping all `steps` states (then `trajectory` is the
        final state with a leading axis of 1); `pad_frames` pads the batch to at least that many frames — a shard
        of a ragged batch must use the GLOBAL maximum (parallel.global_frames) to reproduce the unsharded result,
        because the reference's padding leaks into GRN and the ODE on padded frames; `frame_bucket` (default
        self.frame_bucket) reuses one plan / CUDA graph for all lengths of a bucket, results unchanged;
        `cond_sample_rate` is the rate of a raw-wave `cond` (None: the mel front-end's own rate, 24 kHz) — another rate
        is resampled on the device (audio.resample, torchaudio's default windowed sinc) before the mel.
        `edit_mask` (speech editing, upstream F5-TTS's `CFM.sample(edit_mask=)`): bool [b, n_c], n_c the conditioning's
        frame count (a raw-wave `cond`: the frames of its mel); False frames are regenerated, True frames condition.
        The conditioning mask becomes `lens_to_mask(lens) & edit_mask`, with columns past n_c counting as True.  The
        mask is not part of the plan: an edit reuses the buffers and CUDA graph of any call of the same shape."""
        dev = self.transformer.device
        if method not in METHODS:
            raise ValueError(f"Unknown method: {method}")

        # raw wave (cfm.py:283-286)
        resample_from = None
        if cond_sample_rate is not None and int(cond_sample_rate) != self._mel_spec.sample_rate:
            resample_from = int(cond_sample_rate)
        if cond.ndim == 2:
            if cond.shape[0] != 1:
                raise ValueError("raw-wave conditioning must have batch 1 (cfm.py:284)")
            wave = cond[0].to(dev)
            if resample_from is not None:
                wave = resample(wave, resample_from, self._mel_spec.sample_rate)
            cond = self._mel_spec(wave)
            assert cond.shape[-1] == self.num_channels
        elif resample_from is not None:
            raise ValueError("cond_sample_rate applies to a raw-wave cond [1, t]; this cond is a mel spectrogram")
        cond = cond.to(dev).float()
        batch, cond_seq_len = cond.shape[:2]
        if edit_mask is not None:
            if not isinstance(edit_mask, torch.Tensor) or edit_mask.dtype != torch.bool:
                raise ValueError(f"edit_mask must be a bool tensor, got {getattr(edit_mask, 'dtype', type(edit_mask))}")
            if tuple(edit_mask.shape) != (batch, cond_seq_len):
                raise ValueError(f"edit_mask must have shape [batch, conditioning frames] = {(batch, cond_seq_len)}, "
                                 f"got {tuple(edit_mask.shape)}")
            edit_mask = edit_mask.detach().cpu()
        if not exists(lens):
            lens = torch.full((batch,), cond_seq_len, dtype=torch.float32)
        lens = lens.detach().cpu().float()

        # text (cfm.py:294-303)
        if isinstance(text, list):
            if exists(self._vocab_char_map):
                text = list_str_to_idx(text, self._vocab_char_map)
            else:
                text = list_str_to_tensor(text)
            assert text.shape[0] == batch
        text = text.detach().cpu().to(torch.int32)
        _check_prefix_padding(text)
        text_lens = (text != -1).sum(dim=-1)
        lens = torch.maximum(text_lens.float(), lens)

        # duration (cfm.py:307-319)
        if duration is None and self._duration_predictor is not None:
            duration = self.predict_duration(cond, text.to(dev), speed)
        elif duration is None:
            raise ValueError("Duration must be provided or a duration predictor must be set.")
        cond_mask = lens_to_mask(lens)
        if edit_mask is not None:
            w = cond_mask.shape[-1]                                   # max(lens): past n_c when the text is longer
            em = edit_mask[:, :w]
            cond_mask = cond_mask & F.pad(em, (0, w - em.shape[-1]), value=True)
        if isinstance(duration, int):
            duration = torch.full((batch,), duration, dtype=torch.float32)
        duration = torch.as_tensor(duration).detach().cpu().float().reshape(-1)
        duration = torch.maximum(lens + 1, duration)
        duration = torch.clip(duration, 0, max_duration)
        N = int(duration.max().item())
        if pad_frames is not None:
            N = max(N, int(pad_frames))

        # pad cond / cond_mask to N; step_cond (cfm.py:321-331)
        cond = F.pad(cond, (0, 0, 0, N - cond_seq_len)) if N >= cond_seq_len else cond[:, :N]
        cond_mask = F.pad(cond_mask, (0, N - cond_mask.shape[-1]), value=False)[..., None].to(dev)
        step_cond = torch.where(cond_mask, cond, torch.zeros_like(cond))
        masked = batch > 1                                            # cfm.py:333-336
        seq_len = duration.to(torch.int32).to(dev) if masked else None

        # frame / text bucketing: buffers and graph of the bucket, the real N in a device scalar
        bucket = self.frame_bucket if frame_bucket is None else int(frame_bucket)
        NB = N
        if bucket > 0:
            NB = -(-N // bucket) * bucket
            tb = max(1, self.text_bucket)
            tcols = -(-max(text.shape[1], 1) // tb) * tb
            if tcols != text.shape[1]:
                text = F.pad(text, (0, tcols - text.shape[1]), value=-1)
        plan = self._plan(batch, NB, text.shape[1], steps, method, sway_sampling_coef, cfg_strength, masked,
                          return_trajectory, bucket > 0)
        self.last_plan = plan

        # noise (cfm.py:369-375): same seed for every element, drawn as (mel, dur) then transposed
        if y0 is None:
            ys = []
            for dur in duration.tolist():
                gen = torch.Generator().manual_seed(int(seed)) if exists(seed) else None
                ys.append(torch.randn(self.num_channels, int(dur), generator=gen))
            y0 = pad_sequence(ys, padding_value=0).permute(0, 2, 1)
        y0 = y0.to(dev).float()
        if NB != N:
            y0 = F.pad(y0, (0, 0, 0, NB - N))
            step_cond_in = F.pad(step_cond, (0, 0, 0, NB - N))
        else:
            step_cond_in = step_cond
        plan.session.set_inputs(text, step_cond_in, plan.tvals.to(dev), seq_len, frames_valid=N if bucket > 0 else None)
        plan.y.copy_(y0)

        plan.run(self, self.use_cuda_graph)

        # fresh tensors, like the reference: the plan's buffers are overwritten by the next call / graph replay
        if plan.trajectory is not None:
            trajectory = plan.trajectory[:, :, :N].clone()
            sampled = trajectory[-1]
        else:
            sampled = plan.y[:, :N].clone()
            trajectory = sampled[None]
        out = torch.where(cond_mask, cond, sampled)                  # cfm.py:395-397
        if exists(self._vocoder):
            out = self._vocoder(out)                                  # cfm.py:399-400
        return out, trajectory

    @classmethod
    def from_pretrained(cls, hf_model_name_or_path: str, convert_weights=None, quantization_bits=None, fp8=None,
                        fp8_attention=False, model_version="v1", vocoder=None):
        """fp8: None (bf16), "tensor" or "block" — the DiT's FP8 mode and its scaling (DESIGN.md section 8);
        fp8_attention (with fp8="block"): the attention on e4m3 Q, K and V as well; model_version: "v1", "v0"
        (F5TTS_Base checkpoints) or "e2" (E2TTS_Base, the UNetT backbone), see pretrained.from_pretrained; vocoder:
        None / "vocos" (default) or "bigvgan" (F5TTS_Base_bigvgan checkpoints, see pretrained.from_pretrained)."""
        from .pretrained import from_pretrained
        return from_pretrained(cls, hf_model_name_or_path, convert_weights, quantization_bits, fp8=fp8,
                               fp8_attention=fp8_attention, model_version=model_version, vocoder=vocoder)


CFM = F5TTS
