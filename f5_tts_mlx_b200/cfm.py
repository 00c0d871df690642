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
from .audio import MelSpec
from .dit import DiT, DitSession, _check_prefix_padding
from .utils import default, exists, lens_to_mask, list_str_to_idx, list_str_to_tensor, pad_sequence

METHODS = {"euler": 0, "midpoint": 1, "rk4": 2}


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


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
    DiT session buffers, ODE state buffers and the captured CUDA graph of precompute + ODE loop."""

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
        lib = _lib.load()
        tg = self.t_grid.numpy().ctypes.data_as(C.POINTER(C.c_float))
        _lib.check(lib.f5_ode_sample(
            C.byref(tr.packed.c_struct()), C.byref(self.session.c), tg, self.steps, METHODS[self.method],
            C.c_float(self.cfg_strength), C.c_void_p(self.y.data_ptr()),
            C.c_void_p(self.trajectory.data_ptr()) if self.trajectory is not None else None,
            C.c_void_p(self.scratch.data_ptr()) if self.scratch is not None else None, _stream()))

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
    ) -> Tuple[torch.Tensor, torch.Tensor]:
        """cfm.py:264-402.  Extensions (default-compatible): `y0` injects the initial noise
        (b, n, mel) — MLX's RNG stream cannot be reproduced, so seeded parity is defined on injected
        noise; `return_trajectory=False` skips keeping all `steps` states (then `trajectory` is the
        final state with a leading axis of 1); `pad_frames` pads the batch to at least that many frames — a shard
        of a ragged batch must use the GLOBAL maximum (parallel.global_frames) to reproduce the unsharded result,
        because the reference's padding leaks into GRN and the ODE on padded frames; `frame_bucket` (default
        self.frame_bucket) reuses one plan / CUDA graph for all lengths of a bucket, results unchanged."""
        dev = self.transformer.device
        if method not in METHODS:
            raise ValueError(f"Unknown method: {method}")

        # raw wave (cfm.py:283-286)
        if cond.ndim == 2:
            if cond.shape[0] != 1:
                raise ValueError("raw-wave conditioning must have batch 1 (cfm.py:284)")
            cond = self._mel_spec(cond[0].to(dev))
            assert cond.shape[-1] == self.num_channels
        cond = cond.to(dev).float()
        batch, cond_seq_len = cond.shape[:2]
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
    def from_pretrained(cls, hf_model_name_or_path: str, convert_weights=None, quantization_bits=None):
        from .pretrained import from_pretrained
        return from_pretrained(cls, hf_model_name_or_path, convert_weights, quantization_bits)


CFM = F5TTS
