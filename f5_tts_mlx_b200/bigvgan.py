"""BigVGAN v2 vocoder and its mel front-end — what upstream F5-TTS runs for F5TTS_Base_bigvgan checkpoints
(`--vocoder_name bigvgan`, NVIDIA's bigvgan_v2_24khz_100band_256x).

The arithmetic runs in the sm_90a kernels behind `f5_bigvgan_decode` (implicit-conv wgmma GEMMs, the anti-aliased
Snake / SnakeBeta kernel, conv_post) and `f5_mel_forward_bigvgan`; this module reads the checkpoint, folds the weight
norm, packs the weights into the layouts those kernels take (include/f5_b200.h) and builds the constant tables.

There is no BigVGAN source here: the definition followed is the one written out in DESIGN.md section 5 (and restated
by tests/bigvgan_emul.py).  No trained BigVGAN checkpoint was available when this was written, so parity with one rests
on that restatement.
"""
from __future__ import annotations

import ctypes as C
import json
import math
from dataclasses import dataclass
from functools import lru_cache
from pathlib import Path
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import _lib
from .audio import hanning

MAX_UPS = 8        # F5_BIGVGAN_MAX_UPS
MAX_KERNELS = 4    # F5_BIGVGAN_MAX_KERNELS
ACTIVATIONS = ("snake", "snakebeta")


@dataclass(frozen=True)
class BigVGANConfig:
    """The generator hyperparameters of a BigVGAN config.json; the defaults are bigvgan_v2_24khz_100band_256x."""
    num_mels: int = 100
    upsample_rates: Tuple[int, ...] = (4, 4, 2, 2, 2, 2)
    upsample_kernel_sizes: Tuple[int, ...] = (8, 8, 4, 4, 4, 4)
    upsample_initial_channel: int = 1536
    resblock: str = "1"
    resblock_kernel_sizes: Tuple[int, ...] = (3, 7, 11)
    resblock_dilation_sizes: Tuple[Tuple[int, ...], ...] = ((1, 3, 5), (1, 3, 5), (1, 3, 5))
    activation: str = "snakebeta"
    snake_logscale: bool = True
    use_tanh_at_final: bool = False
    use_bias_at_final: bool = False

    @classmethod
    def from_dict(cls, d: dict) -> "BigVGANConfig":
        try:
            cfg = cls(num_mels=int(d["num_mels"]), upsample_rates=tuple(int(u) for u in d["upsample_rates"]),
                      upsample_kernel_sizes=tuple(int(k) for k in d["upsample_kernel_sizes"]),
                      upsample_initial_channel=int(d["upsample_initial_channel"]), resblock=str(d["resblock"]),
                      resblock_kernel_sizes=tuple(int(k) for k in d["resblock_kernel_sizes"]),
                      resblock_dilation_sizes=tuple(tuple(int(x) for x in ds) for ds in d["resblock_dilation_sizes"]),
                      activation=str(d["activation"]), snake_logscale=bool(d["snake_logscale"]),
                      use_tanh_at_final=bool(d.get("use_tanh_at_final", True)),
                      use_bias_at_final=bool(d.get("use_bias_at_final", True)))
        except KeyError as e:
            raise ValueError(f"BigVGAN config.json lacks {e.args[0]!r}") from None
        cfg.validate()
        return cfg

    @classmethod
    def from_json(cls, path) -> "BigVGANConfig":
        return cls.from_dict(json.loads(Path(path).read_text()))

    @property
    def hop_length(self) -> int:
        return math.prod(self.upsample_rates)

    def stage_channels(self) -> list:
        """Output channels of each upsampling stage."""
        return [self.upsample_initial_channel >> (i + 1) for i in range(len(self.upsample_rates))]

    def validate(self) -> None:
        """ValueError for anything f5_bigvgan_decode does not build."""
        if self.resblock != "1":
            raise ValueError(f"BigVGAN resblock {self.resblock!r} is not supported (AMPBlock1, resblock \"1\", only)")
        if self.activation not in ACTIVATIONS:
            raise ValueError(f"BigVGAN activation {self.activation!r} is not one of {ACTIVATIONS}")
        if not 1 <= self.num_mels <= 128:
            raise ValueError(f"num_mels={self.num_mels} not in [1, 128]")
        nu, nk = len(self.upsample_rates), len(self.resblock_kernel_sizes)
        if len(self.upsample_kernel_sizes) != nu or not 1 <= nu <= MAX_UPS:
            raise ValueError(f"{nu} upsample rates with {len(self.upsample_kernel_sizes)} kernels (at most {MAX_UPS})")
        if not 1 <= nk <= MAX_KERNELS or len(self.resblock_dilation_sizes) != nk:
            raise ValueError(f"{nk} resblock kernels with {len(self.resblock_dilation_sizes)} dilation lists "
                             f"(at most {MAX_KERNELS})")
        for k, ds in zip(self.resblock_kernel_sizes, self.resblock_dilation_sizes):
            if k < 1 or k % 2 == 0 or len(ds) != 3 or min(ds) < 1:
                raise ValueError(f"resblock kernel {k} with dilations {ds}: needs an odd kernel and three dilations >= 1")
        for u, k in zip(self.upsample_rates, self.upsample_kernel_sizes):
            if u < 1 or k < u or (k - u) % 2:
                raise ValueError(f"upsampling (kernel {k}, stride {u}) is not a length-u polyphase convolution: needs "
                                 "k >= u and k - u even")
        c = self.upsample_initial_channel
        for i in range(nu):
            if c % 16:
                raise ValueError(f"stage {i} has {c} input channels: a multiple of 16 is needed")
            c //= 2


# ---------------------------------------------------------------- constant tables and weight transforms
def hz_to_mel_slaney(f):
    f = np.asarray(f, dtype=np.float64)
    logstep = math.log(6.4) / 27.0
    return np.where(f >= 1000.0, 15.0 + np.log(np.maximum(f, 1e-300) / 1000.0) / logstep, f / (200.0 / 3.0))


def mel_to_hz_slaney(m):
    m = np.asarray(m, dtype=np.float64)
    logstep = math.log(6.4) / 27.0
    return np.where(m >= 15.0, 1000.0 * np.exp(logstep * (m - 15.0)), m * (200.0 / 3.0))


def slaney_filterbank_f64(sample_rate: int = 24000, n_fft: int = 1024, n_mels: int = 100) -> np.ndarray:
    """librosa.filters.mel(sr, n_fft, n_mels, fmin=0, fmax=None) (Slaney scale, Slaney area norm) in float64:
    (n_mels, n_fft // 2 + 1)."""
    fmax = sample_rate / 2.0
    mel_f = mel_to_hz_slaney(np.linspace(hz_to_mel_slaney(0.0), hz_to_mel_slaney(fmax), n_mels + 2))
    fft_f = np.linspace(0.0, fmax, n_fft // 2 + 1)
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fft_f[None, :]
    lower = -ramps[:-2] / fdiff[:-1, None]
    upper = ramps[2:] / fdiff[1:, None]
    w = np.maximum(0.0, np.minimum(lower, upper))
    return w * (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]


@lru_cache(maxsize=None)
def slaney_filterbank(sample_rate: int = 24000, n_fft: int = 1024, n_mels: int = 100) -> torch.Tensor:
    """The fp32 filterbank: the float64 table rounded once."""
    return torch.from_numpy(slaney_filterbank_f64(sample_rate, n_fft, n_mels).astype(np.float32))


def kaiser_sinc_filter1d(cutoff: float = 0.25, half_width: float = 0.3, kernel_size: int = 12) -> torch.Tensor:
    """The anti-aliasing filter a BigVGAN Activation1d is built with (float64, rounded once to fp32): a Kaiser-windowed
    sinc, normalised to a sum of 1."""
    half = kernel_size // 2
    a = 2.285 * (half - 1) * math.pi * (4 * half_width) + 7.95
    beta = 0.1102 * (a - 8.7) if a > 50 else (0.5842 * (a - 21) ** 0.4 + 0.07886 * (a - 21) if a >= 21 else 0.0)
    window = torch.kaiser_window(kernel_size, beta=beta, periodic=False, dtype=torch.float64)
    time = torch.arange(-half, half, dtype=torch.float64) + 0.5 if kernel_size % 2 == 0 else \
        torch.arange(kernel_size, dtype=torch.float64) - half
    h = 2 * cutoff * window * torch.special.sinc(2 * cutoff * time)
    return (h / h.sum()).float()


def fold_weight_norm(g: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """w = g * v / ||v||, the norm over every dimension but dim 0 of the stored tensor (fp32)."""
    v = v.float()
    norm = v.reshape(v.shape[0], -1).norm(dim=1).reshape([v.shape[0]] + [1] * (v.dim() - 1))
    return g.float() * v / norm


def conv_weight(sd: Dict[str, torch.Tensor], prefix: str) -> torch.Tensor:
    """The folded weight of a checkpoint convolution: `.weight`, or `.weight_g` / `.weight_v`."""
    if prefix + ".weight" in sd:
        return sd[prefix + ".weight"].float()
    try:
        return fold_weight_norm(sd[prefix + ".weight_g"], sd[prefix + ".weight_v"])
    except KeyError:
        raise ValueError(f"BigVGAN checkpoint has no {prefix}.weight or {prefix}.weight_g / weight_v") from None


def polyphase_taps(k: int, u: int) -> Tuple[int, int]:
    """(taps, pad) of ConvTranspose1d(kernel k, stride u, padding (k - u) // 2) as a conv over the input frames."""
    p = (k - u) // 2
    dmax = max((q + p) // u for q in range(u))
    dmin = min(-((k - 1 - q - p) // u) for q in range(u))
    return dmax - dmin + 1, dmax


def pack_polyphase(w: torch.Tensor, u: int) -> Tuple[torch.Tensor, int, int]:
    """ConvTranspose1d weight (C_in, C_out, k) -> (W [u * C_out, taps, C_in], taps, pad): output frame n u + q, channel
    c_out, is row (q, c_out) of the conv with tap t reading input frame n + t - pad."""
    cin, cout, k = w.shape
    p = (k - u) // 2
    taps, pad = polyphase_taps(k, u)
    out = torch.zeros(u, cout, taps, cin, dtype=w.dtype)
    for q in range(u):
        for t in range(taps):
            j = (pad - t) * u + q + p
            if 0 <= j < k:
                out[q, :, t, :] = w[:, :, j].t()
    return out.reshape(u * cout, taps, cin), taps, pad


def _act_tables(sd, prefix, cfg: BigVGANConfig) -> Dict[str, torch.Tensor]:
    f = (lambda t: torch.exp(t.double()).float()) if cfg.snake_logscale else (lambda t: t.float())
    out = {"alpha": f(sd[prefix + ".act.alpha"]).reshape(-1),
           "h_up": sd[prefix + ".upsample.filter"].float().reshape(-1),
           "h_down": sd[prefix + ".downsample.lowpass.filter"].float().reshape(-1)}
    if cfg.activation == "snakebeta":
        out["beta"] = f(sd[prefix + ".act.beta"]).reshape(-1)
    if out["h_up"].numel() != 12 or out["h_down"].numel() != 12:
        raise ValueError(f"{prefix}: the anti-aliasing filters must have 12 taps")
    return out


def _tap_major(w: torch.Tensor, kp: int) -> torch.Tensor:
    """(C_out, taps, C_in) -> bf16 [C_out, taps * kp], each tap's channels zero-padded to kp."""
    co, taps, ci = w.shape
    out = torch.zeros(co, taps, kp)
    out[:, :, :ci] = w
    return out.reshape(co, taps * kp).bfloat16()


def pack_bigvgan(cfg: BigVGANConfig, sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Checkpoint state dict -> the CPU tensors f5_bigvgan_decode reads (names as in f5_bigvgan_weights)."""
    cfg.validate()
    P: Dict[str, torch.Tensor] = {}
    kp = lambda c: -(-c // 64) * 64
    w = conv_weight(sd, "conv_pre")                                   # (C0, num_mels, 7)
    if tuple(w.shape) != (cfg.upsample_initial_channel, cfg.num_mels, 7):
        raise ValueError(f"conv_pre weight {tuple(w.shape)} does not match the config")
    P["conv_pre_w"] = _tap_major(w.permute(0, 2, 1), 128)
    P["conv_pre_b"] = sd["conv_pre.bias"].float()
    nk = len(cfg.resblock_kernel_sizes)
    c = cfg.upsample_initial_channel
    for i, (u, k) in enumerate(zip(cfg.upsample_rates, cfg.upsample_kernel_sizes)):
        wt = conv_weight(sd, f"ups.{i}.0")                            # (C_in, C_out, k)
        if tuple(wt.shape) != (c, c // 2, k):
            raise ValueError(f"ups.{i}.0 weight {tuple(wt.shape)} does not match the config")
        pw, taps, pad = pack_polyphase(wt, u)
        P[f"up{i}_w"] = _tap_major(pw, kp(c))
        P[f"up{i}_b"] = sd[f"ups.{i}.0.bias"].float().repeat(u)
        P[f"up{i}_taps"], P[f"up{i}_pad"] = torch.tensor(taps), torch.tensor(pad)
        c //= 2
        for j, (kr, ds) in enumerate(zip(cfg.resblock_kernel_sizes, cfg.resblock_dilation_sizes)):
            n = i * nk + j
            for m in range(3):
                for s in ("convs1", "convs2"):
                    cw = conv_weight(sd, f"resblocks.{n}.{s}.{m}")     # (C, C, k)
                    if tuple(cw.shape) != (c, c, kr):
                        raise ValueError(f"resblocks.{n}.{s}.{m} weight {tuple(cw.shape)} does not match the config")
                    P[f"rb{n}.{s}.{m}_w"] = _tap_major(cw.permute(0, 2, 1), kp(c))
                    P[f"rb{n}.{s}.{m}_b"] = sd[f"resblocks.{n}.{s}.{m}.bias"].float()
            for a in range(6):
                for key, t in _act_tables(sd, f"resblocks.{n}.activations.{a}", cfg).items():
                    P[f"rb{n}.act{a}.{key}"] = t
    for key, t in _act_tables(sd, "activation_post", cfg).items():
        P[f"post.{key}"] = t
    w = conv_weight(sd, "conv_post")                                  # (1, C_last, 7)
    P["conv_post_w"] = w[0].t().contiguous()                          # [7, C_last]
    if cfg.use_bias_at_final:
        P["conv_post_b"] = sd["conv_post.bias"].float().reshape(1)
    return P


def random_bigvgan_weights(cfg: BigVGANConfig = BigVGANConfig(), seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded random generator weights in the checkpoint's key layout (weight-normed convolutions, stored Snake
    parameters, the Kaiser-sinc filters a fresh generator writes).  Gains keep the activations of order one."""
    cfg.validate()
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}

    def wn(prefix, shape, gain, bias=True):
        sd[prefix + ".weight_v"] = torch.randn(*shape, generator=g)
        sd[prefix + ".weight_g"] = gain * (1 + 0.1 * torch.randn(shape[0], 1, 1, generator=g))
        if bias:
            sd[prefix + ".bias"] = 0.02 * torch.randn(shape[1] if prefix.startswith("ups") else shape[0], generator=g)

    h = kaiser_sinc_filter1d().reshape(1, 1, 12)

    def act(prefix, ch):
        sd[prefix + ".act.alpha"] = 0.2 * torch.randn(ch, generator=g) + (0.0 if cfg.snake_logscale else 1.0)
        if cfg.activation == "snakebeta":
            sd[prefix + ".act.beta"] = 0.2 * torch.randn(ch, generator=g) + (0.0 if cfg.snake_logscale else 1.0)
        sd[prefix + ".upsample.filter"] = h.clone()
        sd[prefix + ".downsample.lowpass.filter"] = h.clone()

    wn("conv_pre", (cfg.upsample_initial_channel, cfg.num_mels, 7), 1.0)
    c = cfg.upsample_initial_channel
    nk = len(cfg.resblock_kernel_sizes)
    for i, (u, k) in enumerate(zip(cfg.upsample_rates, cfg.upsample_kernel_sizes)):
        wn(f"ups.{i}.0", (c, c // 2, k), math.sqrt(u / 2))
        c //= 2
        for j, kr in enumerate(cfg.resblock_kernel_sizes):
            n = i * nk + j
            for m in range(3):
                wn(f"resblocks.{n}.convs1.{m}", (c, c, kr), 1.0)
                wn(f"resblocks.{n}.convs2.{m}", (c, c, kr), 0.3)
            for a in range(6):
                act(f"resblocks.{n}.activations.{a}", c)
    act("activation_post", c)
    wn("conv_post", (1, c, 7), 0.1, bias=cfg.use_bias_at_final)
    return sd


def load_checkpoint(directory) -> Tuple[BigVGANConfig, Dict[str, torch.Tensor]]:
    """config.json and bigvgan_generator.pt ({"generator": state_dict}) of a BigVGAN directory."""
    d = Path(directory)
    cfg = BigVGANConfig.from_json(d / "config.json")
    ck = torch.load(str(d / "bigvgan_generator.pt"), map_location="cpu", weights_only=True)
    return cfg, ck["generator"] if "generator" in ck else ck


# ---------------------------------------------------------------- C ABI mirrors
class BigVGANActC(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("alpha", "beta", "h_up", "h_down")]


class BigVGANAmpWeightsC(C.Structure):
    _fields_ = [("kernel", C.c_int32), ("dilation", C.c_int32 * 3),
                ("conv1_w", C.c_void_p * 3), ("conv1_b", C.c_void_p * 3),
                ("conv2_w", C.c_void_p * 3), ("conv2_b", C.c_void_p * 3),
                ("act", BigVGANActC * 6)]


class BigVGANWeightsC(C.Structure):
    _fields_ = [("num_mels", C.c_int32), ("num_upsamples", C.c_int32), ("num_kernels", C.c_int32),
                ("channels0", C.c_int32), ("use_tanh_at_final", C.c_int32), ("reserved", C.c_int32 * 3),
                ("up_rate", C.c_int32 * MAX_UPS), ("up_taps", C.c_int32 * MAX_UPS), ("up_pad", C.c_int32 * MAX_UPS),
                ("conv_pre_w", C.c_void_p), ("conv_pre_b", C.c_void_p),
                ("up_w", C.c_void_p * MAX_UPS), ("up_b", C.c_void_p * MAX_UPS),
                ("blocks", C.POINTER(BigVGANAmpWeightsC)),
                ("act_post", BigVGANActC),
                ("conv_post_w", C.c_void_p), ("conv_post_b", C.c_void_p)]


class BigVGANBuffersC(C.Structure):
    _fields_ = [("batch", C.c_int32), ("frames", C.c_int32), ("reserved", C.c_int32 * 2),
                ("stage_elems", C.c_int64),
                ("mel_bf16", C.c_void_p), ("a_bf16", C.c_void_p), ("x_up", C.c_void_p), ("t", C.c_void_p),
                ("xk", C.c_void_p)]


def act_struct(tabs: Dict[str, torch.Tensor]) -> BigVGANActC:
    a = BigVGANActC()
    for n in ("alpha", "beta", "h_up", "h_down"):
        setattr(a, n, tabs[n].data_ptr() if n in tabs else None)
    return a


def stage_elems(cfg: BigVGANConfig, frames: int) -> int:
    """Per-utterance scratch size (f5_bigvgan_buffers.stage_elems)."""
    need, t = frames * cfg.upsample_initial_channel, frames
    for u, c in zip(cfg.upsample_rates, cfg.stage_channels()):
        t *= u
        need = max(need, t * c)
    return need


class BigVGAN:
    """`BigVGAN(config, device).load_weights(state_dict)`, then `.decode(mel)`: (b, n, num_mels) log-mel -> waveform
    (b, n * hop_length), 1-D for b = 1 like Vocos.decode.  Each utterance of a batch is computed exactly as alone."""

    def __init__(self, config: BigVGANConfig = BigVGANConfig(), device: str | torch.device = "cuda"):
        config.validate()
        self.config = config
        self.device = torch.device(device)
        self.packed: Optional[Dict[str, torch.Tensor]] = None
        self._t: Dict[str, torch.Tensor] = {}
        self._c: Optional[BigVGANWeightsC] = None
        self._bufs: Dict[tuple, tuple] = {}

    def load_weights(self, state_dict: Dict[str, torch.Tensor]) -> "BigVGAN":
        cfg = self.config
        self.packed = P = pack_bigvgan(cfg, state_dict)
        T = self._t = {k: v.to(self.device).contiguous() for k, v in P.items() if v.dim() > 0}
        nu, nk = len(cfg.upsample_rates), len(cfg.resblock_kernel_sizes)
        c = BigVGANWeightsC()
        c.num_mels, c.num_upsamples, c.num_kernels = cfg.num_mels, nu, nk
        c.channels0, c.use_tanh_at_final = cfg.upsample_initial_channel, int(cfg.use_tanh_at_final)
        c.conv_pre_w, c.conv_pre_b = T["conv_pre_w"].data_ptr(), T["conv_pre_b"].data_ptr()
        for i, u in enumerate(cfg.upsample_rates):
            c.up_rate[i], c.up_taps[i], c.up_pad[i] = u, int(P[f"up{i}_taps"]), int(P[f"up{i}_pad"])
            c.up_w[i], c.up_b[i] = T[f"up{i}_w"].data_ptr(), T[f"up{i}_b"].data_ptr()
        blks = (BigVGANAmpWeightsC * (nu * nk))()
        for i in range(nu):
            for j, (kr, ds) in enumerate(zip(cfg.resblock_kernel_sizes, cfg.resblock_dilation_sizes)):
                n = i * nk + j
                b = blks[n]
                b.kernel = kr
                for m in range(3):
                    b.dilation[m] = ds[m]
                    b.conv1_w[m], b.conv1_b[m] = T[f"rb{n}.convs1.{m}_w"].data_ptr(), T[f"rb{n}.convs1.{m}_b"].data_ptr()
                    b.conv2_w[m], b.conv2_b[m] = T[f"rb{n}.convs2.{m}_w"].data_ptr(), T[f"rb{n}.convs2.{m}_b"].data_ptr()
                for a in range(6):
                    b.act[a] = act_struct({k.split(".")[-1]: v for k, v in T.items() if k.startswith(f"rb{n}.act{a}.")})
        c.blocks = blks
        c.act_post = act_struct({k.split(".")[-1]: v for k, v in T.items() if k.startswith("post.")})
        c.conv_post_w = T["conv_post_w"].data_ptr()
        c.conv_post_b = T["conv_post_b"].data_ptr() if "conv_post_b" in T else None
        self._blks, self._c = blks, c
        return self

    def _buffers(self, batch: int, frames: int):
        key = (batch, frames)
        if key not in self._bufs:
            if len(self._bufs) >= 2:
                self._bufs.pop(next(iter(self._bufs)))
            cfg, dev = self.config, self.device
            se = stage_elems(cfg, frames)
            nk = len(cfg.resblock_kernel_sizes)
            t = dict(mel_bf16=torch.zeros(batch * frames, 128, dtype=torch.bfloat16, device=dev),
                     a_bf16=torch.empty(batch * se, dtype=torch.bfloat16, device=dev),
                     x_up=torch.empty(batch * se, device=dev), t=torch.empty(batch * se, device=dev),
                     xk=torch.empty(nk * batch * se, device=dev))
            c = BigVGANBuffersC()
            c.batch, c.frames, c.stage_elems = batch, frames, se
            for n, v in t.items():
                setattr(c, n, v.data_ptr())
            self._bufs[key] = (t, c)
        return self._bufs[key]

    def decode(self, mel: torch.Tensor) -> torch.Tensor:
        if self._c is None:
            raise RuntimeError("BigVGAN has no weights: call load_weights() first")
        if not mel.is_cuda:
            raise _lib.F5Error("BigVGAN.decode needs a CUDA tensor: there is no CPU path")
        if mel.ndim != 3 or mel.shape[-1] != self.config.num_mels:
            raise ValueError(f"BigVGAN.decode takes (b, n, {self.config.num_mels}), got {tuple(mel.shape)}")
        b, n, _ = mel.shape
        wave = torch.empty(b, n * self.config.hop_length, device=mel.device, dtype=torch.float32)
        if b * n > 0:
            _, c = self._buffers(b, n)
            mel = mel.float().contiguous()
            _lib.check(_lib.load().f5_bigvgan_decode(C.byref(self._c), C.byref(c), C.c_void_p(mel.data_ptr()),
                                                     C.c_void_p(wave.data_ptr()),
                                                     C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        return wave[0] if b == 1 else wave

    __call__ = decode


# ---------------------------------------------------------------- mel front-end
def bigvgan_frames(samples: int, n_fft: int = 1024, hop_length: int = 256) -> int:
    pad = (n_fft - hop_length) // 2
    if samples <= pad:
        raise ValueError(f"BigVGAN's mel reflect-pads {pad} samples and needs more than {pad}, got {samples}")
    return (samples + 2 * pad - n_fft) // hop_length + 1


@lru_cache(maxsize=8)
def _tables(sample_rate: int, n_fft: int, n_mels: int, device: str):
    return hanning(n_fft).to(device), slaney_filterbank(sample_rate, n_fft, n_mels).T.contiguous().to(device)


def bigvgan_mel_spectrogram(audio: torch.Tensor, sample_rate: int = 24_000, n_mels: int = 100, n_fft: int = 1024,
                            hop_length: int = 256) -> torch.Tensor:
    """Upstream F5-TTS get_bigvgan_mel_spectrogram: [t] or [b, t] -> (b, frames, n_mels) fp32 on the GPU
    (f5_mel_forward_bigvgan); frames = (t + 768 - 1024) // 256 + 1."""
    if not audio.is_cuda:
        raise _lib.F5Error("bigvgan_mel_spectrogram needs a CUDA tensor: there is no CPU path")
    if n_fft != 1024:
        raise NotImplementedError("f5_mel_forward_bigvgan implements n_fft = 1024")
    if audio.ndim == 1:
        audio = audio[None]
    audio = audio.float().contiguous()
    b, t = audio.shape
    frames = bigvgan_frames(t, n_fft, hop_length)
    window, filters = _tables(sample_rate, n_fft, n_mels, str(audio.device))
    out = torch.empty(b, frames, n_mels, device=audio.device, dtype=torch.float32)
    _lib.check(_lib.load().f5_mel_forward_bigvgan(
        C.c_void_p(audio.data_ptr()), b, t, C.c_void_p(window.data_ptr()), C.c_void_p(filters.data_ptr()),
        n_mels, hop_length, C.c_void_p(out.data_ptr()), frames, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return out


class BigVGANMelSpec:
    """The mel module of F5TTS_Base_bigvgan (F5TTS(mel_spec_module=BigVGANMelSpec()))."""

    def __init__(self, sample_rate=24_000, n_fft=1024, hop_length=256, n_mels=100):
        self.sample_rate, self.n_fft, self.hop_length, self.n_mels = sample_rate, n_fft, hop_length, n_mels

    def __call__(self, audio: torch.Tensor, **kwargs) -> torch.Tensor:
        return bigvgan_mel_spectrogram(audio, sample_rate=self.sample_rate, n_mels=self.n_mels, n_fft=self.n_fft,
                                       hop_length=self.hop_length)
