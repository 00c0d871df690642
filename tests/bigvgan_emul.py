"""BigVGAN v2 restated on the CPU in float64 with torch.nn.functional, from the definition in DESIGN.md section 5
(upstream F5-TTS get_bigvgan_mel_spectrogram and BigVGAN's generator, resblock "1"), plus an emulation with the GPU
path's rounding points.

`generator(mel, sd, cfg)` is the definition: weight norm folded in float64, every op in float64.
`generator(mel, sd, cfg, emulate=True)` rounds where f5_bigvgan_decode rounds: the folded weights to bf16 (after an fp32
fold, as the packing does), the Snake parameters to fp32, the mel and every GEMM operand (conv_pre output, activation
outputs, the resblock mean before the next ups) to bf16, every other stage output to fp32.  Arithmetic between those
points stays float64, so the emulation's distance from the definition is the drift the rounding points alone cause.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

F64 = torch.float64


# ---------------------------------------------------------------- Slaney filterbank (librosa.filters.mel)
def hz_to_mel(f: float) -> float:
    return f / (200.0 / 3.0) if f < 1000.0 else 15.0 + math.log(f / 1000.0) / (math.log(6.4) / 27.0)


def mel_to_hz(m: float) -> float:
    return m * (200.0 / 3.0) if m < 15.0 else 1000.0 * math.exp((math.log(6.4) / 27.0) * (m - 15.0))


def slaney_filterbank(sr: int = 24000, n_fft: int = 1024, n_mels: int = 100) -> np.ndarray:
    """The formula of the definition, element by element: (n_mels, n_fft // 2 + 1) float64."""
    top = hz_to_mel(sr / 2)
    mel_f = [mel_to_hz(top * i / (n_mels + 1)) for i in range(n_mels + 2)]
    nf = n_fft // 2 + 1
    fft_f = [sr / 2 * j / (nf - 1) for j in range(nf)]
    w = np.zeros((n_mels, nf))
    for i in range(n_mels):
        for j, f in enumerate(fft_f):
            lo = -(mel_f[i] - f) / (mel_f[i + 1] - mel_f[i])
            hi = (mel_f[i + 2] - f) / (mel_f[i + 2] - mel_f[i + 1])
            w[i, j] = max(0.0, min(lo, hi)) * 2.0 / (mel_f[i + 2] - mel_f[i])
    return w


def mel(wave: torch.Tensor, fb: np.ndarray, hop: int = 256, n_fft: int = 1024) -> torch.Tensor:
    """[b, t] -> (b, frames, n_mels) float64: reflect pad (n_fft - hop) / 2, non-centred frames, periodic Hann, DFT,
    sqrt(|X|^2 + 1e-9), filterbank, log(clamp(., 1e-5))."""
    x = wave.to(F64)
    pad = (n_fft - hop) // 2
    x = F.pad(x[:, None], (pad, pad), mode="reflect")[:, 0]
    frames = x.unfold(-1, n_fft, hop)                                     # (b, frames, n_fft)
    win = torch.hann_window(n_fft, periodic=True, dtype=F64)
    spec = torch.fft.rfft(frames * win, dim=-1)
    mag = torch.sqrt(spec.real ** 2 + spec.imag ** 2 + 1e-9)
    return torch.log(torch.clamp(mag @ torch.from_numpy(fb).T, min=1e-5))


# ---------------------------------------------------------------- generator
def fold(sd, prefix):
    if prefix + ".weight" in sd:
        return sd[prefix + ".weight"].to(F64)
    g, v = sd[prefix + ".weight_g"].to(F64), sd[prefix + ".weight_v"].to(F64)
    n = v.reshape(v.shape[0], -1).norm(dim=1).reshape([v.shape[0]] + [1] * (v.dim() - 1))
    return g * v / n


def fold_emul(sd, prefix):
    """fp32 fold (as bigvgan.conv_weight), rounded to bf16: the packed GEMM weights."""
    if prefix + ".weight" in sd:
        w = sd[prefix + ".weight"].float()
    else:
        g, v = sd[prefix + ".weight_g"].float(), sd[prefix + ".weight_v"].float()
        w = g * v / v.reshape(v.shape[0], -1).norm(dim=1).reshape([v.shape[0]] + [1] * (v.dim() - 1))
    return w


def activation1d(x, alpha, beta, h_up, h_down):
    """Activation1d(SnakeBeta / Snake) on (b, C, T) float64; beta None = Snake."""
    C = x.shape[1]
    hu = h_up.to(F64).reshape(1, 1, -1).expand(C, 1, -1)
    hd = h_down.to(F64).reshape(1, 1, -1).expand(C, 1, -1)
    y = F.pad(x, (5, 5), mode="replicate")
    y = 2 * F.conv_transpose1d(y, hu, stride=2, groups=C)[..., 15:-15]
    a = alpha.to(F64)[None, :, None]
    b = (beta if beta is not None else alpha).to(F64)[None, :, None]
    y = y + 1.0 / (b + 1e-9) * torch.sin(a * y) ** 2
    y = F.pad(y, (5, 6), mode="replicate")
    return F.conv1d(y, hd, stride=2, groups=C)


def act_params(sd, prefix, cfg, emulate):
    def f(t):
        v = torch.exp(t.to(F64)) if cfg.snake_logscale else t.to(F64)
        return v.float().to(F64) if emulate else v
    beta = f(sd[prefix + ".act.beta"]) if cfg.activation == "snakebeta" else None
    return (f(sd[prefix + ".act.alpha"]), beta, sd[prefix + ".upsample.filter"].reshape(-1),
            sd[prefix + ".downsample.lowpass.filter"].reshape(-1))


def generator(mel_in: torch.Tensor, sd, cfg, emulate: bool = False) -> torch.Tensor:
    """(b, n, num_mels) -> (b, n * hop) float64."""
    bf = (lambda t: t.to(torch.bfloat16).to(F64)) if emulate else (lambda t: t)
    f32 = (lambda t: t.float().to(F64)) if emulate else (lambda t: t)
    W = (lambda p: fold_emul(sd, p).to(torch.bfloat16).to(F64)) if emulate else (lambda p: fold(sd, p))
    B = lambda p: sd[p + ".bias"].to(F64) if p + ".bias" in sd else None
    act = lambda t, p: activation1d(t, *act_params(sd, p, cfg, emulate))
    x = bf(mel_in.to(F64)).transpose(1, 2)
    x = bf(F.conv1d(x, W("conv_pre"), B("conv_pre"), padding=3))
    nk = len(cfg.resblock_kernel_sizes)
    nu = len(cfg.upsample_rates)
    for i, (u, k) in enumerate(zip(cfg.upsample_rates, cfg.upsample_kernel_sizes)):
        x = f32(F.conv_transpose1d(x, W(f"ups.{i}.0"), B(f"ups.{i}.0"), stride=u, padding=(k - u) // 2))
        xs = []
        for j, (kr, ds) in enumerate(zip(cfg.resblock_kernel_sizes, cfg.resblock_dilation_sizes)):
            n, xj = i * nk + j, x
            for m, d in enumerate(ds):
                p = f"resblocks.{n}"
                t = bf(act(xj, f"{p}.activations.{2 * m}"))
                t = f32(F.conv1d(t, W(f"{p}.convs1.{m}"), B(f"{p}.convs1.{m}"), dilation=d, padding=(kr * d - d) // 2))
                t = bf(act(t, f"{p}.activations.{2 * m + 1}"))
                xj = f32(xj + F.conv1d(t, W(f"{p}.convs2.{m}"), B(f"{p}.convs2.{m}"), padding=(kr - 1) // 2))
            xs.append(xj)
        if emulate:                                 # the mean kernel: fp32 sum in order, one fp32 division
            s = xs[0].float()
            for xj in xs[1:]:
                s = s + xj.float()
            s = (s / float(nk)).to(F64)
            x = bf(s) if i + 1 < nu else s
        else:
            x = sum(xs) / nk
    x = f32(act(x, "activation_post"))
    x = F.conv1d(x, W("conv_post") if not emulate else fold_emul(sd, "conv_post").to(F64), B("conv_post"), padding=3)
    x = torch.tanh(x) if cfg.use_tanh_at_final else torch.clamp(x, -1, 1)
    return x[:, 0]
