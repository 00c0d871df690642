"""MelSpec / log_mel_spectrogram — host-side mirror of f5_tts_mlx/audio.py:162-230.

The arithmetic (zero-padded centred framing, periodic-Hann 1024-point real FFT, magnitude, HTK mel
filterbank, log(max(., 1e-5))) runs in the sm_90a kernel behind `f5_mel_forward`; this module only
builds the two constant tables (window, filterbank) and marshals pointers.
"""
from __future__ import annotations

import ctypes as C
import math
from functools import lru_cache

import numpy as np
import torch

from . import _lib


@lru_cache(maxsize=None)
def mel_filters(sample_rate: int, n_fft: int, n_mels: int) -> torch.Tensor:
    """HTK triangular filterbank, norm=None — audio.py:12-98 as called at audio.py:187-189.
    Returns (n_mels, n_fft // 2 + 1) fp32 (a constant table, host math)."""
    hz_to_mel = lambda f: 2595.0 * math.log10(1.0 + f / 700.0)
    n_freqs = n_fft // 2 + 1
    all_freqs = torch.linspace(0, sample_rate // 2, n_freqs, dtype=torch.float32)
    m_pts = torch.linspace(hz_to_mel(0.0), hz_to_mel(sample_rate / 2), n_mels + 2, dtype=torch.float32)
    f_pts = 700.0 * (10.0 ** (m_pts / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts[None, :] - all_freqs[:, None]
    down = (-slopes[:, :-2]) / f_diff[:-1]
    up = slopes[:, 2:] / f_diff[1:]
    return torch.clamp(torch.minimum(down, up), min=0.0).T.contiguous()


@lru_cache(maxsize=None)
def hanning(size: int) -> torch.Tensor:
    """Periodic Hann window, np.hanning(size + 1)[:-1] — audio.py:101-112."""
    return torch.from_numpy(np.hanning(size + 1)[:-1].astype(np.float32))


@lru_cache(maxsize=8)
def _tables(sample_rate: int, n_fft: int, n_mels: int, device: str):
    # the kernel wants the filterbank transposed: [n_fft//2+1, n_mels]
    return hanning(n_fft).to(device), mel_filters(sample_rate, n_fft, n_mels).T.contiguous().to(device)


def log_mel_spectrogram(audio: torch.Tensor, sample_rate: int = 24_000, n_mels: int = 100, n_fft: int = 1024,
                        hop_length: int = 256, padding: int = 0) -> torch.Tensor:
    """audio.py:162-210: audio [t] or [b, t] -> (b, t // hop_length, n_mels) fp32."""
    if not audio.is_cuda:
        raise _lib.F5Error("log_mel_spectrogram needs a CUDA tensor: there is no CPU path")
    if audio.ndim == 1:
        audio = audio[None]
    audio = audio.float().contiguous()
    if padding > 0:
        audio = torch.nn.functional.pad(audio, (0, padding))
    if n_fft != 1024:
        raise NotImplementedError("f5_mel_forward implements the path's n_fft = 1024")
    b, t = audio.shape
    # stft yields (t + 2*(n_fft//2) - n_fft + hop) // hop frames (audio.py:156) and the last one is
    # dropped (audio.py:203): t // hop frames remain
    frames = (t + hop_length) // hop_length - 1
    window, filters = _tables(sample_rate, n_fft, n_mels, str(audio.device))
    out = torch.empty(b, max(frames, 0), n_mels, device=audio.device, dtype=torch.float32)
    if frames > 0:
        _lib.check(_lib.load().f5_mel_forward(
            C.c_void_p(audio.data_ptr()), b, t, C.c_void_p(window.data_ptr()), C.c_void_p(filters.data_ptr()),
            n_mels, hop_length, C.c_void_p(out.data_ptr()), frames,
            C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return out


class MelSpec:
    """audio.py:213-230."""

    def __init__(self, sample_rate=24_000, n_fft=1024, hop_length=256, n_mels=100):
        self.sample_rate, self.n_fft, self.hop_length, self.n_mels = sample_rate, n_fft, hop_length, n_mels

    def __call__(self, audio: torch.Tensor, **kwargs) -> torch.Tensor:
        return log_mel_spectrogram(audio, sample_rate=self.sample_rate, n_mels=self.n_mels, n_fft=self.n_fft,
                                   hop_length=self.hop_length)
