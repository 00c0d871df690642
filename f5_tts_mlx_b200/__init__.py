"""f5_tts_mlx_b200 — H100 (sm_90a) implementation of the f5-tts-mlx sampling hot path.

Same public surface as the reference package for that path (`from f5_tts_mlx import F5TTS`,
f5_tts_mlx/__init__.py:1): F5TTS (alias CFM), DiT, MelSpec, generate().  Importing this package
does not need a GPU; every compute call does (there is no CPU fallback).
"""
from .weights import BASE_CONFIG, GATE_CONFIG, DiTConfig, VocosConfig  # noqa: F401
from .dit import DiT  # noqa: F401
from .audio import MelSpec, log_mel_spectrogram  # noqa: F401
from .cfm import CFM, F5TTS, odeint_euler, odeint_midpoint, odeint_rk4  # noqa: F401

__version__ = "0.1.0"
