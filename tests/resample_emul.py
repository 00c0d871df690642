"""Float64 restatement of the windowed-sinc resampler that `f5_resample_table` / `f5_resample` implement
(include/f5_b200.h): torchaudio.functional.resample at its defaults (sinc_interp_hann, lowpass_filter_width 6,
rolloff 0.99).  Written from the definition in the header, not from either implementation."""
from __future__ import annotations

import math

import numpy as np


def geometry(orig: int, new: int):
    """(O, N, w, taps, base) of a rate pair."""
    g = math.gcd(orig, new)
    O, N = orig // g, new // g
    base = min(O, N) * 0.99
    w = math.ceil(6 * O / base)
    return O, N, w, 2 * w + O, base


def table(orig: int, new: int) -> np.ndarray:
    """h[p][k], float64 [N, taps]."""
    O, N, w, taps, base = geometry(orig, new)
    k = np.arange(taps, dtype=np.float64)[None, :]
    p = np.arange(N, dtype=np.float64)[:, None]
    t = np.clip(((k - w) / O - p / N) * base, -6.0, 6.0)
    c = np.cos(np.pi * t / 12.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        s = np.where(t == 0.0, 1.0, np.sin(np.pi * t) / (np.pi * t))
    return s * c * c * base / O


def out_len(orig: int, new: int, length: int) -> int:
    O, N = geometry(orig, new)[:2]
    return -(-N * length // O)


def gather_index(orig: int, new: int, length: int, j: np.ndarray | None = None):
    """(phase, input index [J, taps], valid [J, taps]) of outputs j (default: all): x[(j // N) * O + k - w]."""
    O, N, w, taps, _ = geometry(orig, new)
    if j is None:
        j = np.arange(out_len(orig, new, length), dtype=np.int64)
    idx = (j // N * O - w)[:, None] + np.arange(taps, dtype=np.int64)[None, :]
    return j % N, idx, (idx >= 0) & (idx < length)


def _reduce(x: np.ndarray, orig: int, new: int, fn, chunk: int = 8192) -> np.ndarray:
    """fn(h[j % N][k] * x[...]) reduced over k for every output j, float64 [..., J] (x: [..., L]), in chunks of j."""
    x = np.asarray(x, dtype=np.float64)
    h = table(orig, new)
    L = x.shape[-1]
    J = out_len(orig, new, L)
    out = np.empty(x.shape[:-1] + (J,), dtype=np.float64)
    for j0 in range(0, J, chunk):
        p, idx, valid = gather_index(orig, new, L, np.arange(j0, min(J, j0 + chunk), dtype=np.int64))
        xs = np.where(valid, x[..., np.clip(idx, 0, L - 1)], 0.0)
        out[..., j0:j0 + chunk] = fn(h[p] * xs)
    return out


def resample(x: np.ndarray, orig: int, new: int) -> np.ndarray:
    """float64 resample of x [..., L] -> [..., ceil(N L / O)]; equal rates return x."""
    if orig == new:
        return np.asarray(x, dtype=np.float64)
    return _reduce(x, orig, new, lambda t: t.sum(axis=-1))


def error_bound(x: np.ndarray, orig: int, new: int) -> np.ndarray:
    """Per-output bound on |fp32 kernel - float64 resample| for fp32 input x: the table's fp32 rounding (2^-24
    relative per entry, at most 2^-24 sum |h x| in all) plus a chain of fp32 fused multiply-adds whose first product
    is rounded once and whose taps - 1 later sums are each rounded by at most 2^-24 of a partial sum no larger than
    sum |h x| (to first order): taps * 2^-24 * sum_k |h[p][k] x[...]| covers both."""
    taps = geometry(orig, new)[3]
    return taps * 2.0 ** -24 * _reduce(x, orig, new, lambda t: np.abs(t).sum(axis=-1))
