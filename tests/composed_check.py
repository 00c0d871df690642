"""Row-wise checker for composed stages (DiT buffers, sample(), duration model, Vocos): pure torch, CPU or GPU.

A bug in how kernels are composed (a row offset at an utterance boundary, conv padding at the first or last frames,
the CFG null half, bucket rows) usually damages a few rows.  One relative L2 over the whole output dilutes that damage
below the bf16 noise, so these checks are made per row.

Inputs are shaped [branch, utterance, frame, ...]: `got` (the CUDA path), `ref` (the fp32 oracle) and `emu` (the
oracle with the CUDA path's rounding points).  The error of a row is ||got_row - ref_row|| divided by the RMS over the
utterance's rows of ||ref_row||, so rows where ref is near zero (padded rows, quiet frames) are measured on the
utterance's scale.  `assert_rows` passes when both hold:
  * the worst row error is at most `factor` x emu's worst row error (or below `floor`);
  * per (branch, utterance), rel L2 < min(max(factor x emu's rel L2, 2e-3), 2e-2): the global rule of
    test_gpu_parity.py, applied to each utterance and CFG branch.
A failure names the branch, utterance and frame; on success the worst ratio is returned.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Sequence

import torch


def _rows(t: torch.Tensor) -> torch.Tensor:
    assert t.dim() >= 3, "expected [branch, utterance, frame, ...]"
    return t.detach().double().cpu().reshape(t.shape[0], t.shape[1], t.shape[2], -1)


def row_errors(got: torch.Tensor, ref: torch.Tensor, lens: Optional[Sequence[int]] = None) -> torch.Tensor:
    """[branch, utterance, frame] errors ||got_row - ref_row|| / RMS_rows(||ref_row||).  `lens` (per utterance) limits
    each utterance to its first lens[u] frames: the scale is taken over those rows and the others get error 0."""
    g, r = _rows(got), _rows(ref)
    assert g.shape == r.shape, (tuple(got.shape), tuple(ref.shape))
    valid = torch.ones(r.shape[:3], dtype=torch.bool)
    if lens is not None:
        valid = (torch.arange(r.shape[2])[None, :] < torch.as_tensor(list(lens))[:, None])[None].expand_as(valid)
    rn2 = r.pow(2).sum(-1) * valid
    scale = (rn2.sum(-1) / valid.sum(-1).clamp_min(1)).sqrt()            # [branch, utterance]
    scale = torch.where(scale > 0, scale, torch.ones_like(scale))        # an all-zero utterance is measured absolutely
    return (g - r).norm(dim=-1) * valid / scale[..., None]


def _rel(a: torch.Tensor, b: torch.Tensor) -> float:
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


@dataclass
class RowReport:
    ratio: float          # worst row error / emu's worst row error
    worst: tuple          # (branch, utterance, frame) of the worst row
    err: float            # its error
    emu_err: float        # emu's worst row error
    rel_ratio: float      # worst per-(branch, utterance) rel L2 / its bound

    def __str__(self):
        b, u, n = self.worst
        return (f"worst row {self.ratio:.2f}x emu's (branch {b}, utterance {u}, frame {n}: {self.err:.2e} vs "
                f"{self.emu_err:.2e}); per-utterance rel at {self.rel_ratio:.2f} of its bound")


def assert_rows(got: torch.Tensor, ref: torch.Tensor, emu: torch.Tensor, *, factor: float = 3.0, floor: float = 1e-3,
                lens: Optional[Sequence[int]] = None, what: str = "") -> RowReport:
    g, r, e = _rows(got), _rows(ref), _rows(emu)
    assert torch.isfinite(g).all(), f"{what}: non-finite output"
    eg, ee = row_errors(g, r, lens), row_errors(e, r, lens)
    emu_worst = ee.max().item()
    k = int(eg.argmax())
    worst = tuple(int(i) for i in torch.unravel_index(torch.tensor(k), eg.shape))
    err = eg.flatten()[k].item()
    rep = RowReport(err / max(emu_worst, 1e-30), worst, err, emu_worst, 0.0)
    bound = max(factor * emu_worst, floor)
    assert err <= bound, f"{what}: row error {err:.3e} > {bound:.3e} = max({factor} x emu's worst row, {floor}); {rep}"
    if lens is not None:
        keep = (torch.arange(r.shape[2])[None, :] < torch.as_tensor(list(lens))[:, None])[None, :, :, None]
        g, r, e = g * keep, r * keep, e * keep
    for b in range(r.shape[0]):
        for u in range(r.shape[1]):
            rb = _rel(g[b, u], r[b, u])
            tol = min(max(factor * _rel(e[b, u], r[b, u]), 2e-3), 2e-2)
            rep.rel_ratio = max(rep.rel_ratio, rb / tol)
            assert rb < tol, f"{what}: branch {b}, utterance {u}: rel {rb:.3e} >= {tol:.3e}; {rep}"
    return rep


def exact_zero_rows(buf: torch.Tensor, valid_len, what: str = "") -> None:
    """buf [utterance, frame, ...]: every row at or beyond valid_len (int or per utterance) holds exactly zero."""
    t = buf.detach().cpu()
    t = t.reshape(t.shape[0], t.shape[1], -1)
    vl = torch.as_tensor(valid_len).reshape(-1).expand(t.shape[0])
    bad = (t != 0).any(-1) & (torch.arange(t.shape[1])[None, :] >= vl[:, None])
    if bad.any():
        u, n = (int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{what}: bucket row not zero: utterance {u}, frame {n} (valid_len {int(vl[u])}), "
                             f"max |value| {t[u, n].abs().max().item():.3e}")
