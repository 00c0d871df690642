"""Speech editing restated test-side: the oracle's sample() (cfm.py:264-402) with the conditioning mask ANDed with an
edit mask, as upstream F5-TTS's CFM.sample(edit_mask=) does.  oracle/f5_oracle.py stays untouched; this composes its
prologue, noise, time grid and solvers.

    cond_mask = lens_to_mask(lens) & edit_mask      (columns past the mask's n_c count as True), then padded to N
    step_cond = where(cond_mask, cond, 0);  out = where(cond_mask, cond, trajectory[-1])

`forward(x, cond, text, time, drop_audio_cond, drop_text, mask, W, cfg, prec)` is the backbone: the oracle's DiT by
default, `functools.partial(v0_emul.dit_forward, pe_attn_head=1)` for v0, `unett_emul.unett_forward` for E2.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch
import torch.nn.functional as F

from oracle import f5_oracle as O


def sample(cond, text, duration, W, cfg, *, edit_mask: Optional[torch.Tensor] = None, lens=None,
           forward: Callable = O.dit_forward, steps: int = 8, method: str = "rk4", cfg_strength: float = 2.0,
           sway_sampling_coef: Optional[float] = -1.0, seed: Optional[int] = None, y0: Optional[torch.Tensor] = None,
           prec: O.Precision = O.FP32):
    prep = O.sample_prologue(cond, text, duration, W, lens=lens)
    cond_mask = prep.cond_mask                                             # (b, N, 1), False past max(lens)
    if edit_mask is not None:
        N = cond_mask.shape[1]
        em = edit_mask[:, :N]
        cond_mask = cond_mask & F.pad(em, (0, N - em.shape[1]), value=True)[..., None]
    step_cond = torch.where(cond_mask, prep.cond, torch.zeros_like(prep.cond))
    txt, mask = prep.text, prep.mask

    def fn(t, x):
        pred = forward(x, step_cond, txt, t, False, False, mask, W, cfg, prec)
        if cfg_strength < 1e-5:
            return pred
        null_pred = forward(x, step_cond, txt, t, True, True, mask, W, cfg, prec)
        return pred + (pred - null_pred) * cfg_strength

    if y0 is None:
        ys = []
        for dur in prep.duration.tolist():
            gen = torch.Generator().manual_seed(seed if seed is not None else 0)
            ys.append(torch.randn(100, int(dur), generator=gen))
        y0 = O.pad_sequence(ys, padding_value=0).permute(0, 2, 1)
    t = O.time_grid(steps, sway_sampling_coef)
    solver = {"euler": O.odeint_euler, "midpoint": O.odeint_midpoint, "rk4": O.odeint_rk4}[method]
    trajectory = solver(fn, y0.float(), t)
    return torch.where(cond_mask, prep.cond, trajectory[-1]), trajectory
