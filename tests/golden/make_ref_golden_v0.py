"""Fixture of the REFERENCE'S OWN CODE for unmasked text padding: DiT(text_mask_padding=False) (dit.py:182-229, 342-352).

Like make_ref_golden.py (see there): the unmodified reference sources are imported on top of tests/mlx_shim and run
with the repo's seeded synthetic weights, on the gate config (4 layers, 512 dims, 8 heads).  Writes ref_dit_v0.npz:
DiT.__call__ with drop_text False and True (and the CFG pass's drop of both), and a short Euler sample() with CFG.
tests/test_v0.py requires the oracle's mask_padding=False path, composed by tests/v0_emul.py, to match it to 2e-6
relative.  The reference rotates every attention head; the v0 rotation (first head only) is restated test-side in
tests/v0_emul.py and is not part of this fixture.  The fixture holds numbers only.

    python tests/golden/make_ref_golden_v0.py       # rewrites tests/golden/ref_dit_v0.npz, prints oracle deviations
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import mlx_shim as shim                                                  # noqa: E402
import v0_emul as V                                                      # noqa: E402
from f5_tts_mlx_b200.weights import GATE_CONFIG, random_dit_weights      # noqa: E402

torch.set_num_threads(8)
ref = shim.import_reference()
A = ref.mx.array


def a2n(a):
    return np.asarray(a)


def rel(a, b):
    a, b = torch.as_tensor(np.asarray(a)).double(), torch.as_tensor(np.asarray(b)).double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


cfg = GATE_CONFIG
W = random_dit_weights(cfg, seed=1234)
dit = ref.dit.DiT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult, mel_dim=cfg.mel_dim,
                  text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim, conv_layers=cfg.conv_layers,
                  text_mask_padding=False)
dit.load_weights([(k[len("transformer."):], A(v)) for k, v in W.items() if k.startswith("transformer.")])
ocfg = V.ocfg_v0(cfg)
report = {}

# DiT.__call__, batch 1: filler tokens inside the text row (pad -1) and rows past the text
g = torch.Generator().manual_seed(202)
N, nt = 80, 24
x = torch.randn(1, N, 100, generator=g)
cond = torch.randn(1, N, 100, generator=g)
text = torch.randint(0, 2545, (1, nt), generator=g, dtype=torch.int32)
text[0, 19:] = -1
tval = torch.tensor(0.4321)
outs = {}
for name, (dac, dt) in {"out": (False, False), "out_drop_text": (False, True), "out_drop": (True, True)}.items():
    outs[name] = a2n(dit(x=A(x), cond=A(cond), text=A(text), time=A(tval), drop_audio_cond=dac, drop_text=dt, mask=None))
    report[name] = rel(V.dit_forward(x, cond, text, tval, dac, dt, None, W, ocfg), outs[name])

# F5TTS.sample, Euler with CFG (the text-dropped pass runs on all-filler text)
f5 = ref.cfm.F5TTS(transformer=dit)
nref, Ns = 40, 96
scond = (torch.randn(1, nref, 100, generator=g) * 2.24 - 1.27).clamp(-11.51, 5)
stext = torch.randint(0, 2545, (1, 24), generator=g, dtype=torch.int32)
kw = dict(steps=4, method="euler", cfg_strength=2.0, sway_sampling_coef=-1.0, seed=7)
o, tr = f5.sample(A(scond), A(stext), Ns, **kw)
oo, otr = V.sample(scond, stext, Ns, W, ocfg, **kw)
report["sample_euler_cfg"], report["sample_euler_cfg_traj"] = rel(oo, a2n(o)), rel(otr, a2n(tr))

np.savez_compressed(os.path.join(HERE, "ref_dit_v0.npz"), x=x.numpy(), cond=cond.numpy(), text=text.numpy(),
                    t=tval.numpy(), **outs, scond=scond.numpy(), stext=stext.numpy(), duration=Ns,
                    sample_out=a2n(o), sample_traj=a2n(tr), weight_seed=1234)
for k, v in report.items():
    print(f"{k:28s} oracle rel {v:.3e}")
