"""Regenerates the golden fixtures in this directory (run in the build container, where
/root/reference exists; the GPU box never runs this).

The reference ships no golden vectors and its runtime (MLX) is not installable here, so these are
outputs of the CPU oracle (oracle/f5_oracle.py) under fixed seeds — a regression pin for the oracle
and a transportable target for the CUDA path — plus one real-audio input taken from the
reference's only fixture (tests/test_en_1_ref_short.wav, first second, int16).
"""
import os, sys, wave
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import f5_oracle as O                                    # noqa: E402
from f5_tts_mlx_b200.weights import GATE_CONFIG, VocosConfig, random_dit_weights, random_vocos_weights  # noqa: E402

torch.manual_seed(0)
torch.set_num_threads(8)

# (a) real audio -> log-mel
wav = "/root/reference/tests/test_en_1_ref_short.wav"
with wave.open(wav, "rb") as f:
    assert f.getframerate() == 24000 and f.getnchannels() == 1 and f.getsampwidth() == 2
    pcm = np.frombuffer(f.readframes(f.getnframes()), dtype=np.int16)
full_frames = O.log_mel_spectrogram(torch.from_numpy(pcm.astype(np.float32) / 32768.0)).shape[1]
pcm1 = pcm[24000:48000].copy()                                        # 1 s from the middle of the clip
mel1 = O.log_mel_spectrogram(torch.from_numpy(pcm1.astype(np.float32) / 32768.0))[0].numpy()
np.savez_compressed(os.path.join(HERE, "mel_fixture.npz"), pcm=pcm1, mel=mel1.astype(np.float32),
                    full_clip_samples=np.int64(pcm.size), full_clip_frames=np.int64(full_frames))

cfg = GATE_CONFIG
ocfg = O.DiTConfig(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult, text_num_embeds=cfg.text_num_embeds,
                   text_dim=cfg.text_dim, conv_layers=cfg.conv_layers)
W = random_dit_weights(cfg, seed=1234)
g = torch.Generator().manual_seed(11)

# (b) one DiT forward (batch 2, ragged, masked)
B, N, nt = 2, 64, 20
x = torch.randn(B, N, 100, generator=g); cond = torch.randn(B, N, 100, generator=g)
text = torch.randint(0, 2545, (B, nt), generator=g, dtype=torch.int32); text[1, 13:] = -1
lens = torch.tensor([64, 50]); mask = torch.arange(N)[None, :] < lens[:, None]
t = torch.tensor(0.4321)
out = O.dit_forward(x, cond, text, t, False, False, mask, W, ocfg)
out_drop = O.dit_forward(x, cond, text, t, True, True, mask, W, ocfg)
np.savez_compressed(os.path.join(HERE, "dit_gate_forward.npz"), x=x.numpy(), cond=cond.numpy(), text=text.numpy(),
                    lens=lens.numpy(), t=t.numpy(), out=out.numpy(), out_drop=out_drop.numpy(), weight_seed=1234)

# (c) sample(): euler, 4 grid points, CFG 2, sway -1, injected noise; and midpoint without CFG
N, nref = 96, 40
cond = (torch.randn(1, nref, 100, generator=g) * 2.24 - 1.27).clamp(-11.51, 5)
text = torch.randint(0, 2545, (1, 24), generator=g, dtype=torch.int32)
y0 = torch.randn(1, 100, N, generator=g).permute(0, 2, 1).contiguous()
o1, tr1 = O.sample(cond, text, N, W, ocfg, steps=4, method="euler", cfg_strength=2.0, sway_sampling_coef=-1.0, y0=y0)
o2, tr2 = O.sample(cond, text, N, W, ocfg, steps=3, method="midpoint", cfg_strength=0.0, sway_sampling_coef=None, y0=y0)
o3, tr3 = O.sample(cond, text, N, W, ocfg, steps=3, method="rk4", cfg_strength=2.0, sway_sampling_coef=-1.0, y0=y0)
np.savez_compressed(os.path.join(HERE, "sample_gate.npz"), cond=cond.numpy(), text=text.numpy(), y0=y0.numpy(), duration=N,
                    euler_out=o1.numpy(), euler_traj_last=tr1[-1].numpy(), midpoint_nocfg_out=o2.numpy(), rk4_out=o3.numpy(),
                    weight_seed=1234)

# (d) schedule known answers
kat = {}
for steps in (2, 8, 32):
    for sway in (None, -1.0):
        kat[f"t_{steps}_{'none' if sway is None else 'm1'}"] = O.time_grid(steps, sway).numpy()
np.savez_compressed(os.path.join(HERE, "schedule_kat.npz"), **kat)

# (e) Vocos
vw = random_vocos_weights(VocosConfig(), seed=4321)
mel = (torch.randn(1, 12, 100, generator=g) * 2.24 - 1.27).clamp(-11.5, 5)
w1 = O.vocos_decode(mel, vw, O.VocosConfig())
w2 = O.vocos_decode(mel, vw, O.VocosConfig(istft_norm="window_sq", istft_trim=True))
np.savez_compressed(os.path.join(HERE, "vocos_small.npz"), mel=mel.numpy(), wave_window=w1.numpy(), wave_window_sq_trim=w2.numpy(),
                    weight_seed=4321)
for f in sorted(os.listdir(HERE)):
    print(f, os.path.getsize(os.path.join(HERE, f)))

# (f) DurationPredictor
from f5_tts_mlx_b200.weights import random_duration_weights  # noqa: E402
dW = random_duration_weights(seed=777)
dWo = {"duration." + k: v for k, v in dW.items()}
gd = torch.Generator().manual_seed(21)
mel = (torch.randn(2, 90, 100, generator=gd) * 2.24 - 1.27)
text = torch.randint(0, 2545, (2, 30), generator=gd, dtype=torch.int32); text[1, 18:] = -1
lens = torch.tensor([90, 61])
sec = O.duration_predictor(mel, text, dWo, O.DurationConfig(), lens=lens)
np.savez_compressed(os.path.join(HERE, "duration_small.npz"), mel=mel.numpy(), text=text.numpy(), lens=lens.numpy(),
                    seconds=sec.numpy(), weight_seed=777)
print("duration", sec)

# (g) per-operator input/output pairs on a small DiT (dim 128, 2 heads, 1 block)
from f5_tts_mlx_b200.weights import DiTConfig as PkgDiTConfig                     # noqa: E402
tiny = PkgDiTConfig(dim=128, depth=1, heads=2, ff_mult=2, text_dim=64, conv_layers=1, text_num_embeds=50)
tcfg = O.DiTConfig(dim=128, depth=1, heads=2, ff_mult=2, text_num_embeds=50, text_dim=64, conv_layers=1)
Wt = random_dit_weights(tiny, seed=77)
g = torch.Generator().manual_seed(5)
B, N = 2, 40
x = torch.randn(B, N, 128, generator=g)
t_emb = O.timestep_embedding(torch.tensor([0.25, 0.9]), Wt)
mask = torch.arange(N)[None, :] < torch.tensor([40, 23])[:, None]
rope = O.rotary_freqs(N)
text = torch.randint(0, 50, (B, 12), generator=g, dtype=torch.int32); text[1, 7:] = -1
xt = torch.randn(B, N, 64, generator=g)
pairs = dict(
    x=x.numpy(), text=text.numpy(), xt=xt.numpy(), weight_seed=77,
    time_embed=t_emb.numpy(),
    grn=O.grn(torch.randn(B, N, 128, generator=torch.Generator().manual_seed(6)),
              Wt["transformer.text_embed.text_blocks.layers.0.grn.gamma"],
              Wt["transformer.text_embed.text_blocks.layers.0.grn.beta"]).numpy(),
    convnext=O.convnext_v2_block(xt, Wt, "transformer.text_embed.text_blocks.layers.0.").numpy(),
    text_embed=O.text_embedding(text, N, False, Wt, tcfg).numpy(),
    text_embed_drop=O.text_embedding(text, N, True, Wt, tcfg).numpy(),
    conv_pos=O.conv_position_embedding(x, Wt).numpy(),
    attention=O.attention(x, mask, rope, Wt, "transformer.transformer_blocks.0.attn.", 2).numpy(),
    attention_nomask=O.attention(x, None, rope, Wt, "transformer.transformer_blocks.0.attn.", 2).numpy(),
    dit_block=O.dit_block(x, t_emb, mask, rope, Wt, 0, tcfg).numpy(),
    rope_q=O.apply_rotary_pos_emb(x[:, None, :, :64], rope).numpy(),
)
np.savez_compressed(os.path.join(HERE, "ops_small.npz"), **pairs)
print("wrote", sorted(f for f in os.listdir(HERE) if f.endswith(".npz")))
