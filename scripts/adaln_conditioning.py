"""Measure the conditioning r = |row mean| / row std of the DiT's residual stream where each AdaLN LayerNorm reads it.

The fused AdaLN (DiT(fused_adaln=True), the default) rounds its GEMM operand x (1 + scale) before the row is centred,
so its rounding error is relative to |x| rather than to the row's spread: the fused path's error grows against the
separate LayerNorm's like sqrt(1 + r^2) (tests/adaln_emul.py; measured on the kernels by
tests/test_gpu_adaln_conditioning.py).  Whether it is worth centring the operand depends on r in real checkpoints.

For every evaluation time of the Euler solver (sway sampling, as sample() uses), the script runs the fp32 oracle forward
on the CPU and prints, per block and LayerNorm site (attn_norm, ff_norm, then norm_out), the 50th / 99th percentile and
maximum of r over the valid rows, and the fused / unfused error ratio that r predicts, sqrt(1 + mean r^2).  The inputs
are one synthetic utterance: noise as y0, a random mel prompt over the first third of the frames, random text.

    python scripts/adaln_conditioning.py                       # random-init base model (seed 1234)
    python scripts/adaln_conditioning.py --model /path/to/dir  # local checkpoint directory (model_v1.safetensors,
                                                               # vocab.txt), read as from_pretrained reads it
"""
from __future__ import annotations

import argparse
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from oracle import f5_oracle as O  # noqa: E402


def row_r(x: torch.Tensor) -> torch.Tensor:
    """r = |mean| / std (biased) of every row of x [B, N, D], as float64 [B N]."""
    xd = x.double().reshape(-1, x.shape[-1])
    return xd.mean(-1).abs() / xd.std(-1, unbiased=False)


def stream_conditioning(x, cond, text, t, W, cfg: O.DiTConfig, drop: bool = False):
    """[(site, r over the rows)] for every LayerNorm the DiT's residual stream enters at time t (fp32 oracle)."""
    tt = O.timestep_embedding(t.float().reshape(1).repeat(x.shape[0]), W)
    te = O.text_embedding(text, x.shape[1], drop, W, cfg)
    h = O.input_embedding(x, cond, te, drop, W)
    rope = O.rotary_freqs(x.shape[1], cfg.dim_head)
    out = []
    for i in range(cfg.depth):
        p = f"transformer.transformer_blocks.{i}."
        out.append((f"block {i:2d} attn_norm", row_r(h)))
        emb = O.linear(torch.nn.functional.silu(tt), W[p + "attn_norm.linear.weight"], W[p + "attn_norm.linear.bias"])
        shift_msa, scale_msa, gate_msa = emb.chunk(6, dim=1)[:3]
        a = O.attention(h, None, rope, W, p + "attn.", cfg.heads, adaln=(scale_msa, shift_msa))
        out.append((f"block {i:2d} ff_norm", row_r(h + gate_msa[:, None] * a)))
        h = O.dit_block(h, tt, None, rope, W, i, cfg)
    out.append(("norm_out", row_r(h)))
    return out


def predicted_ratio(r: torch.Tensor) -> float:
    """Fused / unfused error-norm ratio of the operand rounding over these rows: sqrt(1 + mean r^2)."""
    return float(torch.sqrt(1 + (r * r).mean()))


def load(model: str):
    from f5_tts_mlx_b200.weights import BASE_CONFIG, random_dit_weights
    if model == "random":
        c = BASE_CONFIG
        return random_dit_weights(c, seed=1234), O.DiTConfig(
            dim=c.dim, depth=c.depth, heads=c.heads, ff_mult=c.ff_mult, text_num_embeds=c.text_num_embeds,
            text_dim=c.text_dim, conv_layers=c.conv_layers), "random-init base model (seed 1234)"
    path = Path(model)
    if not path.is_dir():
        raise SystemExit(f"--model: {model} is not a local checkpoint directory")
    from f5_tts_mlx_b200.pretrained import checkpoint_weights
    vocab, weights_fn = checkpoint_weights(path)
    W = {k: v.float() for k, v in weights_fn().items()}
    return W, O.DiTConfig(text_num_embeds=len(vocab) - 1), f"checkpoint {path}"


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--model", default="random", help='"random" or a local checkpoint directory')
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--steps", type=int, default=32, help="Euler grid points (sample()'s steps)")
    ap.add_argument("--times", type=int, default=4, help="how many of the evaluation times to report, spread evenly")
    ap.add_argument("--cfg", action="store_true", help="also the CFG pass without audio prompt and text")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    torch.set_grad_enabled(False)
    W, cfg, what = load(a.model)
    g = torch.Generator().manual_seed(a.seed)
    N = a.frames
    x = torch.randn(1, N, cfg.mel_dim, generator=g)
    cond = torch.randn(1, N, cfg.mel_dim, generator=g) * 2.24 - 1.27
    cond[:, N // 3:] = 0
    text = torch.randint(0, cfg.text_num_embeds, (1, N // 5), generator=g, dtype=torch.int32)
    ts = O.time_grid(a.steps, -1.0)[:-1]
    pick = sorted({round(i * (len(ts) - 1) / max(a.times - 1, 1)) for i in range(a.times)})
    print(f"{what}: {N} frames, Euler {a.steps} grid points (sway -1); r = |row mean| / row std")
    for drop in ([False, True] if a.cfg else [False]):
        for k in pick:
            t = ts[k]
            print(f"\nt = {float(t):.4f} (evaluation {k + 1} of {len(ts)}){' , CFG null pass' if drop else ''}")
            print(f"  {'site':22s} {'p50':>8s} {'p99':>8s} {'max':>8s}   fused/unfused predicted")
            for site, r in stream_conditioning(x, cond, text, t, W, cfg, drop):
                q = torch.quantile(r, torch.tensor([0.5, 0.99], dtype=torch.float64))
                print(f"  {site:22s} {q[0]:8.3f} {q[1]:8.3f} {r.max():8.3f}   {predicted_ratio(r):.4f}")


if __name__ == "__main__":
    main()
