"""Time E2TTS_Base (the UNetT backbone) against F5TTS_v1_Base, both with seeded random weights.

Runs bench.py's headline workload (B = 1 x 10 s, Euler 32 grid points, CFG 2) and the same at 60 s through
bench.measure, in one process, alternating the two models `--rounds` times (a power-capped card's clocks move between
runs).  One JSON line per measurement (ms per step, SM clock, and the GEMM / attention / other split of the step from
the in-graph timers), then per workload the median / min / max of each model, the E2 / F5 ratio of the medians, and the
card's name and power limit.  By FLOP count an E2 step is expected to cost about 1.6-1.8x an F5 step (24 layers at about
26 D^2 GEMM FLOPs per row against 22 at 16 D^2).

    python scripts/unett_timing.py [--rounds 3] [--steps 5] [--warmup 2] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, plim, smax = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": plim, "max_sm_clock": smax}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/unett_timing.jsonl")
    args = ap.parse_args()
    import torch
    import bench
    from f5_tts_mlx_b200 import BASE_CONFIG, DiT, F5TTS, _lib
    from f5_tts_mlx_b200.unett import E2_BASE_CONFIG, UNetT, random_unett_weights
    from f5_tts_mlx_b200.weights import random_dit_weights
    if not torch.cuda.is_available():
        raise SystemExit("scripts/unett_timing.py measures on the GPU; no CUDA device is visible")
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    info = card()
    lines = [info]
    print(json.dumps(info), flush=True)
    c, e = BASE_CONFIG, E2_BASE_CONFIG
    models = {
        "f5_v1": F5TTS(DiT(dim=c.dim, depth=c.depth, heads=c.heads, ff_mult=c.ff_mult, mel_dim=c.mel_dim,
                           text_num_embeds=c.text_num_embeds, text_dim=c.text_dim, conv_layers=c.conv_layers,
                           device=dev).load_weights(random_dit_weights(c, seed=1234))),
        "e2": F5TTS(UNetT(dim=e.dim, depth=e.depth, heads=e.heads, ff_mult=e.ff_mult, text_num_embeds=e.text_num_embeds,
                          text_dim=e.text_dim, pe_attn_head=e.pe_attn_head, device=dev)
                    .load_weights(random_unett_weights(e, seed=1234))),
    }
    NR = bench.REF_SAMPLES // bench.HOP
    workloads = [bench.Workload("b1_10s", 1, bench.TOTAL_SAMPLES // bench.HOP, NR, "euler", 32, 2.0),
                 bench.Workload("b1_60s", 1, 60 * bench.SR // bench.HOP, NR, "euler", 32, 2.0)]
    res = []
    for wl in workloads:
        for rnd in range(args.rounds):
            for name in (("f5_v1", "e2") if rnd % 2 == 0 else ("e2", "f5_v1")):
                r = bench.measure(models[name], lib, wl, 0, 1, dev, args.steps, args.warmup, bench.ClockSampler(0))
                roof = r["roofline"]
                line = {"workload": wl.name, "model": name, "round": rnd, "ms_per_step": r["ms_per_step"],
                        "gemm_ms": roof["gemm_ms_per_step"], "attention_ms": roof["attention"]["ms_per_step"],
                        "other_ms": roof["other_ms_per_step"], "clocks": r.get("clocks")}
                res.append(line)
                lines.append(line)
                print(json.dumps(line), flush=True)
                models[name]._plans.clear()
                models[name].transformer._sessions.clear()
                torch.cuda.empty_cache()
        med = {}
        for name in models:
            rs = sorted((x for x in res if x["workload"] == wl.name and x["model"] == name), key=lambda x: x["ms_per_step"])
            m = rs[len(rs) // 2]
            med[name] = m["ms_per_step"]
            s = {"workload": wl.name, "model": name, "runs": len(rs), "ms_per_step_median": m["ms_per_step"],
                 "ms_per_step_min": rs[0]["ms_per_step"], "ms_per_step_max": rs[-1]["ms_per_step"],
                 "median_run_split_ms": {"gemm": m["gemm_ms"], "attention": m["attention_ms"], "other": m["other_ms"]},
                 **info}
            lines.append(s)
            print(json.dumps(s), flush=True)
        s = {"workload": wl.name, "e2_over_f5_v1": med["e2"] / med["f5_v1"]}
        lines.append(s)
        print(json.dumps(s), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "unett_timing.jsonl"), "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
