"""Measure the DiT's precision modes side by side: bf16, FP8 with per-tensor scales, FP8 with block scales, and FP8 with
block scales and the FP8 attention.

Runs bench.py's headline workload (B = 1 x 10 s, Euler 32, CFG 2) and its config 5 (60 s, N = 5625) in each mode through
bench.measure.  The modes alternate, in a rotated order, over --repeats rounds within one process, because a power-capped
card's clocks move between runs.  One JSON line per run gives ms per step, per-family device times and the clocks of
that run.  One summary line per mode gives the median, minimum and maximum ms per step, the median attention-, GEMM-
and other-family ms per step, the SM clock of each run, and the card's name and power limit.  Each mode's returned mel goes to <out>/<workload>_<mode>.npy, and the rel-L2 of each
FP8 mel against the bf16 mel of the same workload is reported.

    python scripts/fp8_modes.py --out /tmp/fp8_modes [--steps 10] [--no-long]
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402

MODES = {"bf16": dict(fp8=False), "fp8_tensor": dict(fp8=True, fp8_scaling="tensor"),
         "fp8_block": dict(fp8=True, fp8_scaling="block"),
         "fp8_block_attn": dict(fp8=True, fp8_scaling="block", fp8_attention=True)}


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, plim, smax = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": plim, "max_sm_clock": smax}


def quant_pass_us(lib, rows_per_utt: int, utts: int, heads: int, dev, launches: int = 200) -> float:
    """Device time of one f5_qkv_quant_e4m3 (the FP8 attention's quantise pass) at a DiT block's shape: CUDA events
    around `launches` back-to-back launches on random bf16 qkv, after a warm-up."""
    import ctypes as C
    from f5_tts_mlx_b200 import _lib
    D, R = heads * 64, utts * rows_per_utt
    qkv = torch.randn(R, 3 * D, device=dev).bfloat16()
    qk = torch.empty(R, 2 * D, dtype=torch.uint8, device=dev)
    vt = torch.empty(utts, D, (rows_per_utt + 127) // 128 * 128, dtype=torch.uint8, device=dev)
    sc = torch.empty(3 * heads, R, device=dev)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    run = lambda: _lib.check(lib.f5_qkv_quant_e4m3(qkv.data_ptr(), 3 * D, qk.data_ptr(), 2 * D, vt.data_ptr(),
                                                   vt.shape[2], sc.data_ptr(), utts, rows_per_utt, heads, st))
    for _ in range(10):
        run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / launches


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3, help="rounds; each runs every mode once, in a rotated order")
    ap.add_argument("--no-long", action="store_true", help="skip config 5 (60 s)")
    args = ap.parse_args()
    from f5_tts_mlx_b200 import BASE_CONFIG, DiT, F5TTS, _lib
    from f5_tts_mlx_b200.weights import random_dit_weights
    if not torch.cuda.is_available():
        raise SystemExit("scripts/fp8_modes.py measures on the GPU; no CUDA device is visible")
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    cfg = BASE_CONFIG
    W = random_dit_weights(cfg, seed=1234)
    N, NR = bench.TOTAL_SAMPLES // bench.HOP, bench.REF_SAMPLES // bench.HOP
    wls = [(bench.Workload("b1_10s", 1, N, NR, "euler", 32, 2.0), args.steps)]
    if not args.no_long:
        wls.append((bench.Workload("cfg5_long60s", 1, 5625, 499, "euler", 32, 2.0, n_text=bench.N_TEXT * 6), 3))
    info = card()
    print(json.dumps(info), flush=True)
    for wl, steps in wls:
        models = {mode: DiT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult, mel_dim=cfg.mel_dim,
                            text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim, conv_layers=cfg.conv_layers,
                            device=dev, **kw).load_weights(W) for mode, kw in MODES.items()}
        runs = {mode: [] for mode in MODES}
        mels = {}
        order = list(MODES)
        for rep in range(args.repeats):
            for mode in order[rep % len(order):] + order[:rep % len(order)]:     # alternate, rotating the order
                r = bench.measure(F5TTS(models[mode]), lib, wl, 0, 1, dev, steps, args.warmup, bench.ClockSampler(0))
                r.pop("_inputs")
                mel = r.pop("_outputs")["mel"].float().cpu()
                if mode not in mels:
                    mels[mode] = mel
                    np.save(os.path.join(args.out, f"{wl.name}_{mode}.npy"), mel.numpy())
                roof = r["roofline"]
                line = {"workload": wl.name, "mode": mode, "repeat": rep, "ms_per_step": r["ms_per_step"],
                        "gemm_ms_per_step": roof["gemm_ms_per_step"],
                        "attention_ms_per_step": roof["attention"]["ms_per_step"],
                        "other_ms_per_step": roof["other_ms_per_step"], "launches_per_step": r["launches_per_step"],
                        "clocks": r.get("clocks")}
                runs[mode].append(line)
                print(json.dumps(line), flush=True)
        for mode in MODES:
            ms = sorted(x["ms_per_step"] for x in runs[mode])
            clk = [x["clocks"]["sm_mhz"] for x in runs[mode] if x.get("clocks")]
            med = lambda key: sorted(x[key] for x in runs[mode])[len(ms) // 2]
            summary = {"workload": wl.name, "mode": mode, "runs": len(ms), "ms_per_step_median": ms[len(ms) // 2],
                       "ms_per_step_min": ms[0], "ms_per_step_max": ms[-1],
                       "attention_ms_per_step_median": med("attention_ms_per_step"),
                       "gemm_ms_per_step_median": med("gemm_ms_per_step"),
                       "other_ms_per_step_median": med("other_ms_per_step"), "sm_mhz_per_run": clk, **info}
            if MODES[mode].get("fp8_attention"):   # the pass's own device time; its 22 launches per step are in `other`
                us = quant_pass_us(lib, wl.frames, 2 if wl.cfg else 1, cfg.heads, dev)
                summary["quant_pass_us"] = us
                summary["quant_pass_ms_per_step"] = us * cfg.depth * 1e-3
            if mode != "bf16":
                a, b = mels[mode].double(), mels["bf16"].double()
                summary["mel_rel_l2_vs_bf16"] = ((a - b).norm() / b.norm()).item()
            print(json.dumps(summary), flush=True)
        del models
        torch.cuda.empty_cache()

if __name__ == "__main__":
    main()
