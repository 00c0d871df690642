"""In-situ duration of each DiT block GEMM role (QKV / out-proj / FF1 / FF2) on bench.py's headline workload.

Captures the workload's CUDA graph (B = 1 x 10 s, Euler 32 grid points, CFG 2) with the f5_prof_graph_begin timing
slots installed, exactly as bench.py does, replays it `--replays` times with the slots reset, and classifies every
GEMM launch by its (N, K, output type) and row count.  Per role it prints the median in-situ duration over all
launches of all replays (22 blocks x 31 forwards per replay at the headline), with the role's tiles per CTA on the
persistent grid and an MMA-only lower bound: the most tiles any CTA runs x 2 * 128 * BN * K flops at the dense wgmma
rate of one SM (4096 BF16 / 8192 FP8 flops per clock, the data sheet's 989 / 1979 TFLOP/s over 132 SMs at 1830 MHz),
taken at the SM clock sampled during the replays.  The excess over the bound is prologue, pipeline fill and whatever
epilogue the ping-pong does not hide.  An in-situ duration runs from the first CTA past its dependency wait to the last
CTA's exit (ptx.cuh prof_stamp_*).

    python scripts/gemm_tail.py [--fp8] [--replays 5] [--label NAME] [--out DIR]

Runs on the GPU only: without a CUDA device it exits with an error.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
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


def cdiv(a: int, b: int) -> int:
    return (a + b - 1) // b


def launcher_bn(m: int, n: int, sms: int) -> int:
    """The tile width f5_gemm_bf16 picks for a flat GEMM with tile_n = 0 (gemm.cu)."""
    if n <= 64:
        return 64
    return 128 if cdiv(m, 128) * cdiv(n, 128) >= (sms * 13) // 16 else 64


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--fp8", action="store_true", help="the block-scaled FP8 mode of the DiT (bench.py's b1_fp8)")
    ap.add_argument("--replays", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--label", default="", help="a name for this build, echoed in every line")
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/gemm_tail[_LABEL].jsonl")
    args = ap.parse_args()
    import torch
    import bench
    from f5_tts_mlx_b200 import BASE_CONFIG, DiT, F5TTS, _lib
    from f5_tts_mlx_b200.weights import random_dit_weights
    if not torch.cuda.is_available():
        raise SystemExit("scripts/gemm_tail.py measures on the GPU; no CUDA device is visible")
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    info = {**card(), "sms": sms, "label": args.label, "mode": "fp8" if args.fp8 else "bf16"}
    lines = [info]
    print(json.dumps(info), flush=True)

    c = BASE_CONFIG
    model = DiT(dim=c.dim, depth=c.depth, heads=c.heads, ff_mult=c.ff_mult, mel_dim=c.mel_dim,
                text_num_embeds=c.text_num_embeds, text_dim=c.text_dim, conv_layers=c.conv_layers, device=dev,
                fp8=args.fp8).load_weights(random_dit_weights(c, seed=1234))
    f5 = F5TTS(model)
    N, NR = bench.TOTAL_SAMPLES // bench.HOP, bench.REF_SAMPLES // bench.HOP
    g = torch.Generator().manual_seed(100 + 17 + N)
    cond = (torch.randn(1, NR, 100, generator=g) * 2.24 - 1.27).clamp(-11.51, 5.0).to(dev)
    text = torch.randint(0, 2545, (1, bench.N_TEXT), generator=g, dtype=torch.int32)
    y0 = torch.randn(1, 100, N, generator=g).permute(0, 2, 1).contiguous().to(dev)
    kw = dict(steps=32, method="euler", cfg_strength=2.0, sway_sampling_coef=-1.0, return_trajectory=False)

    # eager pass (kernel attributes, validation), then the capture with timing slots, as bench.measure does
    f5.use_cuda_graph = False
    c0 = lib.f5_launch_count()
    f5.sample(cond, text, N, y0=y0, **kw)
    torch.cuda.synchronize()
    cap = int(lib.f5_launch_count() - c0) + 64
    plan = f5.last_plan
    slots = torch.zeros(cap, 2, dtype=torch.int64, device=dev)
    lib.f5_prof_graph_begin(C.c_void_p(slots.data_ptr()), cap)
    plan.capture(f5)
    lib.f5_prof_graph_begin(None, 0)
    kinds = (C.c_int32 * cap)(); flops = (C.c_double * cap)(); nbytes = (C.c_double * cap)()
    n_slots = lib.f5_prof_graph_meta(kinds, flops, nbytes, cap)

    def replay():
        plan.y.copy_(y0)
        plan.graph.replay()

    for _ in range(args.warmup):
        replay()
    torch.cuda.synchronize()

    D, Fi = c.dim, c.dim * c.ff_mult
    roles = {"qkv": (3 * D, D, 2), "out": (D, D, 4), "ff1": (Fi, D, 2), "ff2": (D, Fi, 4)}   # N, K, output bytes

    def classify(i: int):
        if kinds[i] != 0:
            return None
        for name, (n, k, ob) in roles.items():
            m = round(flops[i] / (2.0 * n * k))
            if m > 0 and flops[i] == 2.0 * m * n * k and nbytes[i] == 2.0 * (m * k + n * k) + m * n * ob:
                return name, m
        return None

    cls = [classify(i) for i in range(n_slots)]
    dur: dict[tuple, list] = {}
    clocks = bench.ClockSampler(0)
    clocks.start()
    for _ in range(args.replays):
        slots[:, 0] = -1
        slots[:, 1] = 0
        replay()
        torch.cuda.synchronize()
        sl = slots[:n_slots].cpu().tolist()
        for i, key in enumerate(cls):
            if key is None or sl[i][0] == -1 or sl[i][1] == 0:
                continue
            dur.setdefault(key, []).append((sl[i][1] - sl[i][0]) * 1e-3)     # ns -> us
    clk = clocks.stop()
    mhz = clk.get("sm_mhz") or float(info["max_sm_clock"].split()[0])
    per_clk = 8192 if args.fp8 else 4096

    for (name, m), ds in sorted(dur.items(), key=lambda kv: (-len(kv[1]), kv[0])):
        n, k, _ = roles[name]
        bn = launcher_bn(m, n, sms)
        tiles = cdiv(m, 128) * cdiv(n, bn)
        grid = min(tiles, sms)
        bound = cdiv(tiles, grid) * 2.0 * 128 * bn * k / (per_clk * mhz * 1e6) * 1e6
        med = statistics.median(ds)
        line = {"label": args.label, "mode": info["mode"], "role": name, "M": m, "N": n, "K": k, "BN": bn,
                "launches": len(ds), "launches_per_replay": len(ds) // args.replays, "median_us": round(med, 3),
                "p10_us": round(sorted(ds)[len(ds) // 10], 3), "p90_us": round(sorted(ds)[(9 * len(ds)) // 10], 3),
                "tiles": tiles, "tiles_per_cta": [tiles // grid, cdiv(tiles, grid)], "idle_sms": sms - grid,
                "mma_bound_us": round(bound, 3), "excess_us": round(med - bound, 3), "sm_mhz": mhz}
        lines.append(line)
        print(json.dumps(line), flush=True)
    lines.append({"label": args.label, "clocks": clk})
    print(json.dumps(lines[-1]), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        suffix = f"_{args.label}" if args.label else ""
        with open(os.path.join(args.out, f"gemm_tail{suffix}.jsonl"), "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
