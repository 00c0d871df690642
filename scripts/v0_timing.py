"""Time the F5TTS_Base (v0) model against v1, and v1 against a build of an earlier commit of this library.

Runs bench.py's headline workload (B = 1 x 10 s, Euler 32, CFG 2) through bench.measure.  v0 adds no work (its QKV
epilogue rotates fewer chunks, its text embedding skips a mask), so v0 and v1 should take the same time.  Each run is a
separate process, because one process loads one libf5b200.so: the runs alternate `--rounds` times between the build
under test (which times v1 and v0, alternating) and `--parent-lib` (v1 only), since a power-capped card's clocks move
between runs.  One JSON line per measurement; the summary gives the median / min / max ms per step per arm, whether the
v1 mels of the two builds are bitwise equal, and the card's name and power limit.

    python scripts/v0_timing.py --out /tmp/v0_timing --parent-lib /path/to/parent/libf5b200.so [--rounds 3]
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

VERSIONS = {"v1": dict(), "v0": dict(text_mask_padding=False, pe_attn_head=1)}


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, plim, smax = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": plim, "max_sm_clock": smax}


def run_arm(arm: str, versions: list, out: str, steps: int, warmup: int, rnd: int) -> None:
    """One process: measure each of `versions` once per repeat, alternating, on the library this process loads."""
    import numpy as np
    import torch
    import bench
    from f5_tts_mlx_b200 import BASE_CONFIG, DiT, F5TTS, _lib
    from f5_tts_mlx_b200.weights import random_dit_weights
    if not torch.cuda.is_available():
        raise SystemExit("scripts/v0_timing.py measures on the GPU; no CUDA device is visible")
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    cfg = BASE_CONFIG
    W = random_dit_weights(cfg, seed=1234)
    N, NR = bench.TOTAL_SAMPLES // bench.HOP, bench.REF_SAMPLES // bench.HOP
    wl = bench.Workload("b1_10s", 1, N, NR, "euler", 32, 2.0)
    for v in versions:
        model = DiT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult, mel_dim=cfg.mel_dim,
                    text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim, conv_layers=cfg.conv_layers,
                    device=dev, **VERSIONS[v]).load_weights(W)
        r = bench.measure(F5TTS(model), lib, wl, 0, 1, dev, steps, warmup, bench.ClockSampler(0))
        r.pop("_inputs")
        mel = r.pop("_outputs")["mel"].float().cpu()
        np.save(os.path.join(out, f"{arm}_{v}_r{rnd}.npy"), mel.numpy())
        print(json.dumps({"arm": arm, "version": v, "round": rnd, "ms_per_step": r["ms_per_step"],
                          "clocks": r.get("clocks")}), flush=True)
        del model
        torch.cuda.empty_cache()


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--parent-lib", default=None, help="libf5b200.so built from the commit to compare v1 against")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--arm", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--round", type=int, default=0, help=argparse.SUPPRESS)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    if args.arm is not None:
        vs = ["v1"] if args.arm == "parent" else (["v1", "v0"] if args.round % 2 == 0 else ["v0", "v1"])
        run_arm(args.arm, vs, args.out, args.steps, args.warmup, args.round)
        return
    info = card()
    print(json.dumps(info), flush=True)
    arms = ["branch"] + (["parent"] if args.parent_lib else [])
    lines = []
    for rnd in range(args.rounds):
        for arm in (arms if rnd % 2 == 0 else arms[::-1]):
            env = dict(os.environ)
            if arm == "parent":
                env["F5_LIB"] = str(Path(args.parent_lib).resolve())
            cmd = [sys.executable, __file__, "--out", args.out, "--arm", arm, "--round", str(rnd),
                   "--steps", str(args.steps), "--warmup", str(args.warmup)]
            r = subprocess.run(cmd, env=env, capture_output=True, text=True)
            if r.returncode != 0:
                raise SystemExit(f"{arm} round {rnd} failed:\n{r.stdout}\n{r.stderr}")
            for line in r.stdout.splitlines():
                if line.startswith("{"):
                    print(line, flush=True)
                    lines.append(json.loads(line))
    import numpy as np
    for arm in arms:
        for v in (VERSIONS if arm == "branch" else ["v1"]):
            ms = sorted(x["ms_per_step"] for x in lines if x["arm"] == arm and x["version"] == v)
            print(json.dumps({"arm": arm, "version": v, "runs": len(ms), "ms_per_step_median": ms[len(ms) // 2],
                              "ms_per_step_min": ms[0], "ms_per_step_max": ms[-1], **info}), flush=True)
    if args.parent_lib:
        a = np.load(os.path.join(args.out, "branch_v1_r0.npy")); b = np.load(os.path.join(args.out, "parent_v1_r0.npy"))
        c = np.load(os.path.join(args.out, "branch_v0_r0.npy"))
        print(json.dumps({"v1_mel_bitwise_equal_to_parent": bool(np.array_equal(a.view(np.uint32), b.view(np.uint32))),
                          "v0_mel_rel_l2_vs_v1": float(np.linalg.norm(c - a) / np.linalg.norm(a))}), flush=True)


if __name__ == "__main__":
    main()
