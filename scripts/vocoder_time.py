"""Time the Vocos and BigVGAN v2 decodes of 10 s and 60 s mels at batch 1 on one GPU, alternating the two vocoders in
one process, and report algorithmic FLOPs, achieved TFLOP/s and BigVGAN's launch gaps.

    python scripts/vocoder_time.py [--iters 20] [--warmup 3] [--out vocoder_time.json]

Random weights (seeded); the card name, power limit and SM clock are read in the same run.  FLOPs are 2 * MACs of every
convolution and matmul, computed from the shapes (ConvTranspose1d: the real k / u taps per output, not the zero taps of
the polyphase packing).  The launch gaps come from a torch.profiler trace of one BigVGAN decode: the idle time between
consecutive kernels on the stream.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def bigvgan_flops(cfg, frames: int) -> float:
    f = 2.0 * frames * cfg.upsample_initial_channel * cfg.num_mels * 7
    t, c = frames, cfg.upsample_initial_channel
    for u, k in zip(cfg.upsample_rates, cfg.upsample_kernel_sizes):
        f += 2.0 * (t * u) * (c // 2) * c * (k / u)
        t, c = t * u, c // 2
        for kr in cfg.resblock_kernel_sizes:
            f += 6 * 2.0 * t * c * c * kr
    return f + 2.0 * t * c * 7


def vocos_flops(vc, frames: int) -> float:
    d, i = vc.dim, vc.intermediate_dim
    f = 2.0 * frames * vc.n_mels * d * 7 + vc.num_layers * (2.0 * frames * d * i * 2 + 2.0 * frames * d * 7)
    return f + 2.0 * frames * d * (vc.n_fft + 2)


def gpu_info() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smax = [s.strip() for s in q.split(",")]
        return dict(name=name, power_limit=pl, sm_clock=sm, sm_clock_max=smax)
    except Exception as e:     # the timing itself does not depend on it
        return dict(name=torch.cuda.get_device_name(), error=str(e))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vocoder_time.py needs a GPU")
    from f5_tts_mlx_b200 import _lib
    from f5_tts_mlx_b200.bigvgan import BigVGAN, BigVGANConfig, random_bigvgan_weights
    from f5_tts_mlx_b200.vocos import Vocos
    from f5_tts_mlx_b200.weights import VocosConfig, random_vocos_weights
    dev = torch.device("cuda")
    bcfg, vcfg = BigVGANConfig(), VocosConfig()
    voc = {"vocos": Vocos(vcfg, dev).load_weights(random_vocos_weights()),
           "bigvgan": BigVGAN(bcfg, dev).load_weights(random_bigvgan_weights(bcfg, seed=1))}
    flops = {"vocos": lambda n: vocos_flops(vcfg, n), "bigvgan": lambda n: bigvgan_flops(bcfg, n)}
    g = torch.Generator().manual_seed(0)
    res = {"gpu": gpu_info(), "iters": a.iters, "results": []}
    lib = _lib.load()
    for seconds in (10, 60):
        n = int(seconds * 24000 / 256)
        mel = (torch.randn(1, n, 100, generator=g) - 3).to(dev)
        for name in voc:
            for _ in range(a.warmup):
                voc[name].decode(mel)
        times = {k: [] for k in voc}
        launches = {}
        for _ in range(a.iters):                      # alternate the vocoders decode by decode
            for name in voc:
                c0 = lib.f5_launch_count()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                voc[name].decode(mel)
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1))
                launches[name] = lib.f5_launch_count() - c0
        for name in voc:
            t = sorted(times[name])
            med = t[len(t) // 2]
            res["results"].append(dict(vocoder=name, seconds=seconds, frames=n, median_ms=med, min_ms=t[0], max_ms=t[-1],
                                       gflop=flops[name](n) / 1e9, tflops=flops[name](n) / (med * 1e-3) / 1e12,
                                       launches=launches[name]))
            print(json.dumps(res["results"][-1]), flush=True)
        # launch gaps of one BigVGAN decode
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            voc["bigvgan"].decode(mel)
            torch.cuda.synchronize()
        ev = sorted([e for e in prof.events() if e.device_type.name == "CUDA" and e.device_time_total > 0
                     and "Memcpy" not in e.name and "Memset" not in e.name], key=lambda e: e.time_range.start)
        gaps = [max(0.0, ev[i + 1].time_range.start - ev[i].time_range.end) for i in range(len(ev) - 1)]
        busy = sum(e.time_range.end - e.time_range.start for e in ev)
        res["results"].append(dict(vocoder="bigvgan", seconds=seconds, kernels=len(ev), kernel_busy_us=busy,
                                   gap_total_us=sum(gaps), gap_median_us=sorted(gaps)[len(gaps) // 2] if gaps else 0.0))
        print(json.dumps(res["results"][-1]), flush=True)
    print(json.dumps(res["gpu"]))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
