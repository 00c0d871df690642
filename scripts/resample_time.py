"""Time the resample kernel (f5_resample) on 10 s clips: 44.1 -> 24 kHz (a reference clip on its way into the mel
front-end) and 24 -> 48 kHz (the vocoder's output on its way out), at batch 1.

Each case warms up, then times --iters launches between two CUDA events, --repeats times, in two ways: calls of
audio.resample() from Python (what a user pays per call, host overhead included) and replays of a CUDA graph of 100
f5_resample launches (the kernel back to back).  One JSON line per case gives the median and minimum microseconds per
launch of each, the bytes the kernel must move (input + output + table) and the rate that implies at the graph's
median, and one closing line the card's name, power limit and SM clock ceiling.

    python scripts/resample_time.py [--iters 2000] [--repeats 5]
"""
from __future__ import annotations

import argparse
import json
import math
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import ctypes as C  # noqa: E402

import torch  # noqa: E402

from f5_tts_mlx_b200 import _lib, resample  # noqa: E402
from f5_tts_mlx_b200.audio import _resample_table  # noqa: E402

GRAPH_LAUNCHES = 100

CASES = [(44100, 24000), (24000, 48000)]


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, plim, smax = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": plim, "max_sm_clock": smax}


def time_us(fn, iters: int, repeats: int, per_call: int = 1) -> list:
    us = []
    for _ in range(repeats):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(iters):
            fn()
        t1.record()
        t1.synchronize()
        us.append(t0.elapsed_time(t1) * 1e3 / (iters * per_call))
    return us


def main() -> None:
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=2000)
    p.add_argument("--repeats", type=int, default=5)
    p.add_argument("--seconds", type=float, default=10.0)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("resample_time.py measures the GPU kernel: no CUDA device")
    for orig, new in CASES:
        L = int(a.seconds * orig)
        x = torch.randn(1, L, device="cuda") * 0.1
        for _ in range(20):
            y = resample(x, orig, new)
        torch.cuda.synchronize()
        us_call = time_us(lambda: resample(x, orig, new), a.iters, a.repeats)
        table = _resample_table(orig, new, "cuda:0")
        out = torch.empty_like(y)
        lib = _lib.load()
        graph, side = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side), torch.cuda.graph(graph, stream=side):
            st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            for _ in range(GRAPH_LAUNCHES):
                _lib.check(lib.f5_resample(C.c_void_p(x.data_ptr()), 1, L, orig, new, C.c_void_p(table.data_ptr()),
                                           C.c_void_p(out.data_ptr()), out.shape[1], st))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, y)
        us = time_us(graph.replay, max(1, a.iters // GRAPH_LAUNCHES), a.repeats, GRAPH_LAUNCHES)
        g = math.gcd(orig, new)
        n, o = new // g, orig // g
        w = math.ceil(6 * o / (min(o, n) * 0.99))
        taps = 2 * w + o
        nbytes = 4 * (L + y.shape[1] + n * taps)
        med = statistics.median(us)
        print(json.dumps({"case": f"{orig}->{new}", "seconds": a.seconds, "in_samples": L, "out_samples": y.shape[1],
                          "table": [n, taps], "graph_us_median": round(med, 2), "graph_us_min": round(min(us), 2),
                          "call_us_median": round(statistics.median(us_call), 2),
                          "call_us_min": round(min(us_call), 2), "bytes": nbytes,
                          "GB_per_s_median": round(nbytes / med / 1e3, 1)}))
    print(json.dumps(card()))


if __name__ == "__main__":
    main()
