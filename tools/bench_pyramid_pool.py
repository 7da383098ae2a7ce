"""Serving-trace benchmark of PyramidPool: 64 slots of cfg4 CQT2010v2 (22.05 kHz, 88 bins, hop 512) fed 10-40 ms
packets, about 15 % of the slots idle and about 1 % ending (and restarting) per push.  Compares the pool with one
StreamingPyramid per active client on the same trace and prints one JSON line: host issue time and stream time per
push, frames/s, the state bytes per slot, and the card and power limit read in the same run.

    python tools/bench_pyramid_pool.py [--slots 64] [--pushes 500] [--warmup 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from nnaudio_b200 import features  # noqa: E402
from nnaudio_b200.streaming import PyramidPool, StreamingPyramid  # noqa: E402


def _card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                            f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def _trace(S, n_push, sr, seed):
    """Per push: packet width, per-slot lengths and ends (ended slots restart on the next push)."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n_push):
        n = int(rng.integers(sr // 100, sr * 4 // 100 + 1))
        lengths = np.where(rng.random(S) < 0.15, 0, n)
        end = (lengths > 0) & (rng.random(S) < 0.01)
        out.append((n, lengths, end))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=64)
    ap.add_argument("--pushes", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=100)
    a = ap.parse_args()
    sr, S = 22050, a.slots
    m = features.CQT2010v2(sr=sr, hop_length=512, n_bins=88, verbose=False).cuda()
    # warm-up long enough that every slot's stream is past the pyramid's start-up latency (1.5 s)
    trace = _trace(S, a.warmup + a.pushes, sr, seed=1)
    x = torch.randn(S, sr * 4 // 100 + 1, device="cuda")

    def run_pool():
        pool = PyramidPool(m, S)
        host = frames = 0
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        for k, (n, lengths, end) in enumerate(trace):
            if k == a.warmup:
                torch.cuda.synchronize()
                ev[0].record()
                host, frames = 0.0, 0
            t0 = time.perf_counter()
            out = pool.push(x[:, :n], lengths, end)
            pool.reset(np.flatnonzero(end))
            host += time.perf_counter() - t0
            frames += int(out.counts.sum())
        ev[1].record()
        torch.cuda.synchronize()
        return host, ev[0].elapsed_time(ev[1]) / 1e3, frames

    def run_streamers():
        st = [StreamingPyramid(m, 1) for _ in range(S)]
        host = frames = 0
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        for k, (n, lengths, end) in enumerate(trace):
            if k == a.warmup:
                torch.cuda.synchronize()
                ev[0].record()
                host, frames = 0.0, 0
            t0 = time.perf_counter()
            for s in np.flatnonzero(lengths).tolist():
                frames += st[s].push(x[s:s + 1, :n]).shape[2]
                if end[s]:
                    frames += st[s].flush().shape[2]
                    st[s].reset()
            host += time.perf_counter() - t0
        ev[1].record()
        torch.cuda.synchronize()
        return host, ev[0].elapsed_time(ev[1]) / 1e3, frames

    res = {}
    for name, fn in (("pool", run_pool), ("per_client", run_streamers)):
        fn()  # packed operands, allocator
        host, wall, frames = fn()
        res[name] = {"host_ms_per_push": round(1e3 * host / a.pushes, 3),
                     "stream_ms_per_push": round(1e3 * wall / a.pushes, 3),
                     "frames_per_s": round(frames / wall, 1)}
    card, power = _card()
    state = PyramidPool(m, 1).ring.numel() * 4
    print(json.dumps({"workload": "cfg4 CQT2010v2-88 serving trace", "slots": S, "pushes": a.pushes, **res,
                      "speedup_frames_per_s": round(res["pool"]["frames_per_s"] / res["per_client"]["frames_per_s"], 2),
                      "state_bytes_per_slot": state, "gpu": card, "power_limit": power}))


if __name__ == "__main__":
    main()
