"""Serving trace through nnaudio_b200.streaming.StreamPool, against the two ways to serve it without a pool.

Trace: 256 slots of 16 kHz Mel (n_fft 512, hop 128, 80 mels); each push gives every slot a seeded packet of
160-480 samples, with ~15 % of the slots idle; ~1 % of the slots end their stream (a client leaving) and restart
in every push, streams end after 10 s at the latest.  Per push: host issue time (median of the push call, no
synchronisation), stream time per push from CUDA events over the timed pushes (device time while the GPU is the
bottleneck, the issue time otherwise), and frames/s.  Baselines, compared per frame:
  uniform     StreamingTransform on 256 streams with uniform 320-sample pushes (every client in lock step)
  per_client  one StreamingTransform per active client: one push per client with samples in each tick

    python tools/bench_stream_pool.py [--pushes 500] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nnaudio_b200 import features  # noqa: E402
from nnaudio_b200.streaming import StreamingTransform, StreamPool  # noqa: E402

S, SR, MAX_PACKET = 256, 16000, 480


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the measurement itself needs no nvidia-smi
        return f"unknown ({e})"


def trace(pushes, seed=0):
    """[(lengths, end)] per push: the serving trace of the module docstring."""
    rng = np.random.default_rng(seed)
    stop = rng.integers(SR, 10 * SR + 1, size=S)  # staggered first streams
    pos = np.zeros(S, int)
    out = []
    for _ in range(pushes):
        lengths = np.minimum(rng.integers(160, MAX_PACKET + 1, size=S) * (rng.random(S) < 0.85), stop - pos)
        end = (pos + lengths >= stop) | ((rng.random(S) < 0.01) & (pos + lengths > 4000))
        pos = np.where(end, 0, pos + lengths)
        stop = np.where(end, 10 * SR, stop)
        out.append((lengths, end))
    return out


def _timed(step, n_warm, n):
    """step(i) per push -> (median host issue ms, stream ms per push, wall s of the timed pushes, result sum)."""
    for i in range(n_warm):
        step(i)
    torch.cuda.synchronize()
    issue, acc = [], 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    w0 = time.perf_counter()
    e0.record()
    for i in range(n_warm, n_warm + n):
        t0 = time.perf_counter()
        acc += step(i)
        issue.append((time.perf_counter() - t0) * 1e3)
    e1.record()
    torch.cuda.synchronize()
    wall = time.perf_counter() - w0
    return statistics.median(issue), e0.elapsed_time(e1) / n, wall, acc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pushes", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--client-pushes", type=int, default=60, help="timed ticks of the per-client baseline")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream_pool needs a CUDA device")
    m = features.MelSpectrogram(sr=SR, n_fft=512, hop_length=128, n_mels=80, verbose=False).cuda()
    tr = trace(args.warmup + args.pushes)
    chunk = torch.randn(S, MAX_PACKET, device="cuda")
    res = {"card": _card(), "slots": S, "trace": "Mel 16 kHz n_fft 512 hop 128, packets 160-480, 15 % idle, "
                                                    "1 % end + restart per push, streams <= 10 s"}
    with torch.no_grad():
        pool = StreamPool(m, S, _strict=True)

        def pool_step(i):
            lengths, end = tr[i]
            out = pool.push(chunk, lengths, end)
            if end.any():
                pool.reset(np.flatnonzero(end))
            return int(out.counts.sum())

        issue, dev, wall, frames = _timed(pool_step, args.warmup, args.pushes)
        res["pool"] = {"issue_ms": round(issue, 4), "stream_ms_per_push": round(dev, 4),
                       "frames_per_push": round(frames / args.pushes, 1),
                       "frames_per_s": round(frames / wall), "us_per_frame": round(wall * 1e6 / frames, 4)}

        st = StreamingTransform(m, S, _strict=True)
        x = torch.randn(S, 320, device="cuda")
        issue, dev, wall, frames = _timed(lambda i: int(st.push(x).shape[2]) * S, args.warmup, args.pushes)
        res["uniform"] = {"issue_ms": round(issue, 4), "stream_ms_per_push": round(dev, 4),
                          "frames_per_push": round(frames / args.pushes, 1),
                          "frames_per_s": round(frames / wall), "us_per_frame": round(wall * 1e6 / frames, 4)}

        clients = [StreamingTransform(m, 1, _strict=True) for _ in range(S)]

        def client_step(i):
            lengths, end = tr[i]
            n = 0
            for s in np.flatnonzero(lengths).tolist():
                n += clients[s].push(chunk[s:s + 1, :lengths[s]]).shape[2]
            for s in np.flatnonzero(end).tolist():
                n += clients[s].flush().shape[2]
                clients[s].reset()
            return n

        warm = min(args.warmup, 10)
        issue, dev, wall, frames = _timed(client_step, warm, args.client_pushes)
        res["per_client"] = {"issue_ms_per_tick": round(issue, 4), "stream_ms_per_tick": round(dev, 4),
                             "frames_per_tick": round(frames / args.client_pushes, 1),
                             "frames_per_s": round(frames / wall), "us_per_frame": round(wall * 1e6 / frames, 4)}
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
