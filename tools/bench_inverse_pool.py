"""Serving trace through StreamPool -> spectral gain -> nnaudio_b200.streaming.InversePool (analysis and synthesis
per client, as in speech enhancement), against serving the synthesis half without a pool.

Trace: that of tools/bench_stream_pool.py (256 slots at 16 kHz, packets of 160-480 samples, ~15 % of the slots idle,
~1 % ending and restarting per push, streams of at most 10 s), here through STFT n_fft 512 / hop 128, Complex,
iSTFT=True, a fixed gain on every bin, and the inverse STFT of the same module.  Legs:
  pool        StreamPool -> gain -> InversePool: one tick = one push of each pool
  per_client  the same StreamPool -> gain, then one StreamingInverse per client with new frames (flush on end)
  inverse     InversePool alone, fed the gained frames of the same trace computed beforehand
Per push: host issue time (median of the tick, no synchronisation), stream time per push from CUDA events over
the timed pushes (device time while the GPU is the bottleneck, the issue time otherwise), and output samples/s.

    python tools/bench_inverse_pool.py [--pushes 500] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

here = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(here))
sys.path.insert(0, here)
from bench_stream_pool import MAX_PACKET, S, SR, _card, _timed, trace  # noqa: E402

from nnaudio_b200 import features  # noqa: E402
from nnaudio_b200.streaming import InversePool, StreamingInverse, StreamPool  # noqa: E402

GAIN = 0.5


def _leg(issue, dev, wall, samples, n):
    return {"issue_ms": round(issue, 4), "stream_ms_per_push": round(dev, 4),
            "samples_per_push": round(samples / n, 1), "samples_per_s": round(samples / wall)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pushes", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--client-pushes", type=int, default=60, help="timed ticks of the per-client baseline")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_inverse_pool needs a CUDA device")
    stft = features.STFT(n_fft=512, hop_length=128, output_format="Complex", iSTFT=True, verbose=False).cuda()
    n = args.warmup + args.pushes
    tr = trace(n)
    chunk = torch.randn(S, MAX_PACKET, device="cuda")
    res = {"card": _card(), "slots": S, "trace": "STFT 512/128 Complex 16 kHz -> gain -> iSTFT, packets 160-480, "
                                                  "15 % idle, 1 % end + restart per push, streams <= 10 s"}
    with torch.no_grad():
        fwd, inv = StreamPool(stft, S, _strict=True), InversePool(stft, S)

        def pool_step(i):
            lengths, end = tr[i]
            a = fwd.push(chunk, lengths, end)
            y = inv.push(a.frames * GAIN, a.slots, a.counts, end)
            if end.any():
                fwd.reset(np.flatnonzero(end))
                inv.reset(np.flatnonzero(end))
            return int(y.counts.sum())

        res["pool"] = _leg(*_timed(pool_step, args.warmup, args.pushes), args.pushes)

        fwd = StreamPool(stft, S, _strict=True)
        clients = [StreamingInverse(stft, 1) for _ in range(S)]

        def client_step(i):
            lengths, end = tr[i]
            a = fwd.push(chunk, lengths, end)
            X = a.frames * GAIN
            got = 0
            for r, (s, c) in enumerate(zip(a.slots.tolist(), a.counts.tolist())):
                got += clients[s].push(X[r:r + 1, :, :c]).shape[1]
            for s in np.flatnonzero(end).tolist():
                got += clients[s].flush().shape[1]
                clients[s].reset()
            if end.any():
                fwd.reset(np.flatnonzero(end))
            return got

        # the per-client leg replays the trace from its start, as the pool leg did
        warm = min(args.warmup, 10)
        res["per_client"] = _leg(*_timed(client_step, warm, args.client_pushes), args.client_pushes)

        # the inverse alone: the gained frames of the whole trace first, then the InversePool pushes on them
        fwd = StreamPool(stft, S, _strict=True)
        feed = []
        for i in range(n):
            lengths, end = tr[i]
            a = fwd.push(chunk, lengths, end)
            feed.append((a.frames * GAIN, a.slots, a.counts, end))
            if end.any():
                fwd.reset(np.flatnonzero(end))
        inv = InversePool(stft, S)

        def inverse_step(i):
            X, slots, counts, end = feed[i]
            y = inv.push(X, slots, counts, end)
            if end.any():
                inv.reset(np.flatnonzero(end))
            return int(y.counts.sum())

        res["inverse"] = _leg(*_timed(inverse_step, args.warmup, args.pushes), args.pushes)
    res["pool_vs_per_client"] = round(res["pool"]["samples_per_s"] / res["per_client"]["samples_per_s"], 1)
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
