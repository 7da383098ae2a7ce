"""Device-planned pools against the host-planned ones on the serving traces of tools/bench_stream_pool.py and
tools/bench_inverse_pool.py, eagerly and as one replayed CUDA graph per tick.

Traces: 256 slots at 16 kHz, packets of 160-480 samples, ~15 % of the slots idle, ~1 % ending and restarting per
push, streams of at most 10 s.  Ticks:
  mel          MelSpectrogram n_fft 512 / hop 128 / 80 mels
  enhance      STFT 512 / 128 Complex -> gain -> inverse STFT
Routes per tick: host (StreamPool / InversePool), device_eager (DeviceStreamPool / DeviceInversePool, one call per
push), device_graph (the device pools' tick captured once and replayed).  The device routes read the tick's
lengths / end / restart from device tensors made before the timing; the graph route copies them into its static
inputs (device to device) before each replay.  Per tick: host issue time (median, no synchronisation), stream time
from CUDA events over the timed ticks, frames/s and output samples/s (the routes return the same frames).  The
routes alternate, their order reversed on every other run.

    python tools/bench_device_pool.py [--pushes 500] [--runs 2] [--out results.json]
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
from nnaudio_b200.streaming import DeviceInversePool, DeviceStreamPool, InversePool, StreamPool  # noqa: E402

GAIN = 0.5


def _device_trace(tr):
    """(lengths, end, restart) device tensors per tick; restart = the previous tick's ends."""
    out, prev = [], np.zeros(S, bool)
    for lengths, end in tr:
        out.append((torch.as_tensor(lengths, dtype=torch.int32).cuda(), torch.as_tensor(end).cuda(),
                    torch.as_tensor(prev).cuda()))
        prev = end
    return out


def _routes(kind, tr, dtr, chunk):
    """{route: step(i) -> frames (host route; 0 elsewhere)} for one tick kind."""
    if kind == "mel":
        m = features.MelSpectrogram(sr=SR, n_fft=512, hop_length=128, n_mels=80, verbose=False).cuda()
    else:
        m = features.STFT(n_fft=512, hop_length=128, output_format="Complex", iSTFT=True, verbose=False).cuda()
    fwd = StreamPool(m, S, _strict=True)
    inv = InversePool(m, S) if kind == "enhance" else None

    def host(i):
        lengths, end = tr[i]
        if i > 0 and tr[i - 1][1].any():
            fwd.reset(np.flatnonzero(tr[i - 1][1]))
            if inv is not None:
                inv.reset(np.flatnonzero(tr[i - 1][1]))
        a = fwd.push(chunk, lengths, end)
        if inv is None:
            return int(a.counts.sum())
        return int(inv.push(a.frames * GAIN, a.slots, a.counts, end).counts.sum())

    def device_pools():
        p = DeviceStreamPool(m, S, MAX_PACKET)
        return p, (DeviceInversePool(m, S, frames=p.T_cap) if kind == "enhance" else None)

    dp, ds = device_pools()

    def tick(p, s, lengths, end, restart):
        p.reset(restart)
        p.push(chunk, lengths, end)
        if s is not None:
            s.reset(restart)
            s.push(p.frames * GAIN, p.counts, end)

    def device_eager(i):
        tick(dp, ds, *dtr[i])
        return 0

    gp, gs = device_pools()
    static = tuple(torch.zeros_like(t) for t in dtr[0])
    tick(gp, gs, *static)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        tick(gp, gs, *static)

    def device_graph(i):
        for dst, src in zip(static, dtr[i]):
            dst.copy_(src)
        g.replay()
        return 0

    return {"host": host, "device_eager": device_eager, "device_graph": device_graph}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pushes", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_device_pool needs a CUDA device")
    n = args.warmup + args.pushes
    tr = trace(n)
    dtr = _device_trace(tr)
    chunk = torch.randn(S, MAX_PACKET, device="cuda")
    res = {"card": _card(), "slots": S, "trace": "16 kHz, packets 160-480, 15 % idle, 1 % end + restart per push, "
                                                  "streams <= 10 s", "runs": []}
    with torch.no_grad():
        for run in range(args.runs):
            out = {}
            for kind in ("mel", "enhance"):
                routes = _routes(kind, tr, dtr, chunk)
                order = list(routes) if run % 2 == 0 else list(routes)[::-1]
                legs, frames = {}, None
                for name in order:
                    issue, dev, wall, acc = _timed(routes[name], args.warmup, args.pushes)
                    legs[name] = {"issue_ms": round(issue, 4), "stream_ms_per_tick": round(dev, 4), "wall": wall}
                    if name == "host":
                        frames = acc
                unit = "frames" if kind == "mel" else "samples"
                for leg in legs.values():
                    leg[f"{unit}_per_s"] = round(frames / leg.pop("wall"))
                out[kind] = {k: legs[k] for k in routes}
            res["runs"].append(out)
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
