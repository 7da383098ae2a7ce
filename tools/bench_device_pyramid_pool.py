"""DevicePyramidPool against PyramidPool on the serving trace of tools/bench_pyramid_pool.py, eagerly and as one
replayed CUDA graph per tick.

Trace: 64 slots of cfg4 CQT2010v2 (22.05 kHz, 88 bins, hop 512) fed 10-40 ms packets (220-882 samples), about 15 %
of the slots idle and about 1 % ending per push, ended slots restarting on the next push.  Routes per tick: host
(PyramidPool), device_eager (DevicePyramidPool, one reset and one push call), device_graph (the same tick captured
once and replayed; the tick's lengths / end / restart are copied device to device into its static inputs first).
Before timing, the routes' frames are checked bit for bit against each other over the first ticks.  Per route:
median host issue time per tick (no synchronisation), stream time per tick from CUDA events, frames/s (the frames
PyramidPool returns over the timed ticks, divided by the route's wall time).  The routes alternate, their order
reversed on every other run.  Then the replayed tick's stream time with no slot ending against one slot ending per
tick (every slot computes its octaves at T_cap frames on every push, so the two should match).  The card's name,
power limit and max SM clock are read in the same run.

    python tools/bench_device_pyramid_pool.py [--pushes 400] [--warmup 100] [--runs 2] [--out results.json]
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
from bench_pyramid_pool import _trace  # noqa: E402
from bench_stream_pool import _card, _timed  # noqa: E402

from nnaudio_b200 import features  # noqa: E402
from nnaudio_b200.streaming import DevicePyramidPool, PyramidPool  # noqa: E402

SR, S = 22050, 64
CHUNK = SR * 4 // 100  # the widest packet


def _device_trace(tr):
    """(lengths, end, restart) device tensors per tick; restart = the previous tick's ends."""
    out, prev = [], np.zeros(S, bool)
    for _, lengths, end in tr:
        out.append((torch.as_tensor(lengths, dtype=torch.int32).cuda(), torch.as_tensor(end).cuda(),
                    torch.as_tensor(prev).cuda()))
        prev = end
    return out


def _graph(pool, x):
    static = (torch.zeros(S, dtype=torch.int32, device="cuda"), torch.zeros(S, dtype=torch.bool, device="cuda"),
              torch.zeros(S, dtype=torch.bool, device="cuda"))

    def tick():
        pool.reset(static[2])
        pool.push(x, static[0], static[1])

    tick()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        tick()
    return g, static


def _routes(m, tr, dtr, x):
    host = PyramidPool(m, S)

    def host_step(i):
        if i > 0 and tr[i - 1][2].any():
            host.reset(np.flatnonzero(tr[i - 1][2]))
        return int(host.push(x, tr[i][1], tr[i][2]).counts.sum())

    eager = DevicePyramidPool(m, S, CHUNK)

    def eager_step(i):
        lengths, end, restart = dtr[i]
        eager.reset(restart)
        eager.push(x, lengths, end)
        return 0

    graphed = DevicePyramidPool(m, S, CHUNK)
    g, static = _graph(graphed, x)

    def graph_step(i):
        for dst, src in zip(static, dtr[i]):
            dst.copy_(src)
        g.replay()
        return 0

    return {"host": host_step, "device_eager": eager_step, "device_graph": graph_step}, (host, eager, graphed)


def _check_equal(m, tr, dtr, x, ticks):
    """The routes' frames over the first ticks, bit for bit."""
    routes, (host, eager, graphed) = _routes(m, tr, dtr, x)
    for i in range(ticks):
        if i > 0 and tr[i - 1][2].any():
            host.reset(np.flatnonzero(tr[i - 1][2]))
        out = host.push(x, tr[i][1], tr[i][2])
        routes["device_eager"](i)
        routes["device_graph"](i)
        assert torch.equal(eager.frames, graphed.frames) and torch.equal(eager.counts, graphed.counts), i
        counts = eager.counts.cpu().numpy()
        want = np.zeros(S, int)
        want[out.slots.numpy()] = out.counts.numpy()
        assert (counts == want).all(), i
        for r, s in enumerate(out.slots.tolist()):
            assert torch.equal(eager.frames[s, :, :counts[s]], out.frames[r, :, :counts[s]]), (i, s)
    assert eager.errors.count_nonzero().item() == 0 and graphed.errors.count_nonzero().item() == 0


def _tail_cost(m, x, warm, n):
    """Stream ms per replayed tick, every slot taking CHUNK samples: no slot ending, and one slot ending (the next
    one restarting) per tick."""
    pool = DevicePyramidPool(m, S, CHUNK)
    g, static = _graph(pool, x)
    full = torch.full((S,), CHUNK, dtype=torch.int32, device="cuda")
    eye = torch.eye(S, dtype=torch.bool, device="cuda")
    none = torch.zeros(S, dtype=torch.bool, device="cuda")
    out = {}
    for name, ends in (("no_end", False), ("one_end", True)):
        def step(i):
            static[0].copy_(full)
            static[1].copy_(eye[i % S] if ends else none)
            static[2].copy_(eye[(i - 1) % S] if ends and i > 0 else none)
            g.replay()
            return 0
        for i in range(2 * S):  # every slot past the pyramid's start-up before the first end
            static[0].copy_(full), static[1].copy_(none), static[2].copy_(none)
            g.replay()
        _, dev, _, _ = _timed(step, warm, n)
        out[name] = round(dev, 4)
    assert pool.errors.count_nonzero().item() == 0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pushes", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=100)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--check-ticks", type=int, default=150)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_device_pyramid_pool needs a CUDA device")
    m = features.CQT2010v2(sr=SR, hop_length=512, n_bins=88, verbose=False).cuda()
    tr = _trace(S, args.warmup + args.pushes, SR, seed=1)  # every route reads a packet from the front of x
    dtr = _device_trace(tr)
    x = torch.randn(S, CHUNK, device="cuda")
    res = {"card": _card(), "slots": S, "T_cap": DevicePyramidPool(m, 1, CHUNK).T_cap,
           "trace": "cfg4 CQT2010v2-88, 22.05 kHz, packets 220-882, 15 % idle, 1 % end + restart per push",
           "runs": []}
    with torch.no_grad():
        _check_equal(m, tr, dtr, x, min(args.check_ticks, len(tr)))
        res["bit_for_bit_ticks"] = min(args.check_ticks, len(tr))
        for run in range(args.runs):
            routes, _ = _routes(m, tr, dtr, x)
            order = list(routes) if run % 2 == 0 else list(routes)[::-1]
            legs, frames = {}, None
            for name in order:
                issue, dev, wall, acc = _timed(routes[name], args.warmup, args.pushes)
                legs[name] = {"issue_ms": round(issue, 4), "stream_ms_per_tick": round(dev, 4), "wall": wall}
                if name == "host":
                    frames = acc
            for leg in legs.values():
                leg["frames_per_s"] = round(frames / leg.pop("wall"))
            res["runs"].append({k: legs[k] for k in routes})
        res["graph_tick_stream_ms"] = _tail_cost(m, x, 20, 200)
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
