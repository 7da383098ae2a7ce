"""PCEN (nnaudio_b200.pcen) on the GPU: kernel time, bandwidth, training and serving cost.

Cases (each timed with CUDA events over many calls after a warm-up; the card's name, power limit and maximum SM
clock are read in the same run):
  offline_cfg2     inference on the cfg2 Mel output shape (64, 128, 431)
  offline_serving  inference on one serving tick's Mel frames (256 slots, 80 mels, the device pool's T_cap)
  train_cfg2       forward + backward of PCEN(trainable=True) per channel on (64, 128, 431), upstream grad given
  long_stream      one stream of an hour of 10 ms frames, (1, 128, 360000): the latency-bound case
  tick_mel / tick_mel_pcen
                   a 256-slot DeviceStreamPool Mel tick (n_fft 512, hop 128, 80 mels, 480-sample packets) captured
                   in one CUDA graph, without and with PCENStream.step on its frames
  torch_loop       a torch frame loop (two element-wise ops per frame for M, then P) on (64, 128, 431), for context
Bandwidth is the bytes the algorithm must move (inference: read E, write P = 8 B per entry; training: 12 B forward
with M, 16 B backward) over kernel time, and its share of the H100 SXM data-sheet 3.35 TB/s.

    python tools/bench_pcen.py [--iters 200] [--out results.json]
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
from bench_stream_pool import _card  # noqa: E402

from nnaudio_b200 import features  # noqa: E402
from nnaudio_b200.pcen import PCEN, PCENStream  # noqa: E402
from nnaudio_b200.streaming import DeviceStreamPool  # noqa: E402

HBM = 3.35e12


def _events(fn, iters, warm=10):
    """Mean ms per fn() over ``iters`` calls, from CUDA events around the whole run."""
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _spectrogram(shape, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(shape, device="cuda", generator=g) ** 4 * 100.0


def _bw(name, ms, nbytes, **extra):
    r = dict(case=name, ms=round(ms, 5), bytes=int(nbytes), tb_s=round(nbytes / (ms * 1e-3) / 1e12, 3),
             share_of_hbm=round(nbytes / (ms * 1e-3) / HBM, 3), **extra)
    print(json.dumps(r), flush=True)
    return r


def torch_loop_pcen(E, s, gain, bias, power, eps):
    """The usual frame loop: one small launch chain per frame."""
    M = torch.empty_like(E)
    m = E[:, :, 0]
    for t in range(E.shape[-1]):
        m = (1 - s) * m + s * E[:, :, t]
        M[:, :, t] = m
    return (bias + E * (eps + M) ** -gain) ** power - bias ** power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_pcen needs a CUDA device"
    card = _card()
    print(json.dumps({"gpu": card}), flush=True)
    res = []
    with torch.no_grad():
        m = PCEN(sr=16000, hop_length=160).cuda()
        E = _spectrogram((64, 128, 431))
        res.append(_bw("offline_cfg2", _events(lambda: m(E), a.iters), 8 * E.numel(), shape=list(E.shape)))

        mel = features.MelSpectrogram(sr=16000, n_fft=512, hop_length=128, n_mels=80, verbose=False).cuda()
        S, chunk = 256, 480
        pool = DeviceStreamPool(mel, S, chunk)
        Es = _spectrogram((S, 80, pool.T_cap), 1)
        m80 = PCEN(n_channels=80, sr=16000, hop_length=128).cuda()
        res.append(_bw("offline_serving", _events(lambda: m80(Es), a.iters), 8 * Es.numel(), shape=list(Es.shape)))

        El = _spectrogram((1, 128, 360_000), 2)
        ms = _events(lambda: m(El), 5, warm=2)
        res.append(_bw("long_stream", ms, 8 * El.numel(), shape=list(El.shape),
                       ns_per_frame=round(ms * 1e6 / El.shape[-1], 3)))

    mt = PCEN(n_channels=128, sr=16000, hop_length=160, trainable=True).cuda()
    Eg = E.clone().requires_grad_(True)
    g = torch.randn_like(E)

    def train():
        Eg.grad = None
        for p in mt.parameters():
            p.grad = None
        mt(Eg).backward(g)

    res.append(_bw("train_cfg2", _events(train, a.iters), 28 * E.numel(), shape=list(E.shape)))

    with torch.no_grad():
        x = torch.randn(S, chunk, device="cuda")
        lengths = torch.full((S,), chunk, dtype=torch.int32, device="cuda")
        end = torch.zeros(S, dtype=torch.bool, device="cuda")
        restart = torch.zeros(S, dtype=torch.bool, device="cuda")
        st = PCENStream(m80, S)
        graphs = {}
        for name, with_pcen in (("tick_mel", False), ("tick_mel_pcen", True)):
            pool.reset(restart), st.reset(restart)
            pool.push(x, lengths, end)
            if with_pcen:
                st.step(pool.frames, pool.counts)
            torch.cuda.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                pool.reset(restart)
                pool.push(x, lengths, end)
                if with_pcen:
                    st.reset(restart)
                    st.step(pool.frames, pool.counts)
            graphs[name] = gr
        ticks = {}
        for rnd in range(2):  # alternate the two graphs, order reversed on the second round
            for name in (sorted(graphs) if rnd == 0 else sorted(graphs, reverse=True)):
                ticks.setdefault(name, []).append(_events(graphs[name].replay, a.iters))
        for name, v in ticks.items():
            r = dict(case=name, ms_per_tick=[round(t, 5) for t in v], slots=S, chunk=chunk)
            print(json.dumps(r), flush=True)
            res.append(r)

        s, gain, bias, power = (float(getattr(m, n)) for n in ("s", "gain", "bias", "power"))
        ms = _events(lambda: torch_loop_pcen(E, s, gain, bias, power, m.eps), 3, warm=1)
        r = dict(case="torch_loop", ms=round(ms, 3), shape=list(E.shape))
        print(json.dumps(r), flush=True)
        res.append(r)
        ref = torch_loop_pcen(E.double(), s, gain, bias, power, m.eps)
        err = float(((m(E).double() - ref).abs().max() / ref.abs().max()).item())
        print(json.dumps({"check": "kernel vs float64 frame loop", "max_rel": err}), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"gpu": card, "results": res}, f, indent=1)


if __name__ == "__main__":
    main()
