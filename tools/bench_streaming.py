"""Per-push cost of nnaudio_b200.streaming against two baselines.

For each case, per push: host issue time (the push call, no synchronisation), median issue-to-complete
latency (push + synchronise), device time per push over many pushes (CUDA events), frames/s.  Baselines:
  offline  the module's offline forward on one push's frames (a clip of (T - 1) * hop + K samples,
           center=False), i.e. the launches a push cannot avoid
  concat   the concat route (carried samples + chunk with torch, then the offline call)
The STFT -> iSTFT case pushes each chunk through the streamed STFT and its frames through the streamed inverse
(the offline baseline: STFT of one push's clip, then the offline inverse of its frames).  The pyramid case
(cfg4-like: CQT2010v2, 88 bins, 64 streams, 100 ms pushes) streams through StreamingPyramid; its offline baseline
is the whole-clip call on a clip giving one push's frames (the pyramid has no concat route).

    python tools/bench_streaming.py [--pushes 400] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nnaudio_b200 import _C, features  # noqa: E402
from nnaudio_b200.streaming import StreamingInverse, StreamingPyramid, StreamingTransform  # noqa: E402

CASES = {
    "stft1024_1x256": (lambda: features.STFT(n_fft=1024, hop_length=256, verbose=False), 1, 256),
    "mel16k_256x20ms": (lambda: features.MelSpectrogram(sr=16000, n_fft=512, hop_length=128, n_mels=80,
                                                        verbose=False), 256, 320),
    "cqt44k_1x512": (lambda: features.CQT1992v2(sr=44100, n_bins=84, bins_per_octave=12, fmin=32.7,
                                                verbose=False), 1, 512),
    "stft_istft_1x256": (lambda: features.STFT(n_fft=1024, hop_length=256, output_format="Complex", iSTFT=True,
                                               verbose=False), 1, 256),
}


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the measurement itself needs no nvidia-smi
        return f"unknown ({e})"


def _measure(fn, x, chunk, pushes):
    """fn(chunk tensor) per push -> host issue ms, median latency ms, device ms per push."""
    L = x.shape[1]
    for i in range(20):  # warm-up: every shape the timed window uses
        fn(x[:, (i * chunk) % (L - chunk):][:, :chunk])
    torch.cuda.synchronize()
    issue, lat = [], []
    for i in range(50):
        c = x[:, (i * chunk) % (L - chunk):][:, :chunk]
        t0 = time.perf_counter()
        fn(c)
        t1 = time.perf_counter()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        issue.append((t1 - t0) * 1e3)
        lat.append((t2 - t0) * 1e3)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(pushes):
        fn(x[:, (i * chunk) % (L - chunk):][:, :chunk])
    e1.record()
    torch.cuda.synchronize()
    return statistics.median(issue), statistics.median(lat), e0.elapsed_time(e1) / pushes


def _pyramid_row(pushes):
    """cfg4-like pyramid: 64 streams, 100 ms pushes at 22.05 kHz."""
    m = features.CQT2010v2(sr=22050, hop_length=512, n_bins=88, verbose=False).cuda()
    B, chunk = 64, 2205
    x = torch.randn(B, 200 * chunk + 8192, device="cuda")
    with torch.no_grad():
        st = StreamingPyramid(m, B)
        row = {"batch": B, "chunk": chunk, "fused": _measure(st.push, x, chunk, pushes)}
        T = max(1, round(chunk / st.hop))
        clip = x[:, :T * st.hop - 1].contiguous()  # T frames in every octave
        row["offline"] = _measure(lambda c: m(clip), x, chunk, pushes)
    for k in ("fused", "offline"):
        issue, lat, dev = row[k]
        row[k] = {"issue_ms": round(issue, 4), "latency_ms": round(lat, 4), "device_ms": round(dev, 4),
                  "frames_per_s": round(B * chunk / st.hop / (dev * 1e-3))}
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pushes", type=int, default=400)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_streaming needs a CUDA device")
    res = {"card": _card(), "cases": {}}
    for name, (make, B, chunk) in CASES.items():
        m = make().cuda()
        x = torch.randn(B, 200 * chunk + 8192, device="cuda")
        with torch.no_grad():
            st = StreamingTransform(m, B, _strict=True)
            frames_per_push = chunk / st.hop

            inverse = name == "stft_istft_1x256"
            ist = StreamingInverse(m, B) if inverse else None

            def fused(c):
                X = st.push(c)
                if inverse:
                    ist.push(X)

            row = {"batch": B, "chunk": chunk}
            row["fused"] = _measure(fused, x, chunk, args.pushes)
            T = max(1, round(frames_per_push))
            clip = x[:, :(T - 1) * st.hop + st.K].contiguous()
            kw_name, kw = st._args()
            off = getattr(_C, kw_name)
            if inverse:
                row["offline"] = _measure(lambda c: m.inverse(off(clip, **dict(kw, center=False)), length=chunk),
                                          x, chunk, args.pushes)
            else:
                row["offline"] = _measure(lambda c: off(clip, **dict(kw, center=False)), x, chunk, args.pushes)
            chunk_fn = kw_name.replace("_forward", "_chunk_forward")
            saved = getattr(_C, chunk_fn)
            setattr(_C, chunk_fn, lambda *a, **k: None)  # every push takes the concat route
            try:
                st2 = StreamingTransform(m, B)
                ist2 = StreamingInverse(m, B) if inverse else None
                row["concat"] = _measure(lambda c: ist2.push(st2.push(c)) if inverse else st2.push(c), x, chunk,
                                         args.pushes)
            finally:
                setattr(_C, chunk_fn, saved)
            for k in ("fused", "offline", "concat"):
                issue, lat, dev = row[k]
                row[k] = {"issue_ms": round(issue, 4), "latency_ms": round(lat, 4), "device_ms": round(dev, 4),
                          "frames_per_s": round(B * frames_per_push / (dev * 1e-3))}
        res["cases"][name] = row
        print(name, json.dumps(row), flush=True)
    row = _pyramid_row(args.pushes)
    res["cases"]["pyramid_cfg4_64x100ms"] = row
    print("pyramid_cfg4_64x100ms", json.dumps(row), flush=True)
    print(json.dumps({"card": res["card"]}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
