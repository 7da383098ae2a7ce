#!/usr/bin/env python
"""Input sample type vs time on one GPU: the six bench.py workloads at their bench shapes, fed the same
seeded waveform as float32, bfloat16 and float16.  The three inputs are timed in alternation (``--reps``
rounds of ``--steps`` forward calls each, CUDA events after warm-up); min / median / max ms per call over
the rounds.  For the workloads on the block-partial kernel (cfg2, stft2048, cfg5, gammatone) a separate
profiled pass reports the tensor-core MMA flops the library executed per call and their rate over the
framed-contraction kernel time (bf16 input: two MMA passes instead of three).  One JSON line, with the
card's name, power limit and maximum SM clock.

    python tools/bench_half_input.py [--workloads cfg2,stft2048,...] [--steps 30] [--reps 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import WORKLOADS  # noqa: E402  (the bench shapes, kept in one place)

DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
BLOCK_PARTIAL = ("cfg2", "stft2048", "cfg5", "gammatone")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def timed(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_half_input.py needs a CUDA device")
    warnings.simplefilter("ignore")
    import nnaudio_b200 as nb
    from nnaudio_b200 import _C

    out = dict(gpu_info(), steps=args.steps, reps=args.reps, workloads={})
    for name in args.workloads.split(","):
        w = WORKLOADS[name]
        mod = getattr(nb.features, w["cls"])(verbose=False, **w["ctor"]).cuda()
        x32 = torch.randn(w["B"], w["L"], generator=torch.Generator().manual_seed(0)).cuda()
        xs = {k: x32.to(dt) for k, dt in DTYPES.items()}
        res = {"desc": w["desc"]}
        with torch.no_grad():
            for k in DTYPES:
                for _ in range(args.warmup):
                    mod(xs[k], **w["fwd"])
            torch.cuda.synchronize()
            times = {k: [] for k in DTYPES}
            for _ in range(args.reps):  # alternate the sample types round by round
                for k in DTYPES:
                    times[k].append(timed(lambda: mod(xs[k], **w["fwd"]), args.steps))
            for k, t in times.items():
                res[k + "_ms"] = {"min": min(t), "median": statistics.median(t), "max": max(t)}
            if name in BLOCK_PARTIAL:
                for k in DTYPES:
                    _C.profile_read()
                    _C.profile_read_exec_flops()
                    _C.profile_enable(True)
                    for _ in range(args.steps):
                        mod(xs[k], **w["fwd"])
                    torch.cuda.synchronize()
                    _C.profile_enable(False)
                    framed_ms, launches = _C.profile_read()
                    flops = _C.profile_read_exec_flops()
                    res[k + "_exec_mma_flops_per_call"] = flops / args.steps
                    res[k + "_framed_kernel_ms_per_call"] = framed_ms / args.steps
                    res[k + "_exec_mma_tflops"] = flops / (framed_ms * 1e-3) / 1e12
        out["workloads"][name] = res
        del xs, x32, mod
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
