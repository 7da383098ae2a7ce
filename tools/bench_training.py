#!/usr/bin/env python
"""Timing of the training / inverse paths (SURVEY §8f next #1 / #2) at BASELINE-shaped sizes:
forward only, forward+backward w.r.t. the waveform, forward+backward w.r.t. trainable kernels,
and the inverse STFT.  CUDA events on the current stream, 3 warm-up + N timed iterations,
three rotating inputs (> L2).  Prints one JSON line per measurement.  Not the headline metric
(bench.py is); this documents that the gradients run on the same tensor-core kernel.

    python tools/bench_training.py [--iters 10]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nnaudio_b200 as nb  # noqa: E402


def timed(fn, inputs, iters, warmup=3):
    for i in range(warmup):
        fn(inputs[i % len(inputs)])
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(iters):
        fn(inputs[i % len(inputs)])
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--only", choices=["all", "mel", "cqt"], default="all")
    args = ap.parse_args()
    dev = "cuda"
    out = []

    def report(name, ms, frames, **extra):
        line = dict(case=name, ms_per_step=round(ms, 4), frames_per_s=round(frames / ms * 1e3), **extra)
        out.append(line)
        print(json.dumps(line), flush=True)

    if args.only in ("all", "mel"):
        _mel_and_inverse(args, dev, report)
    if args.only in ("all", "cqt"):
        _pyramid(args, dev, report)
    print(json.dumps(out, indent=1))


def _mel_and_inverse(args, dev, report):
    # ---- cfg2-shaped MelSpectrogram: 64 x 10 s @ 22.05 kHz --------------------------------
    B, L = 64, 220500
    xs = [torch.randn(B, L, device=dev) for _ in range(3)]
    mel = nb.MelSpectrogram(sr=22050, n_fft=2048, hop_length=512, n_mels=128, verbose=False).to(dev)
    T = L // 512 + 1
    with torch.no_grad():
        report("mel_cfg2_forward_fused", timed(lambda x: mel(x), xs, args.iters), B * T)

    def fwd_bwd_input(x):
        x = x.detach().requires_grad_(True)
        mel(x).sum().backward()

    report("mel_cfg2_forward_backward_dX", timed(fwd_bwd_input, xs, args.iters), B * T)

    mel_t = nb.MelSpectrogram(sr=22050, n_fft=2048, hop_length=512, n_mels=128, trainable_mel=True,
                              trainable_STFT=True, verbose=False).to(dev)

    def fwd_bwd_weights(x):
        mel_t.zero_grad(set_to_none=True)
        mel_t(x).sum().backward()

    report("mel_cfg2_forward_backward_dW", timed(fwd_bwd_weights, xs, args.iters), B * T,
           note="trainable_mel + trainable_STFT: dW of both Fourier kernels and the filterbank")

    # ---- STFT -> inverse round trip (cfg2 shape) ----------------------------------------------
    st = nb.STFT(n_fft=2048, hop_length=512, iSTFT=True, output_format="Complex", verbose=False).to(dev)
    with torch.no_grad():
        Xs = [st(x) for x in xs]
        report("istft_cfg2_inverse", timed(lambda X: st.inverse(X, onesided=True, length=L), Xs, args.iters),
               B * T)
    del Xs



def _pyramid(args, dev, report):
    # ---- CQT2010v2 pyramid, 32 x 30 s --------------------------------------------------------
    Bc, Lc = 32, 661500
    xc = [torch.randn(Bc, Lc, device=dev) for _ in range(3)]
    cqt = nb.CQT2010v2(sr=22050, hop_length=512, n_bins=84, verbose=False).to(dev)
    Tc = Lc // 512 + 1
    with torch.no_grad():
        report("cqt2010v2_forward_fused", timed(lambda x: cqt(x), xc, args.iters), Bc * Tc)

    def cqt_bwd(x):
        x = x.detach().requires_grad_(True)
        cqt(x).sum().backward()

    report("cqt2010v2_forward_backward_dX", timed(cqt_bwd, xc, args.iters), Bc * Tc,
           note="octave-by-octave training path (7 octaves, 6 FIR stages); decimation adjoint via "
                + os.environ.get("NNAUDIO_B200_DECIM_BWD", "simt"))


if __name__ == "__main__":
    main()
