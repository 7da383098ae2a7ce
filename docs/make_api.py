#!/usr/bin/env python
"""Regenerates docs/API.md from the live signatures of nnaudio_b200.features."""
import contextlib
import inspect
import io
import os
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nnaudio_b200 as nb  # noqa: E402

REF = {"STFT": "stft.py:66-362", "iSTFT": "stft.py:364-546", "MelSpectrogram": "mel.py:9-194",
       "MFCC": "mel.py:197-329", "Gammatonegram": "gammatone.py:9-194", "CQT1992v2": "cqt.py:561-803",
       "CQT": "cqt.py:1142-1145", "CQT2010v2": "cqt.py:805-1139", "VQT": "vqt.py:9-215",
       "CQT1992": "cqt.py:9-256", "CQT2010": "cqt.py:259-558", "Griffin_Lim": "griffin_lim.py:9-148",
       "Combined_Frequency_Periodicity": "cfp.py:9-246", "CFP": "cfp.py:249-484"}

HEADER = """# API — `nnaudio_b200.features` (generated from the signatures by `python docs/make_api.py`)

Same class names, constructor arguments (names, order, defaults), `forward` signatures, buffer names and public
attributes as `nnAudio.features` v0.3.3 — checked against the unmodified reference by the fixtures in `tests/golden/`
(signatures, buffers bit-identical for 49 + 7 configurations, attribute surface, exception types, outputs ≤1e-4). What differs:

* inputs must be **CUDA float32** tensors on an H100 (sm_90a); anything else raises — there is no CPU fallback;
* exception: a waveform passed to `forward` (every module but `iSTFT` / `Griffin_Lim`, whose inputs are spectrograms)
  may also be **bfloat16 or float16**.  The output is float32 whatever the input dtype, with fp32-grade accuracy on
  the given samples: the result equals that of `x.float()` (on the tensor-core routes bit for bit).  The reference
  raises for a half waveform outside `torch.autocast` and returns half inside it.  Inference reads the 16-bit tensor
  as is; the autograd path upcasts once and returns `x.grad` in the input's dtype;
* multi-GPU: one process per GPU (`nnaudio_b200.parallel.BatchShardedTransform`, INTEGRATION.md) is the fast path;
  `torch.nn.DataParallel`, the reference's own mode, also works (per-device launch attributes and caches);
* `Griffin_Lim.forward(S, rand_phase=None)` takes an optional initial phase (reproducible runs); `device` moves the
  module's buffers at construction, as the reference creates its window there;
* trainable inverse kernels / window of `iSTFT` raise `NotImplementedError` under autograd (no dW path yet);
* `CFP` / `Combined_Frequency_Periodicity` are forward-only (the reference has no parameters there; a waveform that
  requires grad raises `NotImplementedError`); their FFT stages run as dense contractions (DESIGN.md §3.9);
* beyond the reference: `nnaudio_b200.streaming.StreamingTransform(module, batch)` streams live audio chunk by chunk
  through STFT, MelSpectrogram, Gammatonegram, MFCC (`top_db=None`), CQT1992v2 / CQT and CQT1992 (`push(chunk)`,
  `flush()`, `reset()`).  The concatenated outputs equal `module(x)` on the whole stream, bit for bit on the
  tensor-core routes except across the CQT1992v2 kernel's two tile schedules (2e-6; DESIGN.md §3.10).
  `StreamingInverse(istft_module, batch)` does the same for the inverse STFT, to fp32 rounding.
  `StreamPool(module, slots)` serves independent streams of the same modules that advance by their own amounts:
  `push(chunk, lengths, end=None)` gives slot s `chunk[s, :lengths[s]]`, ends the slots flagged in `end` and returns
  a `PoolOutput(frames, slots, counts)` with a row for each slot that has new frames; `reset(slots)` starts new
  streams in some slots while the others carry on.  Each slot's rows equal `module(x)` on its own stream, with the
  rules of `StreamingTransform`.
  `InversePool(istft_module, slots, onesided=None)` does the same for the inverse STFT: `push(X, slots, counts,
  end=None, length=None)` appends `X[r, :, :counts[r]]` to slot `slots[r]`, ends the flagged slots with the
  `StreamingInverse.flush` rules and returns an `InverseOutput(samples, slots, counts)`; a `PoolOutput` of
  `StreamPool` feeds it as is.  Each slot's samples equal `StreamingInverse` on its own frames, to fp32 rounding.
  `DeviceStreamPool(module, slots, chunk, dtype=torch.float32)` and `DeviceInversePool(istft_module, slots, frames,
  onesided=None)` are `StreamPool` and `InversePool` with their counters, lengths and end flags on the GPU: `push(x,
  lengths, end)` / `push(X, counts, end, length)` take device tensors, overwrite the pool-owned `frames` / `samples`
  and `counts` (row s = slot s, `T_cap` / `n_cap` wide) and read nothing on the host, so a tick can be captured in a
  CUDA graph; `reset(restart=None)` takes a device mask, and `check()` raises what the host pool would have raised
  for a dropped slot (DESIGN.md §3.10 "Device pools").
  `StreamingPyramid(module, batch)` streams the CQT pyramid of `CQT2010v2` / `VQT` / `CQT2010` bit for bit on the
  whole-clip call's tensor-core plan (DESIGN.md §3.10).
  `PyramidPool(module, slots)` serves independent pyramid streams with `StreamPool`'s `push(chunk, lengths, end)` /
  `reset(slots)` surface: each slot's rows equal `module(x)` on its own stream bit for bit, and a one-stream
  `StreamingPyramid` fed the same packets.
  `DevicePyramidPool(module, slots, chunk, dtype=torch.float32)` is `PyramidPool` with `DeviceStreamPool`'s surface:
  device `lengths` / `end`, the pool-owned `frames` (slots, n_bins, `T_cap`[, 2]) and `counts`, `reset(restart=None)`
  and `check()`, so a pyramid tick can be captured in a CUDA graph.  A push never sees the lengths on the host, so it
  cannot issue `module(x)`'s reflect-fallback `UserWarning` for a short stream (DESIGN.md §3.10 "Device pyramid
  pools").
  `nnaudio_b200.pcen.PCEN(n_channels=None, sr=22050, hop_length=512, time_constant=0.4, s=None, gain=0.98,
  bias=2.0, power=0.5, eps=1e-6, trainable=False)` is per-channel energy normalisation of a `(B, C, T)` spectrogram:
  one launch per call, a fused backward for the input and the (scalar or per-channel) parameters, which are buffers
  or, with `trainable=True`, parameters.  `PCENStream(pcen, slots)` carries each stream's smoother across
  `step(frames, counts=None, slots=None)` calls on the output of `StreamingTransform`, a `StreamPool` `PoolOutput` or
  a `DeviceStreamPool`, bit for bit with the whole-clip call, with `reset(restart=None)` on a device mask
  (DESIGN.md §3.11).

Environment switches: `NNAUDIO_B200_PATH=auto|simt|tc` (kernel family), `NNAB_TALL_BALANCE=0|1` (balanced tile
schedule of the CQT1992v2 kernel).

"""


def main():
    out = io.StringIO()
    out.write(HEADER)
    for name, where in REF.items():
        cls = getattr(nb.features, name)
        out.write(f"## `{name}`  — reference `{where}`\n\n```python\n")
        out.write(f"{name}{str(inspect.signature(cls.__init__)).replace('(self, ', '(')}\n")
        for meth in ("forward", "inverse"):
            if meth == "inverse" and meth not in cls.__dict__:
                continue
            out.write(f".{meth}{str(inspect.signature(getattr(cls, meth))).replace('(self, ', '(')}\n")
        out.write("```\n\n")
        doc = inspect.getdoc(cls) or ""
        if doc:
            out.write(doc.split("\n\n")[0].replace("\n", " ") + "\n\n")
        kw = {"Griffin_Lim": dict(n_fft=512)}.get(name, {})
        if "verbose" in inspect.signature(cls.__init__).parameters:
            kw["verbose"] = False
        try:
            with contextlib.redirect_stdout(io.StringIO()), warnings.catch_warnings():
                warnings.simplefilter("ignore")
                mod = cls(**kw)
            bufs = ", ".join(f"`{k}` {tuple(v.shape)}" for k, v in mod.state_dict().items())
            out.write(f"state_dict (defaults): {bufs or '—'}\n\n")
        except ValueError as e:  # CQT1992's own defaults exceed Nyquist, in the reference too
            out.write(f"(the default arguments do not construct, as in the reference: {str(e).split(',')[0]})\n\n")
    with open(os.path.join(ROOT, "docs", "API.md"), "w") as f:
        f.write(out.getvalue())


if __name__ == "__main__":
    main()
