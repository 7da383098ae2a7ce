"""Chunk-by-chunk streaming through the forward transforms and the inverse STFT (DESIGN.md §3.10).

``StreamingTransform(module, batch)`` runs ``batch`` streams that advance together.  Each ``push(chunk)``
returns every frame whose samples have all arrived; ``flush()`` returns the rest, with the module's right
padding.  Concatenated along time, the outputs equal ``module(x)`` on the whole stream: same frame count,
same reflect / constant padding at both ends, bit for bit on the tensor-core routes (for a 16-bit stream:
bit for bit ``module(x.float())``).  One exception: the CQT1992v2 tall kernel picks its balanced tile schedule
from a launch's tile count, so a whole-clip call on that schedule and pushes on the static one agree to 2e-6.

Each push is one C call on the offline kernels (``_C.*_chunk_forward``): the tensor-core pre-pass builds its
bf16 planes from the carried fp32 samples and the new chunk.  Plans that read the waveform as fp32 directly
(the SIMT kernels, ``NNAUDIO_B200_PATH=simt``) take the concat route instead: the carried samples and the
upcast chunk, padded and concatenated with torch, through the module's offline call with ``center=False``.
A push never reads the device back or synchronises.

``StreamPool(module, slots)`` serves independent streams that advance by their own amounts: each
``push(chunk, lengths, end)`` appends ``chunk[s, :lengths[s]]`` to slot ``s``'s stream, ends the streams
flagged in ``end``, and returns the new frames of the slots that have some; ``reset(slots)`` starts new streams
in some slots while the others carry on.  Each stream's frames are those of ``StreamingTransform``.

``StreamingPyramid(module, batch)`` streams through the ÷2 resampling pyramid of ``CQT2010v2``, ``VQT`` and
``CQT2010`` on the whole-clip call's tensor-core plan: each push returns the frames final in every octave.

``PyramidPool(module, slots)`` is ``StreamPool`` for the pyramids: independent streams with ragged pushes, each
slot's frames those of a one-stream ``StreamingPyramid``.

``StreamingInverse(module, batch)`` streams complex frames through the inverse STFT: each push returns the
output samples no later frame can change, ``flush(length=None)`` the rest.

``InversePool(module, slots)`` is ``StreamPool``'s counterpart for the inverse STFT: each
``push(X, slots, counts, end, length)`` appends ``X[r, :, :counts[r]]`` to slot ``slots[r]``'s stream and ends the
flagged slots; a ``PoolOutput`` of ``StreamPool`` feeds it as is.

``DeviceStreamPool``, ``DevicePyramidPool`` and ``DeviceInversePool`` are ``StreamPool``, ``PyramidPool`` and
``InversePool`` with their counters, lengths and end flags on the GPU and one fixed geometry per push, so a serving
tick can be captured in a CUDA graph.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np
import torch

from . import _C
from .features.cqt import (CQT1992v2, CQT2010v2, _check_format_and_norm, _pyramid_args, _pyramid_length_plan,
                           _v2_normalization)
from .features.cqt_v1 import CQT1992, CQT2010
from .features.gammatone import Gammatonegram
from .features.mel import MFCC, MelSpectrogram
from .features.stft import STFT, _inverse_args, iSTFT
from .features.vqt import VQT

__all__ = ["StreamingTransform", "StreamPool", "PoolOutput", "StreamingPyramid", "PyramidPool", "StreamingInverse",
           "InversePool", "InverseOutput", "DeviceStreamPool", "DevicePyramidPool", "DeviceInversePool"]

_SUPPORTED = (STFT, MelSpectrogram, Gammatonegram, MFCC, CQT1992v2, CQT1992)
_PYRAMIDS = (CQT2010v2, VQT, CQT2010)


def _ready_frames(total, K, hop, pad, reflect):
    """Frames whose raw samples have all arrived after ``total`` samples: frame t reads up to raw sample
    t * hop + K - pad - 1, and with reflect padding frame 0 also mirrors raw sample ``pad``."""
    if reflect and total < pad + 1:
        return 0
    need = K - pad
    return 0 if total < need else (total - need) // hop + 1


def _carry_start(total, frames, hop, pad):
    """First raw sample the next push reads (the carry ring holds [start, total))."""
    s = frames * hop - pad
    if pad > 0:
        s = min(s, total - (pad + 1))  # the right mirror of the last push reads pad + 1 samples back
    return min(max(s, 0), total)


def _streams(v, what):
    """``batch`` / ``slots`` of a constructor: how many streams one C call may carry."""
    v = int(v)
    if v < 1 or v > _C.MAX_BATCH:
        raise ValueError(f"{what} must be in [1, {_C.MAX_BATCH}], got {v}")
    return v


def _check_chunk(chunk, rows, dtype, where="within a stream", width=None):
    """The checks of a push's chunk: a (rows, n) tensor without grad in a sample type the forward calls read, the
    same as ``dtype`` (the stream's or the pool's, ``where``) once that is set.  A device pool fixes the width and
    the sample type (``width``, ``dtype``)."""
    if not isinstance(chunk, torch.Tensor):
        raise TypeError("chunk must be a torch.Tensor")
    if chunk.requires_grad:
        raise NotImplementedError("the streaming API is forward-only: the chunk requires grad")
    if chunk.dim() != 2 or chunk.shape[0] != rows or (width is not None and chunk.shape[1] != width):
        raise ValueError(f"chunk must be ({rows}, {'n' if width is None else width}), got {tuple(chunk.shape)}")
    if width is not None:
        if chunk.dtype != dtype:
            raise ValueError(f"chunk must be {dtype} (the pool's sample type), got {chunk.dtype}")
        return
    if chunk.dtype not in _C._WAVE_DTYPES:
        raise ValueError(f"chunk must be float32, bfloat16 or float16, got {chunk.dtype}")
    if dtype is not None and chunk.dtype != dtype:
        raise ValueError(f"chunk dtype changed from {dtype} to {chunk.dtype} {where}")


def _for_slot(s, check, *args):
    """``check(*args)``, re-raising what it raises with slot ``s`` named."""
    try:
        return check(*args)
    except Exception as e:
        raise type(e)(f"slot {s}: {e}") from None


def _cpu_ints(v, what, n=None, kind="integers"):
    """A CPU array of ints (or bools, kind="bools") of shape (n,); device tensors are refused, since reading
    them would synchronise."""
    if isinstance(v, torch.Tensor):
        if v.device.type != "cpu":
            raise TypeError(f"{what} must be on the CPU: reading it from {v.device} would synchronise")
        v = v.numpy()
    a = np.asarray(v)
    if n is not None and a.shape != (n,):
        raise ValueError(f"{what} must hold {n} values, got shape {a.shape}")
    if a.ndim != 1:
        raise ValueError(f"{what} must be one-dimensional, got shape {a.shape}")
    if kind == "integers" and a.dtype != bool and (np.issubdtype(a.dtype, np.integer) or a.size == 0):
        return a.astype(np.int64)
    if kind == "bools" and (a.dtype == bool or (np.issubdtype(a.dtype, np.integer) and np.isin(a, (0, 1)).all())):
        return a.astype(bool)
    raise TypeError(f"{what} must be {kind}, got {a.dtype}")


def _ended_error(s):
    return RuntimeError(f"slot {s}: its stream has ended; call reset([{s}]) to start a new one")


class StreamingTransform:
    """Stream ``batch`` signals chunk by chunk through ``module``.

    ``module``: ``STFT``, ``MelSpectrogram``, ``Gammatonegram``, ``MFCC`` (``top_db=None`` only),
    ``CQT1992v2`` / ``CQT`` or ``CQT1992``.  ``forward_kwargs`` are passed on as the module's ``forward``
    keywords (``output_format``, ``normalization_type``).
    """

    def __init__(self, module, batch, _strict=False, **forward_kwargs):
        if not isinstance(module, _SUPPORTED):
            raise TypeError(
                f"StreamingTransform supports STFT, MelSpectrogram, Gammatonegram, MFCC, CQT1992v2 / CQT and "
                f"CQT1992, not {type(module).__name__}"
                + (": stream the CQT2010 pyramids with StreamingPyramid" if isinstance(module, _PYRAMIDS) else "")
            )
        if isinstance(module, MFCC) and module.top_db is not None:
            raise ValueError(
                "MFCC with top_db set cannot be streamed: its floor is a maximum over the whole clip. "
                "Build the module with top_db=None."
            )
        batch = _streams(batch, "batch")
        self.module, self.batch, self._strict = module, batch, bool(_strict)
        if isinstance(module, (CQT1992v2, CQT1992)):
            fmt = forward_kwargs.get("output_format") or module.output_format
            norm = forward_kwargs.get("normalization_type", "librosa")
            self._args = lambda: module._infer_args(fmt, norm)
            self._check_length = lambda n: module._check_length(self.batch, n)
            self.K = module.kernel_width
        else:
            stft = module.melspec_layer.stft if isinstance(module, MFCC) else (
                module if isinstance(module, STFT) else module.stft)
            if isinstance(module, STFT):
                fmt = forward_kwargs.get("output_format") or module.output_format
                self._args = lambda: module._infer_args(fmt)
            else:
                self._args = module._infer_args
            self._check_length = stft._check_length
            self.K = stft.n_fft
        name, kw = self._args()
        self.hop = kw["hop"]
        self.pad = self.K // 2 if kw["center"] else 0
        self._reflect = self.pad > 0 and kw["pad_mode"] == _C.PAD_REFLECT
        device = next(iter(module.buffers())).device
        self.ring = torch.empty((batch, self.K), dtype=torch.float32, device=device)  # carried raw samples
        self.reset()

    def reset(self):
        """Start new streams (same module, same batch)."""
        self.received = self.n_carry = self.frames = 0
        self.dtype = None
        self._flushed = False

    # ------------------------------------------------------------------------------------------------ #
    def push(self, chunk: torch.Tensor) -> torch.Tensor:
        """Feed ``chunk`` (batch, n), any n >= 0; returns the frames completed by it."""
        if self._flushed:
            raise RuntimeError("push() after flush(): call reset() to start new streams")
        _check_chunk(chunk, self.batch, self.dtype)
        self.dtype = chunk.dtype
        n = chunk.shape[1]
        T = _ready_frames(self.received + n, self.K, self.hop, self.pad, self._reflect) - self.frames
        return self._advance(chunk, n, False, T)

    def flush(self) -> torch.Tensor:
        """End of stream: the remaining frames, with the module's right padding."""
        if self._flushed:
            raise RuntimeError("flush() after flush(): call reset() to start new streams")
        self._check_length(self.received)  # the exception module(x) raises for a stream this short
        if self.dtype is None:
            self.dtype = torch.float32
        T = (self.received + 2 * self.pad - self.K) // self.hop + 1 - self.frames
        out = self._advance(None, 0, True, T)
        self._flushed = True
        return out

    # ------------------------------------------------------------------------------------------------ #
    def _advance(self, chunk, n, flush, T):
        name, kw = self._args()
        out = getattr(_C, name.replace("_forward", "_chunk_forward"))(self, chunk, flush, T, **kw)
        if out is None:
            if self._strict:
                raise RuntimeError(f"{name}: no fused chunk route for this configuration (NNAB_EUNSUPPORTED)")
            out = self._concat_route(chunk, n, flush, T, name, kw)
        total = self.received + n
        self.received, self.frames = total, self.frames + T
        self.n_carry = total - _carry_start(total, self.frames, self.hop, self.pad)
        return out

    def _concat_route(self, chunk, n, flush, T, name, kw):
        """The push on the module's offline call: the virtual clip (carried samples, chunk, the stream's
        padding at its ends) built with torch, framed with center=False; then the carry ring update."""
        R, K, dev = self.received, self.K, self.ring.device
        total = R + n
        x = chunk.float() if n > 0 else self.ring[:, :0]
        out = None
        if T > 0:
            origin = self.frames * self.hop - self.pad
            r = torch.arange(origin, origin + (T - 1) * self.hop + K, device=dev)
            if self._reflect:
                r = torch.where(r < 0, -r, r)
                if flush:
                    r = torch.where(r >= total, 2 * (total - 1) - r, r)
            live = (r >= 0) & (r < total)
            rc = r.clamp(0, max(total - 1, 0))
            v = self.ring[:, rc % K]
            if n > 0:
                v = torch.where(rc < R, v, x[:, (rc - R).clamp(0, n - 1)])
            v = torch.where(live, v, torch.zeros((), device=dev))
            out = getattr(_C, name)(v, **dict(kw, center=False))
        keep = max(_carry_start(total, self.frames + T, self.hop, self.pad), R)
        if keep < total:
            idx = torch.arange(keep, total, device=dev)
            self.ring[:, idx % K] = x[:, idx - R]
        return out if out is not None else self._empty(name, kw)

    def _empty(self, name, kw):
        """The offline call's output layout with no frame."""
        return torch.empty(_C._SPECS[name].shape(self.batch, 0, kw), device=self.ring.device)


class PoolOutput(NamedTuple):
    """One ``StreamPool.push``: row i of ``frames`` (offline layout, batch = A, T_max frames) holds the new
    frames of slot ``slots[i]``, ``counts[i]`` of them; frames t >= counts[i] are exact zeros.  ``slots``
    (ascending) and ``counts`` are int64 CPU tensors."""
    frames: torch.Tensor
    slots: torch.Tensor
    counts: torch.Tensor


class _HostPool:
    """What the host-planned pools share: the per-slot counters (``_COUNTERS``) and ended flags, kept on the host,
    and their reset."""
    _COUNTERS = ("received", "frames")

    def _init_slots(self, slots):
        self.slots = slots
        for name in self._COUNTERS:
            setattr(self, name, np.zeros(slots, np.int64))  # host counters of every slot's stream
        self.ended = np.zeros(slots, bool)

    def reset(self, slots=None):
        """Start new streams in ``slots`` (all slots by default; then a chunk pool's sample type is free again)."""
        if slots is None:
            idx = np.arange(self.slots)
            if hasattr(self, "dtype"):
                self.dtype = None
        else:
            idx = _cpu_ints(np.reshape(slots.cpu() if isinstance(slots, torch.Tensor) else slots, -1), "slots")
            if ((idx < 0) | (idx >= self.slots)).any():
                raise ValueError(f"slots must be in [0, {self.slots}), got {idx.tolist()}")
        for name in self._COUNTERS:
            getattr(self, name)[idx] = 0
        self.ended[idx] = False

    def _refuse_ended(self, new, end):
        bad = np.flatnonzero(self.ended & (new | end))
        if len(bad):
            raise _ended_error(bad[0])


class _ChunkPool(_HostPool):
    """The push of the waveform pools (``StreamPool``, ``PyramidPool``): argument checks, the lane table, the
    counter commit.  A pool supplies ``_lane_counts`` (its counting rules) and ``_advance`` (the C call)."""

    def push(self, chunk: torch.Tensor, lengths, end=None) -> PoolOutput:
        """Append ``chunk[s, :lengths[s]]`` to every slot s, end the slots flagged in ``end``; returns the new
        frames of the slots that have some."""
        _check_chunk(chunk, self.slots, self.dtype, "within the pool")
        n = chunk.shape[1]
        lengths = _cpu_ints(lengths, "lengths", self.slots)
        end = np.zeros(self.slots, bool) if end is None else _cpu_ints(end, "end", self.slots, "bools")
        bad = np.flatnonzero((lengths < 0) | (lengths > n))
        if len(bad):
            raise ValueError(f"lengths must be in [0, {n}] (the chunk width): slot {bad[0]} has {lengths[bad[0]]}")
        self._refuse_ended(lengths > 0, end)
        active = np.flatnonzero((lengths > 0) | end)
        count, n_carry = self._lane_counts(active, lengths, end)
        order = np.lexsort((active, count == 0))  # the lanes with frames first, slots ascending in each group
        active, count, n_carry = active[order], count[order], n_carry[order]
        A = int((count > 0).sum())
        T_max = int(count.max()) if A else 0
        lanes = np.stack([active, self.received[active], n_carry, self.frames[active], lengths[active],
                          end[active].astype(np.int64)], 1).astype(np.int64)
        out = self._advance(chunk, lanes, A, T_max, count)
        # committed once the push has run: a refused push leaves the pool as it was
        self.dtype = chunk.dtype
        self.received[active] += lengths[active]
        self.frames[active] += count
        self.ended[active] |= end[active]
        return PoolOutput(out, torch.from_numpy(active[:A].copy()), torch.from_numpy(count[:A].copy()))


class StreamPool(_ChunkPool):
    """Serve up to ``slots`` independent streams through ``module``, each advancing by its own amount.

    ``push(chunk, lengths, end=None)``: ``chunk`` is a (slots, n) CUDA float32 / bfloat16 / float16 tensor and
    slot s takes ``chunk[s, :lengths[s]]`` (``lengths``: CPU integers, 0 <= lengths[s] <= n).  ``end[s]`` (CPU
    bools) makes this push the last of slot s's stream: it gets its remaining frames with the module's right
    padding, as ``StreamingTransform.flush`` would give them, and takes no more samples until ``reset([s])``.
    Returns a ``PoolOutput`` with a row for each slot that has new frames.  Concatenated along time, a slot's
    rows up to their counts equal ``module(x)`` on its whole stream, bit for bit on the tensor-core routes (the
    rules and the one CQT1992v2 exception of ``StreamingTransform``).  Every argument is checked before anything
    is enqueued, and a push never reads the device back or synchronises.  ``module`` and ``forward_kwargs``:
    those of ``StreamingTransform``; the pool's sample type is fixed by its first push.

    A push is one C call (``_C.*_pool_forward``): the offline plan on the A slots with new frames, each row's
    virtual clip built by the pre-pass from its own carry ring row and chunk row, the batch's clips all as long
    as the longest; then the zeroing of each row's frames past its count and the carry of every slot that
    received samples.  Idle slots cost nothing.  Plans that read the waveform as fp32 directly (the SIMT
    kernels) take the concat route, as in ``StreamingTransform``.
    """

    def __init__(self, module, slots, _strict=False, **forward_kwargs):
        slots = _streams(slots, "slots")
        # module checks, the offline call's arguments and the (slots, K) fp32 carry ring: StreamingTransform's
        self._st = st = StreamingTransform(module, slots, _strict=_strict, **forward_kwargs)
        self.module, self._strict = module, bool(_strict)
        self.K, self.hop, self.pad, self._reflect = st.K, st.hop, st.pad, st._reflect
        self.ring = st.ring
        self._init_slots(slots)
        self.dtype = None

    def _lane_counts(self, active, lengths, end):
        """Every lane's frame count and carried samples, by the rules of StreamingTransform (push / flush)."""
        K, hop, pad = self.K, self.hop, self.pad
        count = np.zeros(len(active), np.int64)
        n_carry = np.zeros(len(active), np.int64)
        for j, s in enumerate(active.tolist()):
            R, F0 = int(self.received[s]), int(self.frames[s])
            total = R + int(lengths[s])
            if end[s]:
                _for_slot(s, self._st._check_length, total)  # the exception module(x) raises for a stream this short
                count[j] = (total + 2 * pad - K) // hop + 1 - F0
            else:
                count[j] = _ready_frames(total, K, hop, pad, self._reflect) - F0
            n_carry[j] = R - _carry_start(R, F0, hop, pad)
        return count, n_carry

    # ------------------------------------------------------------------------------------------------ #
    def _advance(self, chunk, lanes, A, T_max, count):
        name, kw = self._st._args()
        out = getattr(_C, name.replace("_forward", "_pool_forward"))(self, lanes, chunk, A, T_max, **kw)
        if out is None:
            if self._strict:
                raise RuntimeError(f"{name}: no fused pool route for this configuration (NNAB_EUNSUPPORTED)")
            out = self._concat_route(chunk, lanes, A, T_max, count, name, kw)
        return out

    def _concat_route(self, chunk, lanes, A, T_max, count, name, kw):
        """The push on the module's offline call: every row's virtual clip gathered with torch from its ring
        row and chunk row (one index gather), framed with center=False, the frames past each row's count
        zeroed; then the carry ring update."""
        K, hop, pad, dev = self.K, self.hop, self.pad, self.ring.device
        x = chunk.float() if chunk.shape[1] > 0 else self.ring[:, :0]
        out = self._st._empty(name, kw)[:0]
        if A > 0:
            lt = torch.as_tensor(lanes[:A]).to(dev)
            slot, R, frm, end = lt[:, 0:1], lt[:, 1:2], lt[:, 3:4], lt[:, 5:6] > 0
            total = R + lt[:, 4:5]
            Lv = (T_max - 1) * hop + K
            r = frm * hop - pad + torch.arange(Lv, device=dev)[None]
            if self._reflect:
                r = torch.where(r < 0, -r, r)
                r = torch.where(end & (r >= total) & (r < total + pad), 2 * (total - 1) - r, r)
            live = (r >= 0) & (r < total)
            src = torch.cat([self.ring[slot[:, 0]], x[slot[:, 0]]], 1)  # (A, K + n): ring row, then chunk row
            idx = torch.where(r < R, r.remainder(K), K + r - R).clamp(0, src.shape[1] - 1)
            v = torch.where(live, torch.gather(src, 1, idx), torch.zeros((), device=dev))
            out = getattr(_C, name)(v, **dict(kw, center=False))
            keep = torch.arange(T_max, device=dev)[None] < torch.as_tensor(count[:A]).to(dev)[:, None]
            keep = keep[:, None, :, None] if out.dim() == 4 else keep[:, None, :]
            out = out.masked_fill(~keep, 0.0)
        rows, raw, pos = [np.zeros(0, np.int64)], [np.zeros(0, np.int64)], [np.zeros(0, np.int64)]
        for (s, R, _, F0, m, _), T in zip(lanes.tolist(), count.tolist()):
            r = np.arange(max(_carry_start(R + m, F0 + T, hop, pad), R), R + m)  # what the slot's ring keeps
            rows.append(np.full(len(r), s))
            raw.append(r)
            pos.append(r - R)
        rows, raw, pos = (torch.as_tensor(np.concatenate(a)).to(dev) for a in (rows, raw, pos))
        if rows.numel():
            self.ring[rows, raw.remainder(K)] = x[rows, pos]
        return out


class StreamingPyramid:
    """Stream ``batch`` signals chunk by chunk through the CQT pyramid of ``CQT2010v2``, ``VQT`` or ``CQT2010``.

    ``push(chunk)`` returns every frame final in all octaves; ``flush()`` the rest, raising (and warning) as
    ``module(x)`` does for the stream's total length.  Concatenated along time the outputs are bitwise
    ``module(x)`` (a 16-bit stream: ``module(x.float())``): each push runs the whole-clip call's tensor-core plan
    (generation 2, or generation 1 with or without early downsampling) on the new samples, with the levels
    carried in fp32 rings (DESIGN.md §3.10).  Before the end, sample n of a decimated level is final once
    ``d n + c`` samples of its source have arrived (``c`` = 130 on generation 2, 129 otherwise), and an octave
    frame under the ``_ready_frames`` rule of its own level, so the lowest octave sets the latency.
    ``hop_length`` must be a multiple of ``2 ** (n_octaves - 1)``.  ``forward_kwargs``: ``output_format``,
    ``normalization_type``.
    """

    def __init__(self, module, batch, **forward_kwargs):
        if not isinstance(module, _PYRAMIDS):
            raise TypeError(f"StreamingPyramid supports CQT2010v2, VQT and CQT2010, not {type(module).__name__}")
        batch = _streams(batch, "batch")
        fmt = forward_kwargs.get("output_format") or module.output_format
        norm = forward_kwargs.get("normalization_type", "librosa")
        _check_format_and_norm(fmt, norm)
        if isinstance(module, CQT2010):
            self._args = lambda: _pyramid_args(module, fmt, module._normalization(norm))
        else:
            self._args = lambda: _pyramid_args(module, fmt, _v2_normalization(module, norm, fmt))
        self.module, self.batch = module, batch
        kw = self._args()
        self.widths = [int(b.shape[1]) for b in kw["banks_real"]]
        self.hop, self.early = kw["hop"], kw["early_factor"]
        n_oct = len(self.widths)
        if self.hop % (1 << (n_oct - 1)):
            # hop_i = hop >> i then drifts from hop / 2^i: the octaves' frame counts agree (and module(x) runs)
            # only for clips below a length bound, so no stream of unbounded length can match it
            raise ValueError(f"hop_length {self.hop} is not a multiple of 2^{n_oct - 1}: the octaves frame at "
                             "different rates")
        self._reflect = kw["pad_mode"] == _C.PAD_REFLECT
        # the whole-clip plan: generation 2 without early downsampling when every FIR-source bank is 256 wide
        self.generation = 2 if self.early == 1 and all(w // 2 == 128 for w in self.widths[:-1]) else 1
        n_bytes = _C.cqt_pyramid_chunk_state_bytes(batch, self.widths, self.hop, self.early)
        device = next(iter(module.buffers())).device
        self.ring = torch.empty(n_bytes // 4, dtype=torch.float32, device=device)  # one fp32 ring per level
        self.reset()

    def reset(self):
        """Start new streams (same module, same batch)."""
        self.received = self.n_carry = self.frames = 0
        self.dtype = None
        self._flushed = False

    # ------------------------------------------------------------------------------------------------ #
    def _counts(self, raw):
        """Final samples of every signal after ``raw`` raw samples (the raw samples first when an early stage
        feeds level 0): sample n of the next signal is final once d n + c of this one have arrived."""
        c = 130 if self.generation == 2 else 129
        R = [raw]
        for s in range(len(self.widths) + (self.early > 1) - 1):
            d = self.early if (self.early > 1 and s == 0) else 2
            R.append((R[-1] - c) // d + 1 if R[-1] >= c else 0)
        return R

    def _ready(self, raw):
        """Frames final in every octave after ``raw`` samples."""
        R = self._counts(raw)[1 if self.early > 1 else 0:]
        return min(_ready_frames(R[i], w, self.hop >> i, w // 2, self._reflect) for i, w in enumerate(self.widths))

    def _n_carry(self, raw, frames):
        """Raw samples the raw ring carries (nnab.h): the top octave's (no early stage) and the first FIR stage's
        read-back."""
        keep = raw
        if self.early == 1:
            keep = _carry_start(raw, frames, self.hop, self.widths[0] // 2)
        R = self._counts(raw)
        if len(R) > 1:
            d = self.early if self.early > 1 else 2
            keep = min(keep, max(0, 128 * d * (R[1] // 128) - 128))
        return raw - keep

    def latency(self):
        """Raw samples a push holds back behind frame t's centre t * hop in the steady state: frame t is
        returned once t * hop + latency() samples have arrived."""
        t = 1000 + max(self.widths)  # past every start-up effect
        lo, hi = 0, (t + 8) * self.hop * 4 + (1 << 22)
        while lo < hi:
            mid = (lo + hi) // 2
            if self._ready(mid) > t:
                hi = mid
            else:
                lo = mid + 1
        return lo - t * self.hop

    def push(self, chunk: torch.Tensor) -> torch.Tensor:
        """Feed ``chunk`` (batch, n), any n >= 0; returns the frames final in every octave."""
        if self._flushed:
            raise RuntimeError("push() after flush(): call reset() to start new streams")
        _check_chunk(chunk, self.batch, self.dtype)
        self.dtype = chunk.dtype
        n = chunk.shape[1]
        T = self._ready(self.received + n) - self.frames
        return self._advance(chunk, n, False, T)

    def flush(self) -> torch.Tensor:
        """End of stream: the remaining frames (raises and warns as ``module(x)`` for this length)."""
        if self._flushed:
            raise RuntimeError("flush() after flush(): call reset() to start new streams")
        T_total, _ = _pyramid_length_plan(self.module, self.batch, self.received)
        if self.dtype is None:
            self.dtype = torch.float32
        out = self._advance(None, 0, True, T_total - self.frames)
        self._flushed = True
        return out

    def _advance(self, chunk, n, flush, T):
        out = _C.cqt_pyramid_chunk_forward(self, chunk, flush, T, **self._args())
        if out is None:
            raise RuntimeError(f"{type(self.module).__name__}: no streamed tensor-core pyramid plan for this "
                               "call (NNAB_EUNSUPPORTED, e.g. NNAUDIO_B200_PATH=simt); the stream is unchanged")
        total = self.received + n
        self.received, self.frames = total, self.frames + T
        self.n_carry = self._n_carry(total, self.frames)
        return out


class PyramidPool(_ChunkPool):
    """Serve up to ``slots`` independent streams through the CQT pyramid of ``CQT2010v2``, ``VQT`` or ``CQT2010``,
    each advancing by its own amount.

    ``push(chunk, lengths, end=None)`` and ``reset(slots=None)`` are ``StreamPool``'s, and a push returns a
    ``PoolOutput``.  Each slot's frames follow ``StreamingPyramid``'s rules for its own stream: before its end the
    frames final in every octave, on its end the rest with the stream's right padding, raising (the slot named) and
    warning as ``module(x)`` does for the stream's total length.  Concatenated along time, a slot's rows up to their
    counts equal ``module(x)`` on its whole stream bit for bit (a 16-bit stream: ``module(x.float())``), and a
    one-stream ``StreamingPyramid`` fed the same packets.  Every argument is checked before anything is enqueued,
    and a push never reads the device back or synchronises.  ``module`` and ``forward_kwargs``: those of
    ``StreamingPyramid`` (``hop_length`` a multiple of ``2 ** (n_octaves - 1)``).

    A push is one C call (``_C.cqt_pyramid_pool_forward``): the whole-clip call's tensor-core plan, each stage and
    octave once over the lanes, every row aligned on its own stream (DESIGN.md §3.10 "Pyramid pools").  Idle
    slots cost nothing.  There is no concat route: a plan that cannot read the chunk (``NNAUDIO_B200_PATH=simt``,
    a missing packed operand) raises ``RuntimeError`` with the pool unchanged.
    """

    def __init__(self, module, slots, **forward_kwargs):
        slots = _streams(slots, "slots")
        # module checks, the pyramid arguments, the plan and one ring row per slot per signal: StreamingPyramid's
        self._sp = sp = StreamingPyramid(module, slots, **forward_kwargs)
        self.module = module
        self.widths, self.hop, self.early, self.generation = sp.widths, sp.hop, sp.early, sp.generation
        self._reflect = sp._reflect
        self.ring = sp.ring
        self._init_slots(slots)
        self.dtype = None

    # ---- StreamingPyramid's counters over arrays of lanes ------------------------------------------------- #
    def _counts(self, raw, end):
        """Samples of every signal after ``raw`` raw samples: the final ones, or (``end``) all of them."""
        c = 130 if self.generation == 2 else 129
        R = [raw]
        for s in range(len(self.widths) + (self.early > 1) - 1):
            d = self.early if (self.early > 1 and s == 0) else 2
            r = R[-1]
            R.append(np.where(end, np.where(r < 2, 0, (r - 2) // d + 1), np.where(r >= c, (r - c) // d + 1, 0)))
        return R

    def _ready(self, raw):
        """Frames final in every octave after ``raw`` samples (``StreamingPyramid._ready``)."""
        R = self._counts(raw, False)[1 if self.early > 1 else 0:]
        t = None
        for i, w in enumerate(self.widths):
            pad, need = w // 2, w - w // 2
            f = np.where(R[i] < need, 0, (R[i] - need) // (self.hop >> i) + 1)
            if self._reflect:
                f = np.where(R[i] < pad + 1, 0, f)
            t = f if t is None else np.minimum(t, f)
        return t

    def _n_carry(self, raw, frames):
        """Raw samples the raw ring carries (``StreamingPyramid._n_carry``)."""
        keep = raw
        if self.early == 1:
            pad = self.widths[0] // 2
            s = frames * self.hop - pad
            if pad > 0:
                s = np.minimum(s, raw - (pad + 1))
            keep = np.minimum(np.maximum(s, 0), raw)
        R = self._counts(raw, False)
        if len(R) > 1:
            d = self.early if self.early > 1 else 2
            keep = np.minimum(keep, np.maximum(0, 128 * d * (R[1] // 128) - 128))
        return raw - keep

    # ------------------------------------------------------------------------------------------------ #
    def _lane_counts(self, active, lengths, end):
        """Every lane's frame count and carried raw samples, by the rules of StreamingPyramid (push / flush); per
        lane only the length plan of an end."""
        R, F0, e = self.received[active], self.frames[active], end[active]
        total = R + lengths[active]
        count = self._ready(total) - F0
        for j in np.flatnonzero(e).tolist():
            T_total, _ = _for_slot(int(active[j]), _pyramid_length_plan, self.module, 1, int(total[j]))
            count[j] = T_total - F0[j]
        return count, self._n_carry(R, F0)

    def _advance(self, chunk, lanes, A, T_max, count):
        out = _C.cqt_pyramid_pool_forward(self, lanes, chunk, A, T_max, **self._sp._args())
        if out is None:
            raise RuntimeError(f"{type(self.module).__name__}: no streamed tensor-core pyramid plan for this call "
                               "(NNAB_EUNSUPPORTED, e.g. NNAUDIO_B200_PATH=simt); the pool is unchanged")
        return out


class StreamingInverse:
    """Stream ``batch`` complex spectrograms frame block by frame block through an inverse STFT.

    ``module``: an ``iSTFT``, or an ``STFT`` built with ``iSTFT=True`` (its ``inverse``).  ``onesided``
    defaults to the module's own default (``iSTFT``: False, ``STFT.inverse``: True).  ``push(X)`` takes
    ``(batch, bins, t, 2)`` float32 frames, any t >= 0, and returns the output samples no later frame can change;
    ``flush(length=None)`` returns the rest with the module's ``length`` / ``center`` rules.  The concatenation
    equals ``module(X)`` / ``module.inverse(X)`` on all frames to fp32 rounding (both overlap-add with fp32
    atomics, so neither is bit-repeatable).
    """

    def __init__(self, module, batch, onesided=None):
        if isinstance(module, iSTFT):
            bufs = (module.kernel_cos, module.kernel_sin, module.window_mask)
            onesided = False if onesided is None else bool(onesided)
        elif isinstance(module, STFT) and hasattr(module, "kernel_cos_inv"):
            bufs = (module.kernel_cos_inv, module.kernel_sin_inv, module.window_mask)
            onesided = True if onesided is None else bool(onesided)
        else:
            raise TypeError(f"StreamingInverse takes an iSTFT or an STFT built with iSTFT=True, not "
                            f"{type(module).__name__}{'' if not isinstance(module, STFT) else ' without iSTFT=True'}")
        batch = _streams(batch, "batch")
        self.module, self.batch, self.onesided = module, batch, onesided
        self.n_fft, self.hop, self.center = module.n_fft, module.stride, bool(module.center)
        if self.hop > self.n_fft:
            raise ValueError(f"hop_length {self.hop} > n_fft {self.n_fft}: the frames do not overlap")
        self.f_in = self.n_fft // 2 + 1 if onesided else self.n_fft
        self._args = lambda: _inverse_args(module, self.f_in, *bufs, onesided)
        self.offset = self.n_fft // 2 if self.center else 0
        device = next(iter(module.buffers())).device
        self.state = torch.empty((batch, self.n_fft), dtype=torch.float32, device=device)  # open partial sums
        self.reset()

    def reset(self):
        self.frames = self.emitted = 0
        self._flushed = False

    def _emit_end(self, n):
        """End (overlap-add position) of the samples returned after n frames: below n * hop, and below the
        earliest end the output can still have."""
        if n <= 0:
            return self.offset
        end_min = self.n_fft + self.hop * (n - 1) - (self.offset if self.center else 0)
        return max(self.offset, min(n * self.hop, end_min))

    def push(self, X: torch.Tensor) -> torch.Tensor:
        if self._flushed:
            raise RuntimeError("push() after flush(): call reset() to start new streams")
        if not isinstance(X, torch.Tensor):
            raise TypeError("X must be a torch.Tensor")
        if X.requires_grad:
            raise NotImplementedError("the streaming API is forward-only: the frames require grad")
        if X.dim() != 4 or X.shape[0] != self.batch or X.shape[1] != self.f_in or X.shape[3] != 2:
            raise ValueError(f"frames must be ({self.batch}, {self.f_in}, t, 2), got {tuple(X.shape)}")
        T = X.shape[2]
        n_out = self._emit_end(self.frames + T) - (self.offset + self.emitted)
        return self._advance(X, False, None, n_out)

    def flush(self, length=None) -> torch.Tensor:
        if self._flushed:
            raise RuntimeError("flush() after flush(): call reset() to start new streams")
        if self.frames == 0:
            raise RuntimeError("flush() of a stream without frames: the inverse STFT needs at least one")
        ola_len = self.n_fft + self.hop * (self.frames - 1)
        want = length if length is not None else (ola_len - 2 * self.offset if self.center else ola_len)
        want = max(0, min(want, ola_len - self.offset))
        if want < self.emitted:
            raise ValueError(f"length {length} is shorter than the {self.emitted} samples already returned")
        X = self.state.new_empty((self.batch, self.f_in, 0, 2))
        out = self._advance(X, True, length, want - self.emitted)
        self._flushed = True
        return out

    def _advance(self, X, flush, length, n_out):
        _, _, packed, win = self._args()
        out = _C.istft_chunk_forward(self, X, flush, length, n_out, packed, win, self.n_fft, self.hop, self.center)
        self.frames += X.shape[2]
        self.emitted += n_out
        return out


class InverseOutput(NamedTuple):
    """One ``InversePool.push``: row i of ``samples`` (A, n_max) holds the new output samples of slot
    ``slots[i]``, ``counts[i]`` of them, then exact zeros.  ``slots`` (ascending) and ``counts`` are int64 CPU
    tensors."""
    samples: torch.Tensor
    slots: torch.Tensor
    counts: torch.Tensor


class InversePool(_HostPool):
    """Serve up to ``slots`` independent streamed inverse STFTs, each advancing by its own frame count.

    ``module`` and ``onesided``: those of ``StreamingInverse``.  ``push(X, slots, counts, end=None,
    length=None)``: ``X`` is (R, bins, t, 2) float32 CUDA frames and row r appends ``X[r, :, :counts[r]]`` to
    slot ``slots[r]`` (``slots``, ``counts``: R CPU integers; slots distinct, ``0 <= counts[r] <= t``; frames past
    a count are never read).  ``end`` (``slots`` CPU bools) ends the flagged slots: they get the rest of their
    samples under the ``StreamingInverse.flush`` rules, with ``length[s]`` (``slots`` CPU integers, -1: None; read
    only where ``end`` is set), and take no more frames until ``reset([s])``.  A ``PoolOutput`` of
    ``StreamPool`` and the ``end`` given to it can be passed on as they are.  Returns an ``InverseOutput`` with a
    row for each slot that has new samples.  Concatenated, a slot's rows up to their counts equal
    ``StreamingInverse`` on the same packets and ``module(X_s)`` / ``module.inverse(X_s)`` on all its frames, to
    fp32 rounding (every overlap-add uses fp32 atomics).  Every argument is checked before anything is enqueued,
    and a push never reads the device back or synchronises.

    A push is one C call (``_C.istft_pool_forward``): a seed launch (every lane's carried sums), the offline
    pre-pass and FMT_OLA GEMM once over all lanes' frames, and one finalize launch; idle slots cost nothing.
    """

    _COUNTERS = ("frames", "emitted")

    def __init__(self, module, slots, onesided=None):
        slots = _streams(slots, "slots")
        # module checks, the inverse arguments and the (slots, n_fft) fp32 state: StreamingInverse's
        self._si = si = StreamingInverse(module, slots, onesided=onesided)
        self.module, self.onesided = module, si.onesided
        self.n_fft, self.hop, self.center, self.f_in, self.offset = si.n_fft, si.hop, si.center, si.f_in, si.offset
        self.state = si.state  # row s: slot s's open overlap-add sums
        self._init_slots(slots)

    def _emit_end(self, n):
        """``StreamingInverse._emit_end`` over an array of frame counts."""
        end_min = self.n_fft + self.hop * (n - 1) - self.offset
        return np.where(n <= 0, self.offset, np.maximum(self.offset, np.minimum(n * self.hop, end_min)))

    def _flush_end(self, n, length):
        """End position of the output after n frames under ``StreamingInverse.flush(length)`` (length < 0:
        None), over arrays."""
        ola_len = self.n_fft + self.hop * (n - 1)
        want = np.where(length >= 0, length, ola_len - 2 * self.offset)
        return self.offset + np.clip(want, 0, np.maximum(ola_len - self.offset, 0))

    # ------------------------------------------------------------------------------------------------ #
    def push(self, X: torch.Tensor, slots, counts, end=None, length=None) -> InverseOutput:
        """Append ``X[r, :, :counts[r]]`` to slot ``slots[r]`` for every row r, end the slots flagged in ``end``;
        returns the new samples of the slots that have some."""
        if not isinstance(X, torch.Tensor):
            raise TypeError("X must be a torch.Tensor")
        if X.requires_grad:
            raise NotImplementedError("the streaming API is forward-only: the frames require grad")
        if X.dim() != 4 or X.shape[1] != self.f_in or X.shape[3] != 2:
            raise ValueError(f"frames must be (rows, {self.f_in}, t, 2), got {tuple(X.shape)}")
        if X.dtype != torch.float32:
            raise ValueError(f"frames must be float32, got {X.dtype}")
        R, t = X.shape[0], X.shape[2]
        rows_slot = _cpu_ints(slots, "slots", R)
        rows_count = _cpu_ints(counts, "counts", R)
        end = np.zeros(self.slots, bool) if end is None else _cpu_ints(end, "end", self.slots, "bools")
        length = np.full(self.slots, -1, np.int64) if length is None else _cpu_ints(length, "length", self.slots)
        bad = np.flatnonzero((rows_slot < 0) | (rows_slot >= self.slots))
        if len(bad):
            raise ValueError(f"slots must be in [0, {self.slots}): row {bad[0]} has slot {rows_slot[bad[0]]}")
        uniq, first = np.unique(rows_slot, return_counts=True)
        if (first > 1).any():
            raise ValueError(f"slot {uniq[first > 1][0]} appears in more than one row")
        bad = np.flatnonzero((rows_count < 0) | (rows_count > t))
        if len(bad):
            raise ValueError(f"counts must be in [0, {t}] (the frames of X): slot {rows_slot[bad[0]]} has "
                             f"{rows_count[bad[0]]}")
        T = np.zeros(self.slots, np.int64)  # new frames and their row of X, per slot
        row = np.full(self.slots, -1, np.int64)
        T[rows_slot] = rows_count
        row[rows_slot] = np.arange(R)
        row[T == 0] = -1
        self._refuse_ended(T > 0, end)
        n = self.frames + T
        bad = np.flatnonzero(end & (n == 0))
        if len(bad):
            raise RuntimeError(f"slot {bad[0]}: ending a stream without frames; the inverse STFT needs at least one")
        # every slot's output end after the push, by the rules of StreamingInverse (push / flush)
        emit_end = np.where(end, self._flush_end(n, length), self._emit_end(n))
        count = emit_end - (self.offset + self.emitted)
        bad = np.flatnonzero(end & (count < 0))
        if len(bad):
            s = bad[0]
            raise ValueError(f"slot {s}: length {length[s]} is shorter than the {self.emitted[s]} samples already "
                             "returned")
        active = np.flatnonzero((T > 0) | end)
        order = np.lexsort((active, count[active] == 0))  # lanes with samples first, slots ascending in each group
        active = active[order]
        count = count[active]
        A = int((count > 0).sum())
        n_max = int(count.max()) if A else 0
        T_max = int(T[active].max()) if len(active) else 0
        lanes = np.stack([active, row[active], self.frames[active], self.emitted[active], T[active],
                          end[active].astype(np.int64), np.where(end[active], length[active], -1)], 1)
        _, _, packed, win = self._si._args()
        out = _C.istft_pool_forward(self, lanes.astype(np.int64), X, A, n_max, T_max, packed, win, self.n_fft,
                                    self.hop, self.center)
        self.frames[active] += T[active]
        self.emitted[active] += count
        self.ended[active] |= end[active]
        return InverseOutput(out, torch.from_numpy(active[:A].copy()), torch.from_numpy(count[:A].copy()))


# ---- device pools (DESIGN.md §3.10 "Device pools") ------------------------------------------------------------- #
def _device_vector(v, what, slots, dtype, device):
    """``v`` as a device pool's push reads it: a contiguous (slots,) tensor of ``dtype`` on ``device``."""
    if not isinstance(v, torch.Tensor):
        raise TypeError(f"{what} must be a torch.Tensor on {device}, filled in place each push")
    if v.device != device:
        raise TypeError(f"{what} must be on {device}: the push reads it there, got {v.device}")
    if v.dtype != dtype:
        raise TypeError(f"{what} must be {dtype}, got {v.dtype}")
    if tuple(v.shape) != (slots,) or not v.is_contiguous():
        raise ValueError(f"{what} must hold one value per slot ({slots}), contiguous, got shape {tuple(v.shape)}")
    return v


class _DevicePool:
    """What the device pools share: the per-slot counters, error codes and values, counts and lane table on the
    device, the reset and the lookup of the first error."""

    def _init_device(self, slots, lane_fields, dev):
        self.slots = slots
        self.counters = torch.zeros((3, slots), dtype=torch.int64, device=dev)
        self.errors = torch.zeros(slots, dtype=torch.int32, device=dev)
        self.error_info = torch.zeros((slots, 2), dtype=torch.int64, device=dev)
        self.counts = torch.zeros(slots, dtype=torch.int32, device=dev)
        self._lanes = torch.zeros((slots, len(lane_fields)), dtype=torch.int64, device=dev)
        self._no_end = torch.zeros(slots, dtype=torch.bool, device=dev)

    def reset(self, restart=None):
        """Start new streams where the bool device mask ``restart`` is set (None: every slot)."""
        mask = None if restart is None else _device_vector(restart, "restart", self.slots, torch.bool,
                                                           self.counters.device)
        _C.pool_device_reset(self, mask)

    def _first_error(self):
        """(slot, code, info a, info b) of the lowest slot with an error code, or None; synchronises."""
        errors = self.errors.cpu()
        bad = torch.nonzero(errors).flatten()
        if len(bad) == 0:
            return None
        s = int(bad[0])
        a, b = self.error_info[s].tolist()
        return s, int(errors[s]), a, b


class DeviceStreamPool(_DevicePool):
    """``StreamPool`` with every per-push number on the GPU: a push reads nothing on the host and has one fixed
    geometry, so it can be captured in a CUDA graph (``torch.cuda.graph``) and replayed.

    ``DeviceStreamPool(module, slots, chunk, dtype=torch.float32, **forward_kwargs)``: ``module`` and
    ``forward_kwargs`` are ``StreamPool``'s; ``chunk`` is the fixed chunk width and ``dtype`` the fixed sample type
    (float32, bfloat16 or float16).  ``push(x, lengths, end=None)``: ``x`` is a (slots, chunk) CUDA tensor of that
    type, ``lengths`` an int32 and ``end`` a bool (slots,) tensor on the same device; slot s appends
    ``x[s, :lengths[s]]`` and ends where ``end[s]``.  The push overwrites the pool-owned ``frames`` (slots, ...,
    T_cap) float32 and ``counts`` (slots,) int32: row s holds slot s's new frames, ``counts[s]`` of them, then exact
    zeros.  Concatenated up to its counts, a slot's rows equal ``StreamPool`` on the same packets (the same
    bit-for-bit rules and CQT1992v2 exception).  ``reset(restart=None)`` starts new streams where the bool device
    mask ``restart`` is set (None: every slot); it too is one launch and can be captured.

    ``T_cap`` is the most frames one push of at most ``chunk`` samples can return, an end included, derived from
    the framing.  Every slot is computed on every push at ``T_cap`` frames, so an idle slot costs its share of the
    launch (``StreamPool`` computes only the slots with new frames, at their longest count, but reads its
    bookkeeping on the host).  A push cannot raise for its values: a slot whose push ``StreamPool`` would refuse (a
    length outside [0, chunk], samples or an end on an ended stream, an end on a stream too short for the module)
    is dropped whole -- counters, ring and row untouched, count 0 -- and ``errors[s]`` (int32, device) keeps the
    first such code until the slot's reset, while the other slots proceed.  ``check()`` synchronises and raises
    what ``StreamPool`` would have raised, naming the slot.  There is no concat route: a plan without a fused pool
    route (``NNAUDIO_B200_PATH=simt``) raises at construction.  The constructor builds every cache a push uses and
    allocates the state, counters (``counters``: received, frames, ended per slot), outputs and workspace, so a
    captured push allocates nothing.
    """

    def __init__(self, module, slots, chunk, dtype=torch.float32, **forward_kwargs):
        slots, chunk = _streams(slots, "slots"), int(chunk)
        if chunk < 1:
            raise ValueError(f"chunk must be at least 1 sample, got {chunk}")
        if dtype not in _C._WAVE_DTYPES:
            raise ValueError(f"dtype must be float32, bfloat16 or float16, got {dtype}")
        # module checks, the offline call's arguments and the (slots, K) fp32 carry ring: StreamingTransform's
        self._st = st = StreamingTransform(module, slots, _strict=True, **forward_kwargs)
        self.module, self.chunk, self.dtype = module, chunk, dtype
        self.K, self.hop, self.pad = st.K, st.hop, st.pad
        self.ring = st.ring
        dev = self.ring.device
        name, self._kw = st._args()  # packed basis, filterbank table (synchronises once), scales: built here
        self.T_cap = _C.pool_frame_cap(chunk, self.K, self.hop, self.pad, self._kw["pad_mode"])
        self._init_device(slots, _C.LANE_FIELDS, dev)
        self._fn, self.frames, self._ws, self._tail = _C.pool_device_bind(name, self._kw, slots, self.T_cap, dev)
        # an idle push changes nothing; it runs the route once and finds a plan that cannot read the chunk
        idle = torch.zeros(slots, dtype=torch.int32, device=dev)
        if not _C.pool_device_forward(self, torch.zeros((slots, chunk), dtype=dtype, device=dev), idle, self._no_end):
            raise RuntimeError(f"{name}: no fused pool route for this configuration (NNAB_EUNSUPPORTED, e.g. "
                               "NNAUDIO_B200_PATH=simt); DeviceStreamPool has no concat route")

    def push(self, x: torch.Tensor, lengths: torch.Tensor, end: torch.Tensor = None):
        """Append ``x[s, :lengths[s]]`` to every slot s and end the slots flagged in ``end``; the new frames go
        to ``frames`` / ``counts``."""
        _check_chunk(x, self.slots, self.dtype, width=self.chunk)
        if x.device != self.ring.device:
            raise RuntimeError(f"chunk is on {x.device}: the pool runs on {self.ring.device}")
        if x.stride(-1) != 1 or (self.slots > 1 and x.stride(0) < self.chunk):
            x = x.contiguous()
        dev = self.ring.device
        lengths = _device_vector(lengths, "lengths", self.slots, torch.int32, dev)
        end = self._no_end if end is None else _device_vector(end, "end", self.slots, torch.bool, dev)
        if not _C.pool_device_forward(self, x, lengths, end):
            raise RuntimeError("no fused pool route for this configuration (NNAB_EUNSUPPORTED)")

    def check(self):
        """Synchronise and raise what ``StreamPool`` would have raised for the lowest slot with an error code."""
        err = self._first_error()
        if err is None:
            return
        s, code, a, _ = err
        if code == _C.LANE_ELENGTH:
            raise ValueError(f"lengths must be in [0, {self.chunk}] (the chunk width): slot {s} has {a}")
        if code == _C.LANE_EENDED:
            raise _ended_error(s)
        if code == _C.LANE_ESHORT:
            _for_slot(s, self._st._check_length, a)  # the exception module(x) raises for a stream this short
        raise RuntimeError(f"slot {s}: push dropped with error code {code}")


class DevicePyramidPool(_DevicePool):
    """``PyramidPool`` with every per-push number on the GPU, capturable in a CUDA graph like ``DeviceStreamPool``.

    ``DevicePyramidPool(module, slots, chunk, dtype=torch.float32, **forward_kwargs)``: ``module`` and
    ``forward_kwargs`` are ``PyramidPool``'s (``CQT2010v2``, ``VQT`` or ``CQT2010``; ``hop_length`` a multiple of
    ``2 ** (n_octaves - 1)``), ``chunk`` the fixed chunk width and ``dtype`` the fixed sample type.  ``push(x,
    lengths, end=None)``, ``reset(restart=None)``, ``errors``, ``error_info``, ``counters`` and ``check()`` are
    ``DeviceStreamPool``'s; a push overwrites the pool-owned ``frames`` (slots, n_bins, T_cap[, 2]) float32 and
    ``counts`` (slots,) int32.  Concatenated up to its counts, a slot's rows equal ``PyramidPool`` on the same packets
    and ``module(x)`` on its whole stream, bit for bit (a 16-bit stream: ``module(x.float())``).  A push never sees
    the lengths on the host, so it cannot issue the reflect-fallback ``UserWarning`` that ``module(x)`` and
    ``PyramidPool`` give for a short stream; the frames are those of the fallback all the same.  A slot whose push
    ``PyramidPool`` would refuse (a length outside [0, chunk], samples or an end on an ended stream, an end on a
    stream too short for the module) is dropped whole and flagged in ``errors``.

    ``T_cap``, the FIR outputs each stage computes per slot and the samples each ring takes per push are the most
    one push of at most ``chunk`` samples can need, an end included (``_C.cqt_pyramid_pool_device_caps``).  Every
    stage and octave runs on every slot at those caps on every push: an ending stream returns its whole pending
    tail (the pyramid's look-ahead), so ``T_cap`` is that tail in frames plus the chunk's own, and an idle or
    steady slot costs its share of that.  There is no concat route: a plan without a streamed tensor-core route
    (``NNAUDIO_B200_PATH=simt``, a missing packed operand) raises ``RuntimeError`` at construction.  The constructor
    builds every cache a push uses and allocates the rings, counters, outputs and workspace, so a captured push
    allocates nothing.
    """

    def __init__(self, module, slots, chunk, dtype=torch.float32, **forward_kwargs):
        slots, chunk = _streams(slots, "slots"), int(chunk)
        if chunk < 1:
            raise ValueError(f"chunk must be at least 1 sample, got {chunk}")
        if dtype not in _C._WAVE_DTYPES:
            raise ValueError(f"dtype must be float32, bfloat16 or float16, got {dtype}")
        # module checks, the pyramid arguments, the plan and one ring row per slot per signal: StreamingPyramid's
        self._sp = sp = StreamingPyramid(module, slots, **forward_kwargs)
        self.module, self.chunk, self.dtype = module, chunk, dtype
        self.widths, self.hop, self.early, self.generation = sp.widths, sp.hop, sp.early, sp.generation
        self.ring = sp.ring
        dev = self.ring.device
        self._kw = kw = sp._args()  # banks, packed operands, filters, scale: built here and kept alive
        self.T_cap = _C.cqt_pyramid_pool_device_caps(chunk, self.widths, self.hop, self.early, kw["pad_mode"])[0]
        self._init_device(slots, _C.LANE_FIELDS, dev)
        self._fn, self.frames, self._ws, self._tail = _C.pyramid_pool_device_bind(kw, slots, chunk, self.T_cap, dev)
        # an idle push changes nothing; it finds a plan that cannot read the chunk before anything is enqueued
        idle = torch.zeros(slots, dtype=torch.int32, device=dev)
        if not _C.pool_device_forward(self, torch.zeros((slots, chunk), dtype=dtype, device=dev), idle, self._no_end):
            raise RuntimeError(f"{type(module).__name__}: no streamed tensor-core pyramid plan for this call "
                               "(NNAB_EUNSUPPORTED, e.g. NNAUDIO_B200_PATH=simt); DevicePyramidPool has no concat route")

    def push(self, x: torch.Tensor, lengths: torch.Tensor, end: torch.Tensor = None):
        """Append ``x[s, :lengths[s]]`` to every slot s and end the slots flagged in ``end``; the new frames go
        to ``frames`` / ``counts``."""
        _check_chunk(x, self.slots, self.dtype, width=self.chunk)
        if x.device != self.ring.device:
            raise RuntimeError(f"chunk is on {x.device}: the pool runs on {self.ring.device}")
        if x.stride(-1) != 1 or (self.slots > 1 and x.stride(0) < self.chunk):
            x = x.contiguous()
        dev = self.ring.device
        lengths = _device_vector(lengths, "lengths", self.slots, torch.int32, dev)
        end = self._no_end if end is None else _device_vector(end, "end", self.slots, torch.bool, dev)
        if not _C.pool_device_forward(self, x, lengths, end):
            raise RuntimeError("no streamed tensor-core pyramid plan for this call (NNAB_EUNSUPPORTED)")

    def check(self):
        """Synchronise and raise what ``PyramidPool`` would have raised for the lowest slot with an error code."""
        err = self._first_error()
        if err is None:
            return
        s, code, a, _ = err
        if code == _C.LANE_ELENGTH:
            raise ValueError(f"lengths must be in [0, {self.chunk}] (the chunk width): slot {s} has {a}")
        if code == _C.LANE_EENDED:
            raise _ended_error(s)
        if code == _C.LANE_ESHORT:
            _for_slot(s, _pyramid_length_plan, self.module, 1, a)  # the exception module(x) raises for this length
        raise RuntimeError(f"slot {s}: push dropped with error code {code}")


class DeviceInversePool(_DevicePool):
    """``InversePool`` with every per-push number on the GPU, capturable in a CUDA graph like ``DeviceStreamPool``.

    ``DeviceInversePool(module, slots, frames, onesided=None)``: ``module`` and ``onesided`` are ``InversePool``'s,
    ``frames`` the fixed frame capacity of a push.  ``push(X, counts, end=None, length=None)``: ``X`` is (slots,
    bins, frames, 2) float32 CUDA (row s: slot s's frames; a ``DeviceStreamPool``'s ``frames`` in the Complex format
    with ``frames=pool.T_cap`` fits), ``counts`` int32, ``end`` bool and ``length`` int64 (-1: None; read where
    ``end`` is set) (slots,) tensors on the same device; slot s appends ``X[s, :, :counts[s]]``, and ends under
    ``StreamingInverse.flush``'s rules.  The push overwrites the pool-owned ``samples`` (slots, n_cap) and
    ``counts`` (slots,) int32: row s holds slot s's new samples, then exact zeros.  ``n_cap`` is the most samples
    one push of at most ``frames`` frames can return, a flush included.  Concatenated, a slot's rows equal
    ``InversePool`` on the same packets to fp32 rounding (both overlap-add with fp32 atomics).  Errors, ``check()``,
    ``reset(restart=None)`` and the cost of idle slots are ``DeviceStreamPool``'s; the refused pushes are
    ``InversePool``'s (counts outside [0, frames], frames or an end on an ended stream, an end without any frame,
    a length shorter than the samples already returned).
    """

    def __init__(self, module, slots, frames, onesided=None):
        slots, frames = _streams(slots, "slots"), int(frames)
        if frames < 1:
            raise ValueError(f"frames must be at least 1, got {frames}")
        # module checks, the inverse arguments and the (slots, n_fft) fp32 state: StreamingInverse's
        self._si = si = StreamingInverse(module, slots, onesided=onesided)
        self.module, self.onesided, self.frames_cap = module, si.onesided, frames
        self.n_fft, self.hop, self.center, self.f_in = si.n_fft, si.hop, si.center, si.f_in
        self.state = si.state
        dev = self.state.device
        _, _, self._packed, self._window = si._args()
        self.n_cap = _C.istft_pool_sample_cap(frames, self.n_fft, self.hop, self.center)
        self._init_device(slots, _C.ISTFT_LANE_FIELDS, dev)  # counters: frames, emitted, ended
        self.samples = torch.zeros((slots, self.n_cap), dtype=torch.float32, device=dev)
        self._ws = torch.empty(_C.lib().nnab_istft_pool_workspace_bytes(slots, self.f_in, frames, self.n_fft,
                                                                         self.hop), dtype=torch.uint8, device=dev)
        self._no_length = torch.full((slots,), -1, dtype=torch.int64, device=dev)
        idle = torch.zeros(slots, dtype=torch.int32, device=dev)  # an idle push changes nothing
        _C.istft_pool_device_forward(self, torch.zeros((slots, self.f_in, frames, 2), device=dev), idle,
                                     self._no_end, self._no_length)

    def push(self, X: torch.Tensor, counts: torch.Tensor, end: torch.Tensor = None, length: torch.Tensor = None):
        """Append ``X[s, :, :counts[s]]`` to every slot s and end the slots flagged in ``end``; the new samples go
        to ``samples`` / ``counts``."""
        if not isinstance(X, torch.Tensor):
            raise TypeError("X must be a torch.Tensor")
        if X.requires_grad:
            raise NotImplementedError("the streaming API is forward-only: the frames require grad")
        want = (self.slots, self.f_in, self.frames_cap, 2)
        if tuple(X.shape) != want:
            raise ValueError(f"frames must be {want}, got {tuple(X.shape)}")
        if X.dtype != torch.float32:
            raise ValueError(f"frames must be float32, got {X.dtype}")
        dev = self.state.device
        if X.device != dev:
            raise RuntimeError(f"X is on {X.device}: the pool runs on {dev}")
        X = X if X.is_contiguous() else X.contiguous()
        counts = _device_vector(counts, "counts", self.slots, torch.int32, dev)
        end = self._no_end if end is None else _device_vector(end, "end", self.slots, torch.bool, dev)
        length = self._no_length if length is None else _device_vector(length, "length", self.slots, torch.int64, dev)
        _C.istft_pool_device_forward(self, X, counts, end, length)

    def check(self):
        """Synchronise and raise what ``InversePool`` would have raised for the lowest slot with an error code."""
        err = self._first_error()
        if err is None:
            return
        s, code, a, b = err
        if code == _C.LANE_ELENGTH:
            raise ValueError(f"counts must be in [0, {self.frames_cap}] (the frames of X): slot {s} has {a}")
        if code == _C.LANE_EENDED:
            raise _ended_error(s)
        if code == _C.LANE_ENOFRAMES:
            raise RuntimeError(f"slot {s}: ending a stream without frames; the inverse STFT needs at least one")
        if code == _C.LANE_ELENGTH_SHORT:
            raise ValueError(f"slot {s}: length {a} is shorter than the {b} samples already returned")
        raise RuntimeError(f"slot {s}: push dropped with error code {code}")
