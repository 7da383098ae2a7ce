"""Per-channel energy normalisation (PCEN; beyond the reference, DESIGN.md §3.11).

PCEN (Wang et al., 2017, "Trainable frontend for robust and far-field keyword spotting"; the trainable form LEAF
uses) replaces the log of a Mel spectrogram in keyword spotting, speech enhancement and far-field ASR front ends.
Per channel c of a non-negative (B, C, T) spectrogram E, with parameters s, gain, bias, power and eps:

    M[t] = (1 - s) M[t-1] + s E[t]                      M[-1] = E[0]  (the smoother starts settled)
    P[t] = (bias + E[t] (eps + M[t]) ** -gain) ** power - bias ** power

``PCEN`` is the module: one launch per inference call, a fused forward / backward pair under autograd.
``PCENStream(pcen, slots)`` carries each stream's smoother across calls, so the frames of ``StreamingTransform``,
``StreamPool`` or ``DeviceStreamPool`` can be normalised as they arrive, bit for bit equal to the whole-clip call.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn as nn

from . import _C
from .streaming import _device_vector

__all__ = ["PCEN", "PCENStream", "smoothing_coef"]


def smoothing_coef(sr: float, hop_length: int, time_constant: float) -> float:
    """The smoother's ``s`` for a time constant in seconds: ``(sqrt(1 + 4 t^2) - 1) / (2 t^2)`` with
    ``t = time_constant * sr / hop_length`` frames (librosa's ``pcen``)."""
    if not (sr > 0 and hop_length > 0 and time_constant > 0):
        raise ValueError(f"sr, hop_length and time_constant must be positive, got {sr}, {hop_length}, "
                         f"{time_constant}")
    t = float(time_constant) * float(sr) / float(hop_length)
    return (math.sqrt(1.0 + 4.0 * t * t) - 1.0) / (2.0 * t * t)


def _values(name, v, n_channels, ok, rule):
    """``v`` (a number, or one per channel) as the float32 tensor the module stores: shape () for scalars,
    (n_channels,) for per-channel parameters."""
    a = np.asarray(v.detach().cpu() if isinstance(v, torch.Tensor) else v, dtype=np.float64)
    if n_channels is None:
        if a.size != 1:
            raise ValueError(f"{name} must be a number without n_channels, got shape {a.shape}")
        a = a.reshape(())
    else:
        if a.size == 1:
            a = np.full(n_channels, float(a.reshape(())))
        if a.shape != (n_channels,):
            raise ValueError(f"{name} must be a number or hold n_channels = {n_channels} values, got shape {a.shape}")
    if not (np.isfinite(a).all() and ok(a).all()):
        raise ValueError(f"{name} must satisfy {rule}, got {a.tolist()}")
    return torch.tensor(a, dtype=torch.float32)


class _PCENFn(torch.autograd.Function):
    """Differentiable PCEN ``(E, s, gain, bias, power) -> P``: forward = the PCEN kernel, also writing the smoother
    output M; backward = the reverse-time adjoint kernel, and for the parameters the fixed-order reduction of its
    per-row partials over the batch (and the channels, for scalar parameters)."""

    @staticmethod
    def forward(ctx, E, s, gain, bias, power, eps):
        M = torch.empty_like(E)
        P = _C.pcen_forward(E, (s, gain, bias, power), eps, M=M)
        ctx.eps = eps
        ctx.save_for_backward(E, M, s, gain, bias, power)
        return P

    @staticmethod
    def backward(ctx, gP):
        E, M, *params = ctx.saved_tensors
        need = ctx.needs_input_grad
        dE, dp = _C.pcen_backward(E, M, gP.contiguous(), params, ctx.eps, want_E=need[0], want_params=any(need[1:5]))
        grads = [dp[q].reshape(params[q].shape) if need[1 + q] else None for q in range(4)]
        return (dE, *grads, None)


class PCEN(nn.Module):
    """Per-channel energy normalisation of a (B, C, T) float32 CUDA spectrogram (e.g. ``MelSpectrogram`` output).

    ``PCEN(n_channels=None, sr=22050, hop_length=512, time_constant=0.4, s=None, gain=0.98, bias=2.0, power=0.5,
    eps=1e-6, trainable=False)``: librosa's names and defaults.  ``s`` defaults to ``smoothing_coef(sr, hop_length,
    time_constant)``.  The parameters are scalars, or with ``n_channels`` one value per channel (each given as a
    number or a sequence of ``n_channels``).  ``s``, ``gain``, ``bias`` and ``power`` are buffers, or
    ``nn.Parameter`` s with ``trainable=True``; ``eps`` is a constant.  The constructor refuses values outside
    ``0 < s <= 1``, ``gain >= 0``, ``bias > 0``, ``power > 0``, ``eps > 0``; values on the device are not checked
    again (that would synchronise).  The smoother starts settled on the first frame (LEAF's convention; librosa's
    default initial state differs).
    """

    def __init__(self, n_channels=None, sr=22050, hop_length=512, time_constant=0.4, s=None, gain=0.98, bias=2.0,
                 power=0.5, eps=1e-6, trainable=False):
        super().__init__()
        if n_channels is not None and int(n_channels) < 1:
            raise ValueError(f"n_channels must be at least 1, got {n_channels}")
        self.n_channels = None if n_channels is None else int(n_channels)
        if s is None:
            s = smoothing_coef(sr, hop_length, time_constant)
        if not (isinstance(eps, (int, float)) and math.isfinite(eps) and eps > 0):
            raise ValueError(f"eps must be a positive number, got {eps}")
        self.eps = float(eps)
        self.trainable = bool(trainable)
        rules = (("s", s, lambda a: (a > 0) & (a <= 1), "0 < s <= 1"), ("gain", gain, lambda a: a >= 0, "gain >= 0"),
                 ("bias", bias, lambda a: a > 0, "bias > 0"), ("power", power, lambda a: a > 0, "power > 0"))
        for name, v, ok, rule in rules:
            t = _values(name, v, self.n_channels, ok, rule)
            if trainable:
                self.register_parameter(name, nn.Parameter(t, requires_grad=True))
            else:
                self.register_buffer(name, t)

    def _params(self, device):
        out = []
        for name in ("s", "gain", "bias", "power"):
            p = getattr(self, name)
            _C._dev_f32(p.detach(), name)
            if p.device != device:
                raise RuntimeError(f"{name} is on {p.device}, the spectrogram on {device}")
            out.append(p)
        return out

    def _checked(self, E, what="E"):
        """E as the kernels read it: a contiguous (B, C, T) float32 CUDA tensor with C matching the parameters."""
        if not isinstance(E, torch.Tensor):
            raise TypeError(f"{what} must be a torch.Tensor")
        _C._dev_f32(E, what)
        if E.dim() != 3:
            raise ValueError(f"{what} must be (batch, channels, frames), got shape {tuple(E.shape)}")
        if self.n_channels is not None and E.shape[1] != self.n_channels:
            raise ValueError(f"{what} has {E.shape[1]} channels, the per-channel parameters {self.n_channels}")
        return E if E.is_contiguous() else E.contiguous()

    def forward(self, E):
        E = self._checked(E)
        params = self._params(E.device)
        # an empty E still goes through autograd: its backward gives an empty dE and zero parameter gradients, and
        # neither direction launches a kernel
        if torch.is_grad_enabled() and (E.requires_grad or any(p.requires_grad for p in params)):
            return _PCENFn.apply(E, *params, self.eps)
        if E.numel() == 0:
            return torch.empty(E.shape, dtype=torch.float32, device=E.device)
        return _C.pcen_forward(E, [p.detach() for p in params], self.eps)

    def extra_repr(self) -> str:
        return f"n_channels={self.n_channels}, eps={self.eps}, trainable={self.trainable}"


def _rows_map(v, what, R, device, limit=None):
    """A row -> value map of a step as the kernel reads it: an int32 (R,) device tensor.  A device tensor is taken as
    is (a step reads nothing on the host); CPU integers (a ``PoolOutput``'s) are checked, then copied."""
    if isinstance(v, torch.Tensor) and v.is_cuda:
        if v.device != device:
            raise TypeError(f"{what} must be on {device}, got {v.device}")
        if v.dtype != torch.int32 or tuple(v.shape) != (R,) or not v.is_contiguous():
            raise TypeError(f"{what} on the device must be a contiguous int32 ({R},) tensor, got {v.dtype} "
                            f"{tuple(v.shape)}")
        return v
    a = np.asarray(v.numpy() if isinstance(v, torch.Tensor) else v)
    if a.shape != (R,) or not (np.issubdtype(a.dtype, np.integer) or a.size == 0) or a.dtype == bool:
        raise ValueError(f"{what} must hold {R} integers, got {a.dtype} {a.shape}")
    lo, hi = limit
    if ((a < lo) | (a > hi)).any():
        raise ValueError(f"{what} must be in [{lo}, {hi}], got {a.tolist()}")
    host = torch.from_numpy(a.astype(np.int32)).pin_memory()
    return host.to(device, non_blocking=True)


class PCENStream:
    """``pcen`` applied to ``slots`` independent streams of frames as they arrive (forward only).

    ``PCENStream(pcen, slots, n_channels=None)`` keeps each slot's last smoother value and a primed flag on the
    device, (slots, C) each; C is ``pcen.n_channels``, else ``n_channels``, else the channel count of the first
    step.  ``step(frames, counts=None, slots=None)`` returns PCEN of ``frames`` (R, C, T), the same shape:
    row r belongs to slot ``slots[r]`` (None: slot r) and advances by ``counts[r]`` frames (None: all T); entries
    past a row's count are exact zeros and a slot without new frames keeps its state.  The three producers:

    * ``StreamingTransform.push`` output: ``step(frames)``;
    * a ``StreamPool`` ``PoolOutput``: ``step(out.frames, out.counts, out.slots)`` (CPU integers, checked);
    * ``DeviceStreamPool``: ``step(pool.frames, pool.counts)`` (int32 device counts, read on the device only).

    A slot that is not primed starts from its first frame, as the offline call does, so the concatenated steps of a
    stream equal ``pcen(whole)`` bit for bit.  ``reset(restart=None)`` un-primes the slots where the bool device mask
    ``restart`` is set (None: every slot) in one launch.  With device counts (or none) ``step`` and ``reset`` read
    nothing on the host, so a serving tick can be captured in a CUDA graph.
    """

    def __init__(self, pcen: PCEN, slots: int, n_channels=None):
        if not isinstance(pcen, PCEN):
            raise TypeError("pcen must be a nnaudio_b200.pcen.PCEN module")
        slots = int(slots)
        if slots < 1:
            raise ValueError(f"slots must be at least 1, got {slots}")
        self.pcen, self.slots = pcen, slots
        self.device = pcen.s.device  # a step refuses frames on any other device, and every CPU tensor
        C = pcen.n_channels if pcen.n_channels is not None else n_channels
        self.state = self.primed = None
        if C is not None and self.device.type == "cuda":
            self._allocate(int(C))

    def _allocate(self, C):
        self.state = torch.zeros((self.slots, C), dtype=torch.float32, device=self.device)
        self.primed = torch.zeros((self.slots, C), dtype=torch.uint8, device=self.device)

    def reset(self, restart=None):
        """Start new streams where the bool device mask ``restart`` (slots,) is set (None: every slot)."""
        mask = None if restart is None else _device_vector(restart, "restart", self.slots, torch.bool, self.device)
        if self.primed is not None:
            _C.pcen_reset(self.primed, mask)

    def step(self, frames, counts=None, slots=None):
        if isinstance(frames, torch.Tensor) and frames.requires_grad:
            raise NotImplementedError("PCENStream is forward-only: the frames require grad")
        frames = self.pcen._checked(frames, "frames")
        if frames.device != self.device:
            raise RuntimeError(f"frames are on {frames.device}: the stream state is on {self.device}")
        R, C, T = frames.shape
        if self.state is None:
            self._allocate(C)
        if C != self.state.shape[1]:
            raise ValueError(f"frames have {C} channels, the stream state {self.state.shape[1]}")
        if slots is None and R > self.slots:
            raise ValueError(f"frames have {R} rows for {self.slots} slots")
        if slots is not None:
            if not (isinstance(slots, torch.Tensor) and slots.is_cuda):
                a = np.asarray(slots.numpy() if isinstance(slots, torch.Tensor) else slots)
                if len(np.unique(a)) != a.size:
                    raise ValueError(f"slots must be distinct, got {a.tolist()}")
            slots = _rows_map(slots, "slots", R, self.device, (0, self.slots - 1))
        if counts is not None:
            counts = _rows_map(counts, "counts", R, self.device, (0, T))
        params = [p.detach() for p in self.pcen._params(self.device)]
        if frames.numel() == 0:
            return torch.empty(frames.shape, dtype=torch.float32, device=self.device)
        return _C.pcen_forward(frames, params, self.pcen.eps, stream_state=(self.state, self.primed),
                               row_slot=slots, counts=counts)
