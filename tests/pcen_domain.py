"""Float64 reference of PCEN (nnaudio_b200.pcen) and the inputs of its tests.

The reference is the spec: per channel c of a non-negative (B, C, T) spectrogram E,

    M[t] = (1 - s) M[t-1] + s E[t]          M[-1] = E[0]
    u[t] = E[t] (eps + M[t]) ** -gain
    P[t] = (bias + u[t]) ** power - bias ** power  =  bias ** power expm1(power log1p(u[t] / bias))

``smoother`` runs the recursion with scipy's ``lfilter`` (per channel), ``smoother_loop`` as a plain loop;
``reference`` is the NumPy forward, ``reference_torch`` the differentiable float64 forward the gradient tests
run autograd on, and ``naive_fp32`` the cancelling difference form in float32, which the accuracy test shows
failing where the kernel's expm1 / log1p form holds.
"""
from __future__ import annotations

import numpy as np
import torch

PARAMS = ("s", "gain", "bias", "power")


def _per_channel(v, C):
    """A parameter (scalar or (C,)) as a float64 (C,) array."""
    a = np.asarray(v.detach().cpu() if isinstance(v, torch.Tensor) else v, dtype=np.float64).reshape(-1)
    return np.broadcast_to(a, (C,)).copy()


def smoother_loop(E, s):
    """M of the spec by a direct loop over frames (float64)."""
    E = np.asarray(E, np.float64)
    B, C, T = E.shape
    s = _per_channel(s, C)[None, :]
    M = np.empty_like(E)
    if T == 0:
        return M
    m = E[:, :, 0].copy()
    for t in range(T):
        m = (1.0 - s) * m + s * E[:, :, t]
        M[:, :, t] = m
    return M


def smoother(E, s):
    """M of the spec with ``scipy.signal.lfilter``: y[t] = s x[t] + (1 - s) y[t-1], y[-1] = x[0]."""
    from scipy.signal import lfilter

    E = np.asarray(E, np.float64)
    B, C, T = E.shape
    M = np.empty_like(E)
    if T == 0:
        return M
    s = _per_channel(s, C)
    for c in range(C):
        a = 1.0 - s[c]
        M[:, c, :], _ = lfilter([s[c]], [1.0, -a], E[:, c, :], axis=-1, zi=(a * E[:, c, :1]))
    return M


def reference(E, s, gain, bias, power, eps, M=None):
    """(P, M, u) in float64 for a (B, C, T) E; the parameters are scalars or (C,)."""
    E = np.asarray(E, np.float64)
    C = E.shape[1]
    if M is None:
        M = smoother(E, s)
    col = lambda v: _per_channel(v, C)[None, :, None]  # noqa: E731
    u = E * (eps + M) ** -col(gain)
    P = col(bias) ** col(power) * np.expm1(col(power) * np.log1p(u / col(bias)))
    return P, M, u


def reference_torch(E, s, gain, bias, power, eps):
    """The differentiable float64 forward: E (B, C, T) and the parameters (scalars or (C,)) are float64 tensors."""
    T = E.shape[-1]
    col = lambda v: v.reshape(-1)[None, :] if v.dim() else v  # noqa: E731
    sc = col(s)
    m = E[:, :, 0]
    Ms = []
    for t in range(T):
        m = (1.0 - sc) * m + sc * E[:, :, t]
        Ms.append(m)
    M = torch.stack(Ms, -1)
    c3 = lambda v: v.reshape(-1)[None, :, None] if v.dim() else v  # noqa: E731
    u = E * (eps + M) ** -c3(gain)
    return c3(bias) ** c3(power) * torch.expm1(c3(power) * torch.log1p(u / c3(bias)))


def naive_fp32(E, M, gain, bias, power, eps):
    """The cancelling form ``(bias + u) ** power - bias ** power`` evaluated in float32 (torch tensors on any
    device; M the smoother output), for the test that shows the expm1 / log1p form is needed."""
    C = E.shape[1]
    dev = E.device
    c3 = lambda v: torch.tensor(_per_channel(v, C), dtype=torch.float32, device=dev)[None, :, None]  # noqa: E731
    u = E * (eps + M) ** -c3(gain)
    return (c3(bias) + u) ** c3(power) - c3(bias) ** c3(power)


def spectrogram(B, C, T, seed, lo=-10.0, hi=6.0, zeros=0.05):
    """A non-negative (B, C, T) float32 test spectrogram: per-row levels spread over 10**lo .. 10**hi, two decades
    of variation along time, and a fraction ``zeros`` of exact zeros."""
    rng = np.random.default_rng(seed)
    level = 10.0 ** rng.uniform(lo, hi, size=(B, C, 1))
    E = level * 10.0 ** rng.uniform(-1.0, 1.0, size=(B, C, T))
    E[rng.random((B, C, T)) < zeros] = 0.0
    return np.clip(E, 0.0, 10.0 ** hi).astype(np.float32)


def parameters(kind, C, seed=0):
    """(s, gain, bias, power) of a test: librosa's defaults at 16 kHz / hop 160 (``"scalar"``), or per channel
    values spread around them (``"channel"``)."""
    s0 = 0.024689
    if kind == "scalar":
        return s0, 0.98, 2.0, 0.5
    rng = np.random.default_rng(1000 + seed)
    return (rng.uniform(0.01, 0.2, C), rng.uniform(0.5, 1.0, C), rng.uniform(0.5, 4.0, C),
            rng.uniform(0.25, 0.75, C))
