"""Float64 reference of PCEN (nnaudio_b200.pcen) and the inputs of its tests.

The reference is the spec: per channel c of a non-negative (B, C, T) spectrogram E,

    M[t] = (1 - s) M[t-1] + s E[t]          M[-1] = E[0]
    u[t] = E[t] (eps + M[t]) ** -gain
    P[t] = (bias + u[t]) ** power - bias ** power  =  bias ** power expm1(power log1p(u[t] / bias))

``smoother`` runs the recursion with scipy's ``lfilter`` (per channel), ``smoother_loop`` as a plain loop;
``reference`` is the NumPy forward, ``reference_torch`` the differentiable float64 forward the gradient tests
run autograd on, and ``naive_fp32`` the cancelling difference form in float32, which the accuracy test shows
failing where the kernel's expm1 / log1p form holds.

``reference_grad`` is the analytic float64 adjoint (a time-reversed ``lfilter``), fast enough for cfg2 and long
rows; ``forward_bound`` / ``backward_bound`` bound the kernels' float32 error elementwise from their expression
order; ``emulate_forward`` / ``emulate_backward`` replay that order in NumPy float32, with planted slips
(``MUTATIONS``) the bounds must catch; ``ROWS`` is the shape and parameter matrix and ``launch_model`` the kernels
each call launches.
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


# ================================================================================ float64 adjoint ====
def _revfilter(x, a):
    """y[t] = x[t] + a y[t+1] along the last axis (y[T] = 0), a per channel: the adjoint recurrence as a
    time-reversed ``lfilter``.  x is (B, C, T), a (C,)."""
    from scipy.signal import lfilter

    y = np.empty_like(x)
    for c in range(x.shape[1]):
        y[:, c, ::-1] = lfilter([1.0], [1.0, -a[c]], x[:, c, ::-1], axis=-1)
    return y


def _terms(E, s, gain, bias, power, eps, M=None):
    """The float64 quantities of the forward and its derivatives, elementwise (B, C, T), with the parameters as
    (1, C, 1) columns: M, me = eps + M, scale = me^-gain, u, l = log1p(u / bias), w = power l, dP/du."""
    E = np.asarray(E, np.float64)
    C = E.shape[1]
    col = lambda v: _per_channel(v, C)[None, :, None]  # noqa: E731
    s3, g3, b3, r3 = col(s), col(gain), col(bias), col(power)
    if M is None:
        M = smoother(E, s)
    me = eps + M
    scale = me ** -g3
    u = E * scale
    l = np.log1p(u / b3)
    dPdu = r3 * b3 ** (r3 - 1.0) * np.exp((r3 - 1.0) * l)
    return dict(E=E, M=M, me=me, scale=scale, u=u, l=l, w=r3 * l, dPdu=dPdu, s=s3, gain=g3, bias=b3, power=r3)


def _grad_parts(q, W, Mp):
    """dE's direct term D, dP/dM's local term g_M and the per-element terms of the four parameter gradients, from
    the forward quantities ``q`` of ``_terms`` (G, the adjoint of M, enters ds separately)."""
    gu = W * q["dPdu"]
    b3, r3 = q["bias"], q["power"]
    return dict(
        D=gu * q["scale"],
        gM=-q["gain"] * gu * q["u"] / q["me"],
        gain=-gu * q["u"] * np.log(q["me"]),
        bias=W * r3 * b3 ** (r3 - 1.0) * np.expm1((r3 - 1.0) * q["l"]),
        power=W * b3 ** r3 * (np.log(b3) * np.expm1(q["w"]) + np.exp(q["w"]) * q["l"]),
        diff=q["E"] - Mp)


def _prev(E, M):
    """M[t - 1], with M[-1] = E[0]."""
    return np.concatenate([E[:, :, :1], M[:, :, :-1]], axis=2)


def _sum_param(x, per_channel):
    return x.sum(axis=(0, 2)) if per_channel else np.asarray(x.sum())


def reference_grad(E, s, gain, bias, power, eps, W, per_channel=None):
    """The float64 gradients of sum(P * W): {"E": (B, C, T), "s" / "gain" / "bias" / "power": (C,) per channel or
    () for scalars}.  The adjoint of M runs backwards in time,

        G[t] = g_M[t] + (1 - s) G[t + 1],   g_M = dP/dM = -gain W dP/du u / (eps + M)
        dE[t] = W dP/du (eps + M)^-gain + s G[t],  dE[0] += (1 - s) G[0]   (M[-1] = E[0])
        ds = sum_t G[t] (E[t] - M[t - 1])

    as a time-reversed ``lfilter`` per channel; the gain, bias and power gradients are sums of closed-form
    per-element terms."""
    E = np.asarray(E, np.float64)
    W = np.asarray(W, np.float64)
    C = E.shape[1]
    if per_channel is None:
        per_channel = np.asarray(s).size > 1
    q = _terms(E, s, gain, bias, power, eps)
    parts = _grad_parts(q, W, _prev(E, q["M"]))
    sc = _per_channel(s, C)
    G = _revfilter(parts["gM"], 1.0 - sc)
    dE = parts["D"] + q["s"] * G
    dE[:, :, 0] += (1.0 - q["s"][:, :, 0]) * G[:, :, 0]
    out = {"E": dE, "s": _sum_param(G * parts["diff"], per_channel)}
    for n in ("gain", "bias", "power"):
        out[n] = _sum_param(parts[n], per_channel)
    return out


# ================================================================================ error bounds ====
# The kernels' float32 error against the float64 spec, bounded elementwise from their expression order
# (csrc/pcen_kernels.cu).  U = 2^-24 is float32's unit roundoff: +, *, / and fma round once (<= U relative), and
# a CUDA function with a documented maximum error of k ulp (CUDA C Programming Guide, single-precision
# mathematical functions, full range, built without fast math) is within 2 k U of its exact value relative to
# it.  The bounds are first order in U; the inputs E, W and the parameters are float32 values, and the reference
# takes eps as the float32 value the kernel reads.
U = 2.0 ** -24
ULP = {"exp2f": 2, "log2f": 1, "log1pf": 1, "expm1f": 1, "powf": 4, "expf": 2, "logf": 1}
R = {k: 2.0 * v * U for k, v in ULP.items()}  # relative error of each function


def eps32(eps):
    """eps as the kernels read it (a float32 argument)."""
    return float(np.float32(eps))


def smoother_bound(E, s, M=None):
    """b[t] >= |m[t] - M[t]| for the kernel's m = fma(fl(1 - s), m, fl(s E[t])) from m = E[0].

    Each step rounds three times: fl(1 - s) by U (1 - s), s E[t] by U s E[t], the fma by U M[t]; since
    (1 - s) M[t-1] + s E[t] = M[t] these sum to 2 U M[t].  The carried error is multiplied by fl(1 - s) <=
    (1 - s)(1 + U), so b[t] = (1 - s)(1 + 2U) b[t-1] + 2 U (M[t] + s E[t]) with b[-1] = 0, the s E[t] term
    absorbing the second-order products: run with the same ``lfilter`` as M.  In a long-memory channel b / M
    settles near 2 U / s."""
    from scipy.signal import lfilter

    E = np.asarray(E, np.float64)
    B, C, T = E.shape
    if M is None:
        M = smoother(E, s)
    sc = _per_channel(s, C)
    b = np.empty_like(E)
    for c in range(C):
        b[:, c, :] = lfilter([1.0], [1.0, -(1.0 - sc[c]) * (1.0 + 2.0 * U)],
                             2.0 * U * (M[:, c, :] + sc[c] * E[:, c, :]), axis=-1)
    return b


def _scale_rel(q):
    """Relative error of the kernel's (eps + m)^-gain = exp2f(-gain log2f(me)) besides the smoother's own: me's
    rounding U; log2f 2 U |log2 me| and the product -gain L U |gain L|, so the exponent is off by
    gain (3 U |log2 me| + U / ln 2); exp2f's own 4 U; an exponent error dx costs ln 2 dx relative."""
    return q["gain"] * (3.0 * U * np.abs(np.log(q["me"])) + U) + R["exp2f"]


def forward_bound(E, s, gain, bias, power, eps):
    """An elementwise bound on |P_fp32 - P_f64| of the forward kernel (offline and streamed calls alike).

    With b the smoother's bound, me = eps + M and rho_me = b / me + U:
      scale = exp2f(-gain log2f(me)):  rho_sc = gain (rho_me + 3 U |ln me|) + 4 U          (``_scale_rel``)
      u = E scale, v = u / bias:       rho_v = rho_sc + 2 U
      l = log1pf(v):                   dl = v / (1 + v) rho_v + 2 U l
      w = power l:                     dw = power dl + U w
      P = fl(powf(bias, power) expm1f(w)): (bias + u)^power dw + |P| (2 U expm1f + 8 U powf + U)
    and power (bias + u)^power v / (1 + v) = dP/du u, so
      |dP| <= dP/du u rho_v + 3 U (bias + u)^power w + 11 U |P|."""
    eps = eps32(eps)
    q = _terms(E, s, gain, bias, power, eps)
    b = smoother_bound(E, s, q["M"])
    rho_v = q["gain"] * (b / q["me"]) + _scale_rel(q) + 2.0 * U
    P = q["bias"] ** q["power"] * np.expm1(q["w"])
    big = (q["bias"] + q["u"]) ** q["power"]
    return q["dPdu"] * q["u"] * rho_v + 3.0 * U * big * q["w"] + (R["expm1f"] + R["powf"] + U) * np.abs(P)


def _n_reduce(n):
    """Additions of the reduction kernel on one value: its 256-thread strided sum, then the 8-level tree."""
    return -(-n // 256) + 8


def gamma(n):
    return n * U / (1.0 - n * U)


def _local_errors(q, W, Mp, bMp):
    """Absolute rounding errors of the backward kernel's per-element values at the float32 M, first order:
    (errors, magnitudes) dicts keyed like ``_grad_parts``.  The expression order is the kernel's:

      scale = exp2f(-gain log2f(me)), u = e scale, l = log1pf(u / bias)           rho_sc, rho_u = rho_sc + U
      gu = ((g power) powf(bias, power - 1)) expf((power - 1) l)               3 U + 8 U + 4 U + |x| dl-terms
      D = gu scale;  g_M = ((-gain gu) u) / me;  gain term (gu u) logf(me)
      bias term ((g power) powf(bias, power - 1)) expm1f((power - 1) l)
      power term (g powf(bias, power)) (logf(bias) expm1f(w) + expf(w) l)"""
    g3, b3, r3 = q["gain"], q["bias"], q["power"]
    rho_sc = _scale_rel(q)
    rho_u = rho_sc + U
    v = q["u"] / b3
    l = q["l"]
    dl = v / (1.0 + v) * (rho_u + U) + R["log1pf"] * l
    x = (r3 - 1.0) * l
    dx = np.abs(r3 - 1.0) * (dl + 2.0 * U * l)
    rho_b1 = R["powf"] + U * np.abs(np.log(b3) * (r3 - 1.0))  # powf(bias, fl(power - 1))
    gu = W * q["dPdu"]
    rho_gu = 3.0 * U + rho_b1 + dx + R["expf"]
    p = _grad_parts(q, W, Mp)
    err, mag = {}, {}
    err["D"] = np.abs(p["D"]) * (rho_gu + rho_sc + U)
    err["gM"] = np.abs(p["gM"]) * (rho_gu + rho_u + 4.0 * U)
    lnme = np.log(q["me"])
    err["gain"] = np.abs(gu * q["u"]) * (np.abs(lnme) * (rho_gu + rho_u + 2.0 * U + R["logf"]) + U)
    em1 = np.expm1(x)
    bw = W * r3 * b3 ** (r3 - 1.0)
    err["bias"] = np.abs(bw) * (np.exp(x) * dx + np.abs(em1) * (R["expm1f"] + 3.0 * U + rho_b1))
    w = q["w"]
    dw = r3 * dl + U * w
    em, ew, lb = np.expm1(w), np.exp(w), np.log(b3)
    A, Bq = np.abs(lb * em), ew * l
    dA = np.abs(lb) * (ew * dw + R["expm1f"] * np.abs(em)) + A * (R["logf"] + U)
    dB = l * ew * (dw + R["expf"]) + ew * dl + U * Bq
    gb = np.abs(W) * b3 ** r3
    err["power"] = gb * (dA + dB + U * (A + Bq) + (A + Bq) * (R["powf"] + 2.0 * U))
    mag["power"] = gb * (A + Bq)
    err["diff"] = bMp + U * np.abs(p["diff"])
    for n in ("D", "gM", "gain", "bias", "diff"):
        mag[n] = np.abs(p[n])
    return p, err, mag


def _m_sensitivity(E, s, gain, bias, power, eps, W, M, b):
    """|f(M +- b) - f(M)| of every per-element value f of ``_grad_parts``: the float32 M the backward reads is
    within b of the exact one (forward of a training call), propagated by evaluation rather than by hand."""
    base = _grad_parts(_terms(E, s, gain, bias, power, eps, M), W, _prev(E, M))
    out = {k: np.zeros_like(v) for k, v in base.items()}
    for sign in (1.0, -1.0):
        Ms = np.maximum(M + sign * b, 0.0)
        pert = _grad_parts(_terms(E, s, gain, bias, power, eps, Ms), W, _prev(E, M))
        for k in base:
            if k != "diff":
                out[k] = np.maximum(out[k], np.abs(pert[k] - base[k]))
    return out


def backward_bound(E, s, gain, bias, power, eps, W, per_channel=None):
    """Bounds on |grad_fp32 - grad_f64| of the backward kernel and the reduction, for ``reference_grad``'s keys.

    Per element every value of ``_grad_parts`` carries its own rounding (``_local_errors``) plus the float32 M's
    error b propagated through it (``_m_sensitivity``).  The adjoint G = fma(fl(1 - s), G, g_M) runs backwards,
    with H = revfilter(|g_M|) >= |G|: dG[t] = (1 - s)(1 + 2U) dG[t+1] + dg_M[t] + 2 U H[t].  Then
      dE = fma(s, G, D) (and fma(1 - s, G[0], .) at t = 0):  |d dE| <= dD + s dG + U (|D| + s H)  (+ the t = 0 terms)
      ds = sum_t fma(G, fl(E - M[t-1]), .):  sum_t dG |E - M[t-1]| + H d(E - M[t-1]) + gamma_n sum |terms|
      gain, bias, power:  sum of term errors + gamma_n sum |terms|
    where n counts the additions a term passes through: its per-thread register sum over the row's 64-frame tiles,
    the 64-column row sum and the reduction (strided sum and 8-level tree) over B (per channel) or B C rows; ds
    sums all T frames in one register before the reduction."""
    eps = eps32(eps)
    E = np.asarray(E, np.float64)
    W = np.asarray(W, np.float64)
    B, C, T = E.shape
    if per_channel is None:
        per_channel = np.asarray(s).size > 1
    q = _terms(E, s, gain, bias, power, eps)
    M = q["M"]
    b = smoother_bound(E, s, M)
    bMp = _prev(np.zeros_like(E), b)
    p, err, mag = _local_errors(q, W, _prev(E, M), bMp)
    sens = _m_sensitivity(E, s, gain, bias, power, eps, W, M, b)
    for k in sens:
        if k != "diff":
            err[k] = err[k] + sens[k]
    sc = _per_channel(s, C)
    H = _revfilter(mag["gM"], 1.0 - sc)
    dG = _revfilter(err["gM"] + 2.0 * U * H, (1.0 - sc) * (1.0 + 2.0 * U))
    s3 = q["s"]
    dE = err["D"] + s3 * dG + U * (mag["D"] + s3 * H)
    dE[:, :, 0] += (1.0 - s3[:, :, 0]) * (dG[:, :, 0] + 2.0 * U * H[:, :, 0]) + U * (mag["D"][:, :, 0] + H[:, :, 0])
    n_red = _n_reduce(B if per_channel else B * C)
    n_tiles = -(-T // 64)
    out = {"E": dE}
    ds_err = dG * mag["diff"] + (H + dG) * err["diff"]
    ds_mag = (H + dG) * (mag["diff"] + err["diff"])
    out["s"] = _sum_param(ds_err, per_channel) + gamma(T + n_red) * _sum_param(ds_mag, per_channel)
    n = n_tiles + 64 + n_red
    for k in ("gain", "bias", "power"):
        out[k] = _sum_param(err[k], per_channel) + gamma(n) * _sum_param(mag[k] + err[k], per_channel)
    return out


def ratio(diff, bound):
    """max |diff| / bound, elementwise; 0 / 0 counts 0, anything over a zero bound infinity."""
    d = np.abs(np.asarray(diff, np.float64))
    bd = np.broadcast_to(np.asarray(bound, np.float64), d.shape)
    if d.size == 0:
        return 0.0
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(d == 0.0, 0.0, d / bd)
    return float(np.nan_to_num(r, nan=np.inf).max())


# ================================================================================ float32 emulation ====
# The kernels' op order in NumPy float32: +, *, / rounded by NumPy, fma as a float64 op rounded once, and the
# transcendental functions evaluated in float64 and rounded once (correctly rounded: the CUDA functions may be
# a few ulp further off, which the bounds budget for).  ``mutate`` plants one of the slips the bounds must catch.
MUTATIONS = ("shift_M", "ds_uses_M_t", "no_dE0", "drop_last_tile", "reduce_next_channel", "gain_sign_flipped",
             "s_perturbed")
_f32, _f64 = np.float32, np.float64


def _fn(f, x):
    return f(np.asarray(x, _f64)).astype(_f32)


def _powf(b, e):
    return np.power(np.asarray(b, _f64), np.asarray(e, _f64)).astype(_f32)


def _fma(a, b, c):
    return (np.asarray(a, _f64) * np.asarray(b, _f64) + np.asarray(c, _f64)).astype(_f32)


def _row_params(C, B, s, gain, bias, power, mutate=None):
    s64 = _per_channel(s, C) * (1.0 - 1e-4 if mutate == "s_perturbed" else 1.0)
    return [np.tile(_per_channel(v, C), B).astype(_f32) for v in (s64, gain, bias, power)]


def emulate_forward(E, s, gain, bias, power, eps, mutate=None):
    """(P, M) of the forward kernel in emulated float32, (B, C, T) each."""
    E = np.asarray(E, _f32)
    B, C, T = E.shape
    sr, g, bi, pw = (v[:, None] for v in _row_params(C, B, s, gain, bias, power, mutate))
    X = E.reshape(B * C, T)
    M = np.empty_like(X)
    oms = _f32(1.0) - sr[:, 0]
    m = X[:, 0].copy() if T else None
    for t in range(T):
        m = _fma(oms, m, sr[:, 0] * X[:, t])
        M[:, t] = m
    Mc = np.concatenate([X[:, :1], M[:, :-1]], 1) if mutate == "shift_M" else M
    me = _f32(eps) + Mc
    scale = _fn(np.exp2, -g * _fn(np.log2, me))
    u = X * scale
    l = _fn(np.log1p, u / bi)
    P = _powf(bi, pw) * _fn(np.expm1, pw * l)
    return P.reshape(B, C, T), M.reshape(B, C, T)


def emulate_backward(E, M, W, s, gain, bias, power, eps, per_channel, mutate=None):
    """(dE (B, C, T), {"s", "gain", "bias", "power"}) of the backward kernel and the reduction in emulated float32:
    the reverse tile walk, the per-(row, frame column) register partials, the 64-column row sums and the
    reduction's 256-way strided sums and tree."""
    E, M, W = (np.asarray(a, _f32) for a in (E, M, W))
    B, C, T = E.shape
    R = B * C
    sr, g, bi, pw = (v[:, None] for v in _row_params(C, B, s, gain, bias, power))
    X, Mx, Wx = E.reshape(R, T), M.reshape(R, T), W.reshape(R, T)
    oms = _f32(1.0) - sr[:, 0]
    bR, bR1 = _powf(bi, pw), _powf(bi, pw - _f32(1.0))
    lb = _fn(np.log, bi)
    eps = _f32(eps)
    acc = {k: np.zeros((R, 64), _f32) for k in ("gain", "bias", "power")}
    G = np.zeros(R, _f32)
    ds = np.zeros(R, _f32)
    dE = np.zeros((R, T), _f32)
    n_tiles = -(-T // 64)
    for ti in range(n_tiles - 1, -1, -1):
        t0 = ti * 64
        tw = min(64, T - t0)
        if mutate == "drop_last_tile" and ti == n_tiles - 1 and tw < 64:
            continue
        e, mm, gp = X[:, t0:t0 + tw], Mx[:, t0:t0 + tw], Wx[:, t0:t0 + tw]
        mprev = np.concatenate([(Mx[:, t0 - 1] if t0 > 0 else X[:, 0])[:, None], mm[:, :-1]], 1)
        me = eps + mm
        scale = _fn(np.exp2, -g * _fn(np.log2, me))
        u = e * scale
        l = _fn(np.log1p, u / bi)
        w = pw * l
        gu = gp * pw * bR1 * _fn(np.exp, (pw - _f32(1.0)) * l)
        sD = gu * scale
        sG = -g * gu * u / me
        if mutate == "gain_sign_flipped":
            sG = -sG
        acc["gain"][:, :tw] -= gu * u * _fn(np.log, me)
        acc["power"][:, :tw] += gp * bR * (lb * _fn(np.expm1, w) + _fn(np.exp, w) * l)
        acc["bias"][:, :tw] += gp * pw * bR1 * _fn(np.expm1, (pw - _f32(1.0)) * l)
        ref_m = mm if mutate == "ds_uses_M_t" else mprev
        for k in range(tw - 1, -1, -1):
            G = _fma(oms, G, sG[:, k])
            ds = _fma(G, e[:, k] - ref_m[:, k], ds)
            d = _fma(sr[:, 0], G, sD[:, k])
            if t0 + k == 0 and mutate != "no_dE0":
                d = _fma(oms, G, d)
            dE[:, t0 + k] = d
    partial = {"s": ds}
    for k, a in acc.items():
        tot = np.zeros(R, _f32)
        for j in range(64):
            tot = tot + a[:, j]
        partial[k] = tot
    grads = {}
    for k, p in partial.items():
        if per_channel:
            shift = 1 if mutate == "reduce_next_channel" else 0
            grads[k] = np.array([_reduce(p.reshape(B, C)[:, (c + shift) % C]) for c in range(C)], _f32)
        else:
            grads[k] = np.asarray(_reduce(p))
    return dE.reshape(B, C, T), grads


def _reduce(p):
    """The reduction kernel on one output: 256 strided float32 sums in index order, then the tree."""
    red = np.zeros(256, _f32)
    for i in range(0, p.size, 256):
        chunk = p[i:i + 256]
        red[:chunk.size] = red[:chunk.size] + chunk
    h = 128
    while h:
        red[:h] = red[:h] + red[h:2 * h]
        h //= 2
    return red[0]


# ================================================================================ the matrix ====
LIBROSA = (0.024689, 0.98, 2.0, 0.5)
# scalar parameter sets, (s, gain, bias, power, eps): librosa's defaults and each constructor boundary
PARAM_SETS = {
    "librosa": LIBROSA + (1e-6,),
    "s_one": (1.0, 0.98, 2.0, 0.5, 1e-6),      # no memory: M = E, fl(1 - s) = 0
    "s_long": (1e-3, 0.98, 2.0, 0.5, 1e-6),    # long memory: the recurrence's rounding builds to ~2 U / s
    "gain_zero": (0.024689, 0.0, 2.0, 0.5, 1e-6),
    "gain_two": (0.024689, 2.0, 2.0, 0.5, 1e-6),
    "bias_small": (0.024689, 0.98, 1e-3, 0.5, 1e-6),
    "bias_large": (0.024689, 0.98, 1e3, 0.5, 1e-6),
    "power_small": (0.024689, 0.98, 2.0, 0.05, 1e-6),
    "power_one": (0.024689, 0.98, 2.0, 1.0, 1e-6),  # the bias gradient is exactly zero
    "power_two": (0.024689, 0.98, 2.0, 2.0, 1e-6),
    "eps_tiny": (0.024689, 0.98, 2.0, 0.5, 1e-12),
    "eps_one": (0.024689, 0.98, 2.0, 0.5, 1.0),     # eps dominates M in the quiet rows
}
# one extreme per channel, cycled over the channels of the ``mix`` rows
EXTREMES = [(1.0, 0.98, 2.0, 0.5), (1e-3, 0.98, 2.0, 0.5), (0.024689, 0.0, 2.0, 0.5), (0.024689, 2.0, 2.0, 0.5),
            (0.024689, 0.98, 1e-3, 0.5), (0.024689, 0.98, 1e3, 0.5), (0.024689, 0.98, 2.0, 0.05),
            (0.024689, 0.98, 2.0, 1.0), (0.024689, 0.98, 2.0, 2.0)]


def _row(B, C, T, prm="librosa", edge="", kinds=("scalar", "channel")):
    return dict(B=B, C=C, T=T, prm=prm, edge=edge, kinds=kinds)


# one edge per row: 32 rows per block, 64 frames per tile (both kernels)
ROWS = {
    **{f"T{T}": _row(2, 40, T, edge=e) for T, e in (
        (1, "one frame: the settled start is the whole row"),
        (2, "two frames: the backward's dE[0] term next to one scan step"),
        (63, "one partial tile"),
        (64, "exactly one tile: the prefetch never runs"),
        (65, "a full tile then a 1-frame tile: the reverse walk starts on the partial tile"),
        (127, "a full tile then a 63-frame tile"),
        (128, "two full tiles: sM[r][0] = M[63] hands over between them"),
        (129, "two full tiles and a 1-frame tile"),
        (431, "six full tiles and a 47-frame tile (cfg2's frame count)"))},
    "rows1": _row(1, 1, 130, edge="one row: a block of 31 idle lanes"),
    "rows31": _row(31, 1, 65, edge="31 rows: one partial block"),
    "rows32": _row(32, 1, 65, edge="32 rows: exactly one block"),
    "rows33": _row(33, 1, 65, edge="33 rows: a full block and a 1-row block"),
    "rows514": _row(2, 257, 65, edge="C = 257: blocks span batch rows, a 2-row last block"),
    "cfg2": _row(256, 128, 431, edge="cfg2's training size: 1024 blocks, the reduction over 256 or 32768 rows"),
    "long": _row(1, 40, 120_000, edge="one long row: 1875 tiles per thread in the backward"),
    **{f"prm_{k}": _row(3, 40, 200, prm=k, edge=f"parameter boundary {k}") for k in PARAM_SETS if k != "librosa"},
    "s_long_settled": _row(1, 8, 8000, prm="s_long", edge="s = 1e-3 over 8 time constants: the settled error"),
    "mix": _row(3, 40, 129, prm="mix", kinds=("channel",),
                edge="a different extreme per channel: a c = row % C or parameter-stride slip"),
}
ROWS.pop("prm_s_long")
BIG = ("cfg2", "long")  # too large for the float32 emulation on the host


def params_of(row, kind, seed=0):
    """(s, gain, bias, power, eps) of a row: scalars, or per channel (C,) arrays.  A per-channel variant of a
    scalar set scales each channel's values by a factor in [0.6, 1] (every boundary stays inside the domain)."""
    C = row["C"]
    if row["prm"] == "mix":
        ex = np.array([EXTREMES[c % len(EXTREMES)] for c in range(C)])
        return tuple(ex[:, i].astype(np.float32) for i in range(4)) + (1e-6,)
    vals = PARAM_SETS[row["prm"]]
    if kind == "scalar":
        return tuple(np.float32(v) for v in vals[:4]) + (vals[4],)
    rng = np.random.default_rng(2000 + seed)
    return tuple((v * rng.uniform(0.6, 1.0, C)).astype(np.float32) for v in vals[:4]) + (vals[4],)


def problem(row, seed):
    """(E, W) float32 of a row: row r of the B C rows gets input pattern r % 6 (levels over 1e-10 .. 1e6 twice,
    all zeros, a zero first frame then loud frames, impulses, a constant), W the gradient of the output."""
    B, C, T = row["B"], row["C"], row["T"]
    rng = np.random.default_rng(seed)
    R = B * C
    level = 10.0 ** rng.uniform(-10.0, 6.0, (R, 1))
    E = level * 10.0 ** rng.uniform(-1.0, 1.0, (R, T))
    pat = np.arange(R) % 6
    E[pat == 2] = 0.0
    loud = pat == 3
    E[loud] = 10.0 ** rng.uniform(4.0, 6.0, (int(loud.sum()), T))
    E[loud, 0] = 0.0
    imp = pat == 4
    spikes = (rng.random((int(imp.sum()), T)) < 0.05) * 10.0 ** rng.uniform(0.0, 6.0, (int(imp.sum()), T))
    spikes[:, 0] = 10.0 ** rng.uniform(0.0, 6.0, int(imp.sum()))
    E[imp] = spikes
    E[pat == 5] = level[pat == 5]
    E = np.clip(E, 0.0, 1e6).astype(np.float32).reshape(B, C, T)
    W = rng.standard_normal((B, C, T)).astype(np.float32)
    return E, W


# ================================================================================ launch model ====
KERNELS = ("pcen_forward_kernel", "pcen_backward_kernel", "pcen_param_reduce_kernel", "pcen_reset_kernel")


def launch_model(call):
    """The kernels one call launches, in order.  ``call``: dict(kind = "inference" | "train" | "step" | "reset",
    B, C, T, and for "train" want_E / want_params).  An empty spectrogram launches nothing: its parameter gradients
    are cleared by a memset."""
    kind = call["kind"]
    if kind == "reset":
        return ["pcen_reset_kernel"]
    if call["B"] * call["C"] * call["T"] == 0:
        return []
    out = ["pcen_forward_kernel"]
    if kind == "train":
        if call["want_E"] or call["want_params"]:
            out.append("pcen_backward_kernel")
        if call["want_params"]:
            out.append("pcen_param_reduce_kernel")
    return out


def layout(B, C, T):
    """The edges a (B, C, T) call reaches: tiles, the last tile's width, blocks, the last block's rows, and whether
    some block holds rows of two batch entries."""
    R = B * C
    blocks = -(-R // 32)
    spans = any((32 * i) // C != (min(32 * i + 31, R - 1)) // C for i in range(blocks))
    return dict(tiles=-(-T // 64), last_tile=T - 64 * (-(-T // 64) - 1) if T else 0, blocks=blocks,
                last_block=R - 32 * (blocks - 1), spans_batch=spans)
