"""Test infrastructure only: float64 torch stand-ins for the C entry points the host modules call
(forward family, the dX / dW pair, the inverse) with the semantics include/nnab.h documents.  Patched over
``nnaudio_b200._C`` they let the CPU suite check the host-side autograd wiring — which stages
are chained, which padding each one uses, how octave gradients are summed, how the one-sided
mirror is folded — against the reference's autograd goldens without a GPU.  The kernels
themselves are checked on the GPU by tests/test_backward.py; nothing here ships.
"""
from __future__ import annotations

import numpy as np
import torch

from nnaudio_b200 import _C


def _pad(x, pad, pad_mode):
    if pad == 0:
        return x
    mode = "reflect" if pad_mode == _C.PAD_REFLECT else "constant"
    return torch.nn.functional.pad(x[:, None, :], (pad, pad), mode=mode)[:, 0, :]


def _framed(x, w_re, w_im, hop, center, pad_mode):
    """(B, L), (F, K) x2 -> (B, F, T, 2) = (conv(x, w_re), -conv(x, w_im)) in float64."""
    K = w_re.shape[1]
    xp = _pad(x.double(), K // 2 if center else 0, pad_mode)[:, None, :]
    re = torch.nn.functional.conv1d(xp, w_re.double()[:, None, :], stride=hop)
    im = -torch.nn.functional.conv1d(xp, w_im.double()[:, None, :], stride=hop)
    return torch.stack((re, im), -1)


def _scaled(c, scale, scale_all):
    if scale is not None:
        c = c * scale.double().view(1, -1, 1, 1)
    return c * scale_all


def _format(c, out_format, sqrt_eps):
    """The output formats of include/nnab.h on a float64 (B, F, T, 2) complex tensor."""
    re, im = c[..., 0], c[..., 1]
    if out_format == _C.FMT_COMPLEX:
        return c.float()
    if out_format == _C.FMT_MAGNITUDE:
        return torch.sqrt(re * re + im * im + sqrt_eps).float()
    if out_format == _C.FMT_PHASE_ANGLE:
        return torch.atan2(im, re).float()
    if out_format == _C.FMT_PHASE_UNIT:
        ang = torch.atan2(im, re)
        return torch.stack((torch.cos(ang), torch.sin(ang)), -1).float()
    raise ValueError(out_format)


def _mat(w):
    return w.reshape(w.shape[0], -1)


def cqt1992v2_forward(x, k_real, k_imag, packed, k_begin, k_end, hop, center, pad_mode, scale,
                      scale_all, out_format, sqrt_eps, path=None):
    c = _framed(x, k_real, k_imag, hop, center, pad_mode)
    return _format(_scaled(c, scale, scale_all), out_format, sqrt_eps)


def stft_forward(x, wcos, wsin, packed, n_fft, hop, center, pad_mode, out_format, sqrt_eps, path=None):
    return _format(_framed(x, _mat(wcos), _mat(wsin), hop, center, pad_mode), out_format, sqrt_eps)


def _mel_power(x, wcos, wsin, hop, center, pad_mode, sqrt_eps, power, fb):
    c = _framed(x, _mat(wcos), _mat(wsin), hop, center, pad_mode)
    mag = torch.sqrt(c[..., 0] ** 2 + c[..., 1] ** 2 + sqrt_eps)
    return torch.matmul(fb.double(), mag ** power)


def stft_filterbank_forward(x, wcos, wsin, packed, n_fft, hop, center, pad_mode, sqrt_eps, power, fb,
                            fb_table=None, path=None):
    return _mel_power(x, wcos, wsin, hop, center, pad_mode, sqrt_eps, power, fb).float()


def mfcc_forward(x, wcos, wsin, packed, n_fft, hop, center, pad_mode, sqrt_eps, power, mel_basis, amin,
                 ref, top_db, dct, fb_table=None, path=None):
    """nnab_mfcc_forward: mel power -> 10 log10(max(S, amin)) - 10 log10(max(amin, |ref|)), per-clip
    top_db floor, orthonormal DCT-II rows (mel.py:263-307)."""
    S = _mel_power(x, wcos, wsin, hop, center, pad_mode, sqrt_eps, power, mel_basis)
    db = 10.0 * torch.log10(torch.clamp(S, min=amin)) - 10.0 * np.log10(max(amin, abs(ref)))
    if top_db is not None:
        db = torch.maximum(db, db.amax(dim=(1, 2), keepdim=True) - top_db)
    return torch.matmul(dct.double(), db).float()


def cqt_pyramid_forward(x, banks_real, banks_imag, packed, lowpass, lowpass_packed, early_filter,
                        early_packed, early_factor, hop, pad_mode, n_bins, scale, scale_all, out_format,
                        sqrt_eps, T, path=None):
    """nnab_cqt_pyramid_forward: optional early decimation, then per octave (top first) the bank at
    hop / 2^i on the i-times halved signal; reflect padding falls back to zeros when the level is
    too short; octaves stacked low -> high, lowest surplus bins dropped."""
    cur = x.double()
    if early_filter is not None and early_factor > 1:
        cur = fir_decimate(cur, early_filter, early_factor).double()
    octaves = []
    for i, (kr, ki) in enumerate(zip(banks_real, banks_imag)):
        if i > 0:
            cur = fir_decimate(cur, lowpass, 2).double()
            hop //= 2
        mode = pad_mode
        if pad_mode == _C.PAD_REFLECT and kr.shape[1] // 2 >= cur.shape[-1]:
            mode = _C.PAD_CONSTANT
        octaves.insert(0, _framed(cur, kr, ki, hop, True, mode))
    c = torch.cat(octaves, 1)[:, -n_bins:]
    assert c.shape[2] == T
    return _format(_scaled(c, scale, scale_all), out_format, sqrt_eps)


def framed_backward_input(g, packed_adj, K, hop, center, pad_mode, L_in):
    w_re, w_im = packed_adj
    x = torch.zeros((g.shape[0], L_in), dtype=torch.float64, requires_grad=True)
    with torch.enable_grad():
        y = _framed(x, w_re, w_im, hop, center, pad_mode)
        (dx,) = torch.autograd.grad(y, x, g.double())
    return dx.float()


def framed_backward_weight(g, x, K, hop, center, pad_mode):
    F = g.shape[1]
    w_re = torch.zeros((F, K), dtype=torch.float64, requires_grad=True)
    w_im = torch.zeros((F, K), dtype=torch.float64, requires_grad=True)
    with torch.enable_grad():
        y = _framed(x, w_re, w_im, hop, center, pad_mode)
        d_re, d_im = torch.autograd.grad(y, (w_re, w_im), g.double())
    return d_re.float(), d_im.float()


def istft_forward(X, packed, window, n_fft, hop, center, length):
    from oracle import nnaudio_oracle as oracle

    kc, ks, onesided = packed
    y = oracle.istft(X.numpy(), kc.numpy(), ks.numpy(), window.numpy().reshape(1, -1, 1), hop,
                     center=center, onesided=onesided, length=length)
    return torch.from_numpy(np.ascontiguousarray(y)).float()


def fir_decimate(x, fir, factor):
    """conv1d(x, fir, stride=factor, padding=(taps-1)//2) (utils.py:73-100), computed in float64."""
    taps = fir.numel()
    return torch.nn.functional.conv1d(x[:, None, :].double(), fir.reshape(1, 1, -1).double(), stride=factor,
                                      padding=(taps - 1) // 2)[:, 0, :].float()


def fir_decimate_adjoint(g, fir, factor, L_in):
    x = torch.zeros((g.shape[0], L_in), dtype=torch.float64, requires_grad=True)
    with torch.enable_grad():
        taps = fir.numel()
        y = torch.nn.functional.conv1d(x[:, None, :], fir.reshape(1, 1, -1).double(), stride=factor,
                                       padding=(taps - 1) // 2)[:, 0, :]
        (dx,) = torch.autograd.grad(y, x, g.double())
    return dx.float()


def install(monkeypatch):
    """Route the calls of the differentiable host paths to the stand-ins above."""
    monkeypatch.setattr(_C, "_dev_f32", lambda t, name: t)
    monkeypatch.setattr(_C, "pack_basis", lambda w_re, w_im, layout=0: torch.zeros(1))
    monkeypatch.setattr(_C, "pack_basis_block", lambda w_re, hop: torch.zeros(1))
    monkeypatch.setattr(_C, "pack_adjoint_basis", lambda w_re, w_im: (w_re.clone(), w_im.clone()))
    monkeypatch.setattr(_C, "pack_istft_basis",
                        lambda kc, ks, f_in, onesided: (kc.clone(), ks.clone(), bool(onesided)))
    monkeypatch.setattr(_C, "cqt1992v2_forward", cqt1992v2_forward)
    monkeypatch.setattr(_C, "stft_forward", stft_forward)
    monkeypatch.setattr(_C, "stft_filterbank_forward", stft_filterbank_forward)
    monkeypatch.setattr(_C, "mfcc_forward", mfcc_forward)
    monkeypatch.setattr(_C, "cqt_pyramid_forward", cqt_pyramid_forward)
    monkeypatch.setattr(_C, "build_filterbank_table", lambda fb: None)
    monkeypatch.setattr(_C, "pack_fir", lambda fir, dec: torch.zeros(1))
    monkeypatch.setattr(_C, "framed_backward_input", framed_backward_input)
    monkeypatch.setattr(_C, "framed_backward_weight", framed_backward_weight)
    monkeypatch.setattr(_C, "istft_forward", istft_forward)
    monkeypatch.setattr(_C, "fir_decimate", fir_decimate, raising=False)
    monkeypatch.setattr(_C, "fir_decimate_adjoint", fir_decimate_adjoint, raising=False)
