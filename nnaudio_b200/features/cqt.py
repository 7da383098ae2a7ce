"""``CQT1992v2``, ``CQT2010v2`` and the ``CQT`` alias — drop-ins for
``nnAudio.features.cqt`` (cqt.py:561-803, :805-1139, :1142-1145).

Buffer names follow the reference, including its spelling ``lenghts``.
"""
from __future__ import annotations

import warnings
from time import time

import numpy as np
import torch
import torch.nn as nn

from .. import _C, design
from ._common import (AdjointBasis, FramedComplexFn, PackedBasis, PackedFir, PerDeviceCache, as_matrix,
                      broadcast_dim, pad_mode_id, tap_support, upcast_16bit, wants_grad)

_FORMATS = {
    "Magnitude": _C.FMT_MAGNITUDE,
    "Complex": _C.FMT_COMPLEX,
    "Phase": _C.FMT_PHASE_UNIT,
}
_NORMALIZATIONS = ("librosa", "convolutional", "wrap")


def _check_format_and_norm(output_format, normalization_type):
    if normalization_type not in _NORMALIZATIONS:
        raise ValueError(
            "The normalization_type %r is not part of our current options." % normalization_type
        )
    if output_format not in _FORMATS:
        raise ValueError(
            f"output_format must be 'Magnitude', 'Complex' or 'Phase', got {output_format!r}"
        )


def _check_cqt_length(mod, B, n):
    """The reference's exceptions for ``B`` clips of ``n`` samples through a framed CQT (cqt.py:740-750)."""
    pad = mod.kernel_width // 2 if mod.center else 0
    if mod.center and mod.pad_mode == "reflect" and n <= pad:
        raise RuntimeError(
            "Padding size should be less than the corresponding input dimension, but got: "
            f"padding ({pad}, {pad}) at dimension 2 of input {(B, 1, n)}"
        )
    if n + 2 * pad < mod.kernel_width:
        raise RuntimeError("Kernel size can't be greater than actual input size")


class _ScaleCache:
    """sqrt(lenghts) * factor on the device, recomputed when ``lenghts`` changes."""

    def __init__(self):
        self._cache = PerDeviceCache()

    def get(self, lenghts: torch.Tensor, factor: float):
        def build():
            s = torch.sqrt(lenghts.detach().float())
            return (s * factor if factor != 1 else s).contiguous()

        key = (lenghts.data_ptr(), lenghts._version, float(factor))
        return self._cache.lookup(lenghts.device, key, build)


class CQT1992v2(nn.Module):
    """Time-domain constant-Q transform with one wavelet bank spanning all bins
    (cqt.py:655-780).  ``forward(x, output_format=None,
    normalization_type='librosa')`` returns ``(B, n_bins, T)`` (Magnitude) or
    ``(B, n_bins, T, 2)`` (Complex = (real, imag); Phase = (cos, sin))."""

    def __init__(
        self,
        sr=22050,
        hop_length=512,
        fmin=32.70,
        fmax=None,
        n_bins=84,
        bins_per_octave=12,
        filter_scale=1,
        norm=1,
        window="hann",
        center=True,
        pad_mode="reflect",
        trainable=False,
        output_format="Magnitude",
        verbose=True,
    ):
        super().__init__()
        self.trainable = trainable
        self.hop_length = hop_length
        self.center = center
        self.pad_mode = pad_mode
        self.output_format = output_format

        Q = float(filter_scale) / (2 ** (1 / bins_per_octave) - 1)
        if verbose:
            print("Creating CQT kernels ...", end="\r")
        start = time()
        bank, self.kernel_width, lengths, freqs = design.cqt_bank(
            Q, sr, fmin, n_bins, bins_per_octave, norm, window, fmax
        )
        self.register_buffer("lenghts", torch.tensor(lengths).float())
        self.frequencies = freqs

        k_real = torch.tensor(bank.real).unsqueeze(1)
        k_imag = torch.tensor(bank.imag).unsqueeze(1)
        if trainable:
            self.register_parameter("cqt_kernels_real", nn.Parameter(k_real, requires_grad=True))
            self.register_parameter("cqt_kernels_imag", nn.Parameter(k_imag, requires_grad=True))
        else:
            self.register_buffer("cqt_kernels_real", k_real)
            self.register_buffer("cqt_kernels_imag", k_imag)

        self._packed = PackedBasis()
        self._scale = _ScaleCache()
        self._support = PerDeviceCache()
        if verbose:
            print("CQT kernels created, time used = {:.4f} seconds".format(time() - start))

    def _tap_support(self):
        """Host int32 [begin, end) of each wavelet's non-zero taps, from the
        *current* buffer contents (dense when the bank is trainable)."""
        if self.trainable:
            return None, None
        kr, ki = self.cqt_kernels_real, self.cqt_kernels_imag

        def build():
            both = (kr.detach()[:, 0, :] != 0) | (ki.detach()[:, 0, :] != 0)
            return tap_support(both.cpu().numpy())

        key = (kr.data_ptr(), kr._version, ki.data_ptr(), ki._version)
        return self._support.lookup(kr.device, key, build)

    def _check_length(self, B, n):
        """Raise what the reference raises for ``B`` clips of ``n`` samples (also the end of a stream)."""
        _check_cqt_length(self, B, n)

    def _infer_args(self, output_format, normalization_type):
        """(name, keyword arguments after ``x``) of the ``_C`` call of the inference path."""
        k_real, k_imag = as_matrix(self.cqt_kernels_real), as_matrix(self.cqt_kernels_imag)
        packed = self._packed.get(k_real, k_imag,
                                  groups=(not self.trainable) and self.hop_length % 8 == 0)
        k_begin, k_end = self._tap_support()
        scale, scale_all = None, 1.0
        if normalization_type == "librosa":
            scale = self._scale.get(self.lenghts, 1.0)
        elif normalization_type == "wrap":
            scale_all = 2.0
        eps = 1e-8 if (self.trainable and output_format == "Magnitude") else 0.0
        return "cqt1992v2_forward", dict(
            k_real=k_real, k_imag=k_imag, packed=packed, k_begin=k_begin, k_end=k_end, hop=self.hop_length,
            center=self.center, pad_mode=pad_mode_id(self.pad_mode), scale=scale, scale_all=scale_all,
            out_format=_FORMATS[output_format], sqrt_eps=eps,
        )

    def forward(self, x, output_format=None, normalization_type="librosa"):
        output_format = output_format or self.output_format
        _check_format_and_norm(output_format, normalization_type)
        x = broadcast_dim(x)
        self._check_length(x.shape[0], x.shape[-1])

        args = self._infer_args(output_format, normalization_type)[1]
        k_real, k_imag, packed = args["k_real"], args["k_imag"], args["packed"]
        k_begin, k_end = args["k_begin"], args["k_end"]
        scale, scale_all, eps = args["scale"], args["scale_all"], args["sqrt_eps"]
        if wants_grad(self, x):
            # un-normalised complex CQT through the fused kernel + dX / dW kernels; normalisation and
            # output format (cqt.py:752-780) composed in torch for autograd
            if not hasattr(self, "_adjoint"):
                self._adjoint = AdjointBasis()

            def fwd(t):
                return _C.cqt1992v2_forward(t, k_real, k_imag, packed, k_begin, k_end,
                                            self.hop_length, self.center,
                                            pad_mode_id(self.pad_mode), None, 1.0,
                                            _C.FMT_COMPLEX, 0.0)

            def bwd(g, L):
                return _C.framed_backward_input(g, self._adjoint.get(k_real, k_imag),
                                                self.kernel_width, self.hop_length, self.center,
                                                pad_mode_id(self.pad_mode), L)

            def bwd_w(g, xin):
                return _C.framed_backward_weight(g, xin, self.kernel_width, self.hop_length,
                                                 self.center, pad_mode_id(self.pad_mode))

            c = FramedComplexFn.apply(upcast_16bit(x), self.cqt_kernels_real, self.cqt_kernels_imag, fwd,
                                      bwd, bwd_w)
            if scale is not None:
                c = c * scale.view(1, -1, 1, 1)
            elif scale_all != 1.0:
                c = c * scale_all
            if output_format == "Complex":
                return c
            if output_format == "Magnitude":
                return torch.sqrt(c[..., 0].pow(2) + c[..., 1].pow(2) + eps)
            ang = torch.atan2(c[..., 1], c[..., 0])
            return torch.stack((torch.cos(ang), torch.sin(ang)), -1)
        return _C.cqt1992v2_forward(x, **args)


class CQT(CQT1992v2):
    """Alias of :class:`CQT1992v2` (cqt.py:1142-1145)."""

    pass


def _decimated_len(n, factor):
    """Samples conv1d(stride=factor, padding=127) leaves of ``n`` under the 256-tap FIR (utils.py:73-100)."""
    return (n - 2) // factor + 1 if n >= 2 else 0


def _octave_levels(L, hop, n_octaves):
    """(signal lengths, hops) of the octaves of the ÷2 pyramid on a level-0 signal of ``L`` samples."""
    lens, hops = [], []
    cur, h = L, hop
    for i in range(n_octaves):
        if i > 0:
            cur = _decimated_len(cur, 2)
            h = h // 2
        lens.append(cur)
        hops.append(h)
    return lens, hops


def _octave_plan(L, hop, widths, pad_mode):
    """Per-octave signal lengths of the ÷2 pyramid and whether the reference's
    reflect padding would fall back to zero padding (utils.py:505-517).
    Returns (T, fallback_flags) or raises like torch.cat would."""
    lens, hops = _octave_levels(L, hop, len(widths))
    flags = [pad_mode == "reflect" and w // 2 >= cur for w, cur in zip(widths, lens)]
    if min(hops) <= 0 or min(lens) <= 0:
        raise RuntimeError(
            "CQT pyramid: hop_length or signal too small for the number of octaves "
            f"(lengths {lens}, hops {hops})"
        )
    Ts = [l // h + 1 for l, h in zip(lens, hops)]
    if len(set(Ts)) != 1:
        raise RuntimeError(
            f"Sizes of tensors must match except in dimension 1 (octave frame counts {Ts})"
        )
    return Ts[0], flags


class CQT2010v2(nn.Module):
    """Constant-Q transform by the resampling method: one top-octave bank reused
    over a ÷2 anti-aliased pyramid (cqt.py:901-1139).  Like the reference, the
    ``window`` and ``norm`` constructor arguments do not influence the bank
    (cqt.py:1023-1031 never forwards them)."""

    def __init__(
        self,
        sr=22050,
        hop_length=512,
        fmin=32.70,
        fmax=None,
        n_bins=84,
        filter_scale=1,
        bins_per_octave=12,
        norm=True,
        basis_norm=1,
        window="hann",
        pad_mode="reflect",
        earlydownsample=True,
        trainable=False,
        output_format="Magnitude",
        verbose=True,
    ):
        super().__init__()
        self.norm = norm
        self.hop_length = hop_length
        self.pad_mode = pad_mode
        self.n_bins = n_bins
        self.earlydownsample = earlydownsample
        self.trainable = trainable
        self.output_format = output_format

        Q = float(filter_scale) / (2 ** (1 / bins_per_octave) - 1)

        if verbose:
            print("Creating low pass filter ...", end="\r")
        start = time()
        lowpass = torch.tensor(design.lowpass_fir(0.50, 256, 0.001))
        self.register_buffer("lowpass_filter", lowpass[None, None, :])
        if verbose:
            print("Low pass filter created, time used = {:.4f} seconds".format(time() - start))

        n_filters = min(bins_per_octave, n_bins)
        self.n_octaves = int(np.ceil(float(n_bins) / bins_per_octave))
        if verbose:
            print("num_octave = ", self.n_octaves)

        # lowest bin of the top-octave bank (cqt.py:970-983)
        self.fmin_t = fmin * 2 ** (self.n_octaves - 1)
        remainder = n_bins % bins_per_octave
        if remainder == 0:
            fmax_t = self.fmin_t * 2 ** ((bins_per_octave - 1) / bins_per_octave)
        else:
            fmax_t = self.fmin_t * 2 ** ((remainder - 1) / bins_per_octave)
        self.fmin_t = fmax_t / 2 ** (1 - 1 / bins_per_octave)
        if fmax_t > sr / 2:
            raise ValueError(
                "The top bin {}Hz has exceeded the Nyquist frequency, \
                            please reduce the n_bins".format(
                    fmax_t
                )
            )

        if self.earlydownsample:
            if verbose:
                print("Creating early downsampling filter ...", end="\r")
            start = time()
            sr, self.hop_length, self.downsample_factor, early_fir = design.early_downsample_plan(
                sr, hop_length, fmax_t, Q, self.n_octaves
            )
            self.earlydownsample = early_fir is not None
            if verbose:
                if self.earlydownsample:
                    print("Can do early downsample, factor = ", self.downsample_factor)
                else:
                    print("No early downsampling is required, downsample_factor = ",
                          self.downsample_factor)
            self.register_buffer(
                "early_downsample_filter",
                torch.tensor(early_fir)[None, None, :] if early_fir is not None else None,
            )
            if verbose:
                print("Early downsampling filter created, \
                        time used = {:.4f} seconds".format(time() - start))
        else:
            self.downsample_factor = 1.0

        if verbose:
            print("Creating CQT kernels ...", end="\r")
        start = time()
        basis, self.n_fft, _, _ = design.cqt_bank(
            Q, sr, self.fmin_t, n_filters, bins_per_octave, norm=basis_norm, topbin_check=False
        )
        freqs = fmin * 2.0 ** (np.r_[0:n_bins] / np.double(bins_per_octave))
        self.frequencies = freqs
        lenghts = np.ceil(Q * sr / freqs)
        self.register_buffer("lenghts", torch.tensor(lenghts).float())

        self.basis = basis
        k_real = torch.tensor(basis.real).unsqueeze(1)
        k_imag = torch.tensor(basis.imag).unsqueeze(1)
        if trainable:
            self.register_parameter("cqt_kernels_real", nn.Parameter(k_real, requires_grad=True))
            self.register_parameter("cqt_kernels_imag", nn.Parameter(k_imag, requires_grad=True))
        else:
            self.register_buffer("cqt_kernels_real", k_real)
            self.register_buffer("cqt_kernels_imag", k_imag)
        if verbose:
            print("CQT kernels created, time used = {:.4f} seconds".format(time() - start))

        # kept for attribute parity (cqt.py:1065-1068); the kernels pad in-flight
        if self.pad_mode == "constant":
            self.padding = nn.ConstantPad1d(self.n_fft // 2, 0)
        elif self.pad_mode == "reflect":
            self.padding = nn.ReflectionPad1d(self.n_fft // 2)
        self._scale = _ScaleCache()
        self._packed = PackedBasis()

    def _banks(self):
        k_real, k_imag = as_matrix(self.cqt_kernels_real), as_matrix(self.cqt_kernels_imag)
        packed = self._packed.get(k_real, k_imag)  # one bank shared by every octave
        return [k_real] * self.n_octaves, [k_imag] * self.n_octaves, [packed] * self.n_octaves

    def _bank_tensors(self):
        """Per-octave (real, imag) bank tensors as autograd sees them (one shared, possibly
        trainable, bank: its gradient is the sum over the octaves)."""
        return [(self.cqt_kernels_real, self.cqt_kernels_imag)] * self.n_octaves

    def forward(self, x, output_format=None, normalization_type="librosa"):
        output_format = output_format or self.output_format
        _check_format_and_norm(output_format, normalization_type)
        x = broadcast_dim(x)
        return _pyramid_forward(self, x, output_format,
                                _v2_normalization(self, normalization_type, output_format))


def _v2_normalization(mod, normalization_type, output_format):
    """cqt.py:1112-1124 / vqt.py:190-200: (per-bin scale tensor or None, global factor, sqrt eps)."""
    scale, scale_all = None, 1.0
    dsf = float(mod.downsample_factor)
    if normalization_type == "librosa":
        scale = mod._scale.get(mod.lenghts, dsf)
    elif normalization_type == "wrap":
        scale_all = 2.0 * dsf
    else:
        scale_all = dsf
    eps = 1e-8 if (mod.trainable and output_format == "Magnitude") else 0.0
    return scale, scale_all, eps


def _pyramid_length_plan(mod, B, L):
    """(T, per-octave reflect fallbacks) of ``B`` clips of ``L`` samples through ``mod``'s pyramid, with the
    reference's errors and warnings (also the end of a stream)."""
    factor = int(mod.downsample_factor) if mod.earlydownsample else 1
    L0 = _decimated_len(L, factor) if factor > 1 else L
    if factor > 1 and L < 2:
        raise RuntimeError("Kernel size can't be greater than actual input size")
    widths = [int(b.shape[1]) for b in mod._banks()[0]]
    T, fallbacks = _octave_plan(L0, mod.hop_length, widths, mod.pad_mode)
    for i, fb in enumerate(fallbacks):
        if fb:
            warnings.warn(
                f"\ninput size = {(B, 1, L0)}\tkernel size = {widths[i]}\n"
                "padding with reflection mode might not be the best choice, try using constant padding",
                UserWarning,
            )
    return T, fallbacks


def _pyramid_args(mod, output_format, normalization):
    """Keyword arguments after ``x`` (``T`` aside) of the ``_C.cqt_pyramid_forward`` call of the inference
    path; shared with ``nnaudio_b200.streaming.StreamingPyramid``."""
    scale, scale_all, eps = normalization
    banks_real, banks_imag, packed = mod._banks()
    early = mod.early_downsample_filter if mod.earlydownsample else None
    factor = int(mod.downsample_factor) if mod.earlydownsample else 1
    lowpass = mod.lowpass_filter.detach().reshape(-1)
    early_flat = early.detach().reshape(-1) if early is not None else None
    for t in (lowpass, early_flat):
        if t is not None:
            _C._dev_f32(t, "filter")
    if not hasattr(mod, "_fir_packed"):
        mod._fir_packed = (PackedFir(), PackedFir())
    lowpass_packed = mod._fir_packed[0].get(lowpass, 2)
    early_packed = mod._fir_packed[1].get(early_flat, factor) if early_flat is not None else None
    return dict(banks_real=banks_real, banks_imag=banks_imag, packed=packed, lowpass=lowpass,
                lowpass_packed=lowpass_packed, early_filter=early_flat, early_packed=early_packed,
                early_factor=factor, hop=mod.hop_length, pad_mode=pad_mode_id(mod.pad_mode), n_bins=mod.n_bins,
                scale=scale, scale_all=scale_all, out_format=_FORMATS[output_format], sqrt_eps=eps)


def _pyramid_forward(mod, x, output_format, normalization):
    """Shared by CQT2010v2, VQT and CQT2010: plan the octave lengths on the host (for the
    reference's warnings / errors), then one C call.  ``normalization`` = (scale, scale_all, eps)."""
    scale, scale_all, eps = normalization
    T, fallbacks = _pyramid_length_plan(mod, x.shape[0], x.shape[-1])
    if wants_grad(mod, x):
        factor = int(mod.downsample_factor) if mod.earlydownsample else 1
        return _pyramid_forward_autograd(mod, upcast_16bit(x), output_format, fallbacks, factor, scale,
                                         scale_all, eps)
    return _C.cqt_pyramid_forward(x, T=T, **_pyramid_args(mod, output_format, normalization))


def _framed_complex_autograd(mod, tag, sig, w_re, w_im, hop, center, pad_mode):
    """One differentiable framed contraction ``sig (B, L) -> (B, F, T, 2)`` through the fused
    forward kernel and the dX / dW kernels; ``tag`` keys the packed-basis caches on ``mod``."""
    k_re, k_im = as_matrix(w_re), as_matrix(w_im)
    if w_re.grad_fn is not None or w_im.grad_fn is not None:
        # recomputed temporaries (the folded v1 bank under autograd): every call gets a fresh
        # tensor with _version 0 whose address the allocator may recycle from the previous step,
        # so a (data_ptr, _version) key cannot tell them apart -> pack per call, never cache.
        # The packing rides on the temporary itself (shared by the octaves of one forward, freed
        # with it).
        caches = w_re.__dict__.setdefault("_nnab_grad_caches", {})
        caches.setdefault(tag, (PackedBasis(), AdjointBasis()))
    else:
        caches = mod.__dict__.setdefault("_grad_caches", {})
        if tag not in caches:
            caches[tag] = (PackedBasis(), AdjointBasis())
    packed = caches[tag][0].get(k_re, k_im)
    width = int(k_re.shape[1])

    def fwd(t):
        return _C.cqt1992v2_forward(t, k_re, k_im, packed, None, None, hop, center, pad_mode,
                                    None, 1.0, _C.FMT_COMPLEX, 0.0)

    def bwd(g, L):
        return _C.framed_backward_input(g, caches[tag][1].get(k_re, k_im), width, hop, center,
                                        pad_mode, L)

    def bwd_w(g, xin):
        return _C.framed_backward_weight(g, xin, width, hop, center, pad_mode)

    return FramedComplexFn.apply(sig, w_re, w_im, fwd, bwd, bwd_w)


class _FirDecimateFn(torch.autograd.Function):
    """``nnab_fir_decimate`` / ``nnab_fir_decimate_adjoint``: one launch each way (GPU-verified round 2)."""

    @staticmethod
    def forward(ctx, sig, fir, n):
        ctx.fir, ctx.n, ctx.L = fir, n, sig.shape[-1]
        return _C.fir_decimate(sig, fir, n)

    @staticmethod
    def backward(ctx, g):
        return _C.fir_decimate_adjoint(g.contiguous(), ctx.fir, ctx.n, ctx.L), None, None


def _decimate_autograd(mod, tag, sig, fir, n):
    """Differentiable ``downsampling_by_n`` / ``_by_2`` stage ``tag`` of ``mod``'s training path: the
    dedicated CUDA-core FIR stage and its adjoint kernel (``nnab_fir_decimate`` /
    ``nnab_fir_decimate_adjoint``: every input sample written once, no atomics), within the 1e-4 bar on
    every pyramid gradient case.  The stage keeps no per-module state, so ``mod`` and ``tag`` only name it."""
    return _FirDecimateFn.apply(sig, fir.detach().reshape(-1).contiguous(), int(n))


def _pyramid_forward_autograd(mod, x, output_format, fallbacks, factor, scale, scale_all, eps):
    """cqt.py:1085-1139 / vqt.py:160-215 octave by octave with autograd-visible stages
    (training path; inference uses the single fused C call above)."""
    if factor > 1:
        x = _decimate_autograd(mod, "early", x, mod.early_downsample_filter, factor)
    hop = mod.hop_length
    octaves = []
    cur = x
    for i, (w_re, w_im) in enumerate(mod._bank_tensors()):
        if i > 0:
            hop //= 2
            cur = _decimate_autograd(mod, "lowpass", cur, mod.lowpass_filter, 2)
        mode = _C.PAD_CONSTANT if fallbacks[i] else pad_mode_id(mod.pad_mode)
        octaves.insert(0, _framed_complex_autograd(mod, f"bank{i}", cur, w_re, w_im, hop, True,
                                                   mode))
    c = torch.cat(octaves, 1)[:, -mod.n_bins:]
    if scale is not None:  # sqrt(lenghts) * downsample_factor
        c = c * scale.view(1, -1, 1, 1)
    elif scale_all != 1.0:
        c = c * scale_all
    if output_format == "Complex":
        return c
    if output_format == "Magnitude":
        return torch.sqrt(c[..., 0].pow(2) + c[..., 1].pow(2) + eps)
    ang = torch.atan2(c[..., 1], c[..., 0])
    return torch.stack((torch.cos(ang), torch.sin(ang)), -1)
