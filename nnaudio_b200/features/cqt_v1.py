"""``CQT1992`` and ``CQT2010`` — drop-ins for the reference's first-generation, frequency-domain
constant-Q transforms (cqt.py:9-256, :259-558; SURVEY.md §8f next #3).

The reference runs two linear stages per frame: an un-windowed DFT of ``n_fft`` samples
(``conv1d`` with ``wcos`` / ``wsin``) and then a complex matmul with the FFT of the wavelet bank
(``complex_mul``, utils.py:175-203).  Both stages are linear and act on the same frame, so their
product is a single time-domain bank

    E_re = K_re @ W_cos - K_im @ W_sin          E_im = K_re @ W_sin + K_im @ W_cos

of shape ``(n_bins, n_fft)`` — ``n_fft/2+1`` times less work per frame than the two-stage form.
The module keeps the reference's buffers (``wsin``, ``wcos``, ``cqt_kernels_real/imag``,
``lenghts``, …, bit-identical) so ``state_dict`` round-trips, folds them into ``E`` in float64
whenever they change, and runs ``E`` through the same fused kernels as ``CQT1992v2`` /
``CQT2010v2``.  With ``trainable_STFT`` / ``trainable_CQT`` the fold is done under autograd so
the gradients reach the original parameters.
"""
from __future__ import annotations

from time import time

import numpy as np
import torch
import torch.nn as nn
from scipy.fftpack import fft as _fft

from .. import _C, design
from ._common import PackedBasis, PerDeviceCache, broadcast_dim, pad_mode_id, upcast_16bit, wants_grad
from .cqt import (_ScaleCache, _check_cqt_length, _check_format_and_norm, _framed_complex_autograd,
                  _pyramid_forward)


def _register(mod, name, value, trainable):
    if trainable:
        mod.register_parameter(name, nn.Parameter(value, requires_grad=True))
    else:
        mod.register_buffer(name, value)


def _fold(k_re, k_im, wcos, wsin, dtype):
    """(n_bins, F) spectral kernels x (F, 1, n_fft) DFT rows -> (E_re, E_im), each (n_bins, n_fft)."""
    wc = wcos.reshape(wcos.shape[0], -1).to(dtype)
    ws = wsin.reshape(wsin.shape[0], -1).to(dtype)
    kr, ki = k_re.to(dtype), k_im.to(dtype)
    return kr @ wc - ki @ ws, kr @ ws + ki @ wc


class _FoldedBank:
    """Cache of the folded time-domain bank (fp32, from a float64 fold) and its tensor-core
    packing, for both signs of the imaginary rows."""

    def __init__(self):
        self._cache = PerDeviceCache()

    def get(self, mod, negate_imag: bool):
        src = (mod.cqt_kernels_real, mod.cqt_kernels_imag, mod.wcos, mod.wsin)

        def build():
            with torch.no_grad():
                for t in src:
                    _C._dev_f32(t.detach(), "kernel")
                e_re, e_im = _fold(*[t.detach() for t in src], torch.float64)
                e_re, e_im, e_neg = (e_re.float().contiguous(), e_im.float().contiguous(),
                                     (-e_im).float().contiguous())
            return e_re, {False: e_im, True: e_neg}, {False: PackedBasis(), True: PackedBasis()}

        key = tuple((t.data_ptr(), t._version) for t in src)
        e_re, w_im, packed = self._cache.lookup(src[0].device, key, build)
        return e_re, w_im[negate_imag], packed[negate_imag].get(e_re, w_im[negate_imag])

    def differentiable(self, mod, negate_imag: bool):
        """Same fold under autograd (fp32), so dE reaches the trainable DFT rows / spectral kernels."""
        e_re, e_im = _fold(mod.cqt_kernels_real, mod.cqt_kernels_imag, mod.wcos, mod.wsin,
                           torch.float32)
        return e_re, (-e_im if negate_imag else e_im)


def _has_trainable(mod):
    return torch.is_grad_enabled() and any(p.requires_grad for p in mod.parameters())


class CQT1992(nn.Module):
    """Brown & Puckette (1992) CQT, frequency-domain formulation (cqt.py:9-256).
    ``forward(x, output_format=None, normalization_type='librosa')`` returns ``(B, n_bins, T)``
    (Magnitude) or ``(B, n_bins, T, 2)`` (Complex / Phase)."""

    def __init__(
        self,
        sr=22050,
        hop_length=512,
        fmin=220,
        fmax=None,
        n_bins=84,
        trainable_STFT=False,
        trainable_CQT=False,
        bins_per_octave=12,
        filter_scale=1,
        output_format="Magnitude",
        norm=1,
        window="hann",
        center=True,
        pad_mode="reflect",
    ):
        super().__init__()
        self.hop_length = hop_length
        self.center = center
        self.pad_mode = pad_mode
        self.norm = norm
        self.output_format = output_format

        Q = float(filter_scale) / (2 ** (1 / bins_per_octave) - 1)
        print("Creating CQT kernels ...", end="\r")
        start = time()
        bank, self.kernel_width, lengths, freqs = design.cqt_bank(
            Q, sr, fmin, n_bins, bins_per_octave, norm, window, fmax
        )
        self.register_buffer("lenghts", torch.tensor(lengths).float())
        self.frequencies = freqs
        spectral = _fft(bank)[:, : self.kernel_width // 2 + 1]  # single precision, like the reference
        print("CQT kernels created, time used = {:.4f} seconds".format(time() - start))

        print("Creating STFT kernels ...", end="\r")
        start = time()
        kernel_sin, kernel_cos, self.bins2freq, _, window_mask = design.fourier_basis(
            self.kernel_width, window="ones", freq_scale="no", verbose=False
        )
        _register(self, "wsin", torch.tensor(kernel_sin * window_mask), trainable_STFT)
        _register(self, "wcos", torch.tensor(kernel_cos * window_mask), trainable_STFT)
        _register(self, "cqt_kernels_real", torch.tensor(spectral.real), trainable_CQT)
        _register(self, "cqt_kernels_imag", torch.tensor(spectral.imag), trainable_CQT)
        print("STFT kernels created, time used = {:.4f} seconds".format(time() - start))
        self._folded = _FoldedBank()
        self._scale = _ScaleCache()

    def forward(self, x, output_format=None, normalization_type="librosa"):
        output_format = output_format or self.output_format
        _check_format_and_norm(output_format, normalization_type)
        x = broadcast_dim(x)
        self._check_length(x.shape[0], x.shape[-1])
        mode, scale, scale_all, negate = self._plan(output_format, normalization_type)
        if wants_grad(self, x):
            if _has_trainable(self):
                w_re, w_im = self._folded.differentiable(self, negate)
            else:
                w_re, w_im, _ = self._folded.get(self, negate)
            c = _framed_complex_autograd(self, f"folded{int(negate)}", upcast_16bit(x), w_re, w_im,
                                         self.hop_length, self.center, mode)
            if scale is not None:
                c = c * scale.view(1, -1, 1, 1)
            elif scale_all != 1.0:
                c = c * scale_all
            if output_format == "Complex":
                return c
            if output_format == "Magnitude":
                return torch.sqrt(c[..., 0].pow(2) + c[..., 1].pow(2))
            ang = torch.atan2(c[..., 1], c[..., 0])
            return torch.stack((torch.cos(ang), torch.sin(ang)), -1)
        return _C.cqt1992v2_forward(x, **self._infer_args(output_format, normalization_type)[1])

    def _check_length(self, B, n):
        """Raise what the reference raises for ``B`` clips of ``n`` samples (also the end of a stream)."""
        _check_cqt_length(self, B, n)

    def _plan(self, output_format, normalization_type):
        width = self.kernel_width
        mode = pad_mode_id(self.pad_mode) if self.center else _C.PAD_CONSTANT
        scale, scale_all = None, 1.0
        if normalization_type == "librosa":  # sqrt(lenghts) / kernel_width, cqt.py:224-225
            scale = self._scale.get(self.lenghts, 1.0 / width)
        elif normalization_type == "wrap":
            scale_all = 2.0 / width
        # 'Phase' takes atan2 of the *un-negated* imaginary part (cqt.py:246-249), the other
        # formats stack (real, -imag) (cqt.py:222): choose the sign of the imaginary rows to match
        negate = output_format == "Phase"
        return mode, scale, scale_all, negate

    def _infer_args(self, output_format, normalization_type):
        """(name, keyword arguments after ``x``) of the ``_C`` call of the inference path."""
        mode, scale, scale_all, negate = self._plan(output_format, normalization_type)
        w_re, w_im, packed = self._folded.get(self, negate)
        fmt = {"Magnitude": _C.FMT_MAGNITUDE, "Complex": _C.FMT_COMPLEX,
               "Phase": _C.FMT_PHASE_UNIT}[output_format]
        return "cqt1992v2_forward", dict(
            k_real=w_re, k_imag=w_im, packed=packed, k_begin=None, k_end=None, hop=self.hop_length,
            center=self.center, pad_mode=mode, scale=scale, scale_all=scale_all, out_format=fmt, sqrt_eps=0.0,
        )

    def extra_repr(self) -> str:
        return "STFT kernel size = {}, CQT kernel size = {}".format(
            (*self.wcos.shape,), (*self.cqt_kernels_real.shape,)
        )


class CQT2010(nn.Module):
    """Schörkhuber & Klapuri (2010) CQT with the frequency-domain top-octave kernel
    (cqt.py:259-558): the ÷2 pyramid of ``CQT2010v2`` with the folded bank in every octave.
    Unlike v2, the result is *not* multiplied by the early-downsample factor, the imaginary part
    is not negated (utils.py:551-559), and 'librosa' / 'wrap' divide by ``n_fft``."""

    def __init__(
        self,
        sr=22050,
        hop_length=512,
        fmin=32.70,
        fmax=None,
        n_bins=84,
        bins_per_octave=12,
        norm=True,
        basis_norm=1,
        window="hann",
        pad_mode="reflect",
        trainable_STFT=False,
        filter_scale=1,
        trainable_CQT=False,
        output_format="Magnitude",
        earlydownsample=True,
        verbose=True,
    ):
        super().__init__()
        self.norm = norm
        self.hop_length = hop_length
        self.pad_mode = pad_mode
        self.n_bins = n_bins
        self.output_format = output_format
        self.earlydownsample = earlydownsample
        self.trainable = False  # no sqrt-eps variant in the v1 module (cqt.py:543-545)

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
        self.register_buffer("lenghts", torch.tensor(np.ceil(Q * sr / freqs)).float())
        self.basis = basis
        spectral = _fft(basis)[:, : self.n_fft // 2 + 1]
        if verbose:
            print("CQT kernels created, time used = {:.4f} seconds".format(time() - start))
            print("Creating STFT kernels ...", end="\r")
        start = time()
        kernel_sin, kernel_cos, self.bins2freq, _, window_mask = design.fourier_basis(
            self.n_fft, window="ones", freq_scale="no", verbose=False
        )
        if verbose:
            print("STFT kernels created, time used = {:.4f} seconds".format(time() - start))
        _register(self, "wsin", torch.tensor(kernel_sin * window_mask), trainable_STFT)
        _register(self, "wcos", torch.tensor(kernel_cos * window_mask), trainable_STFT)
        _register(self, "cqt_kernels_real", torch.tensor(spectral.real), trainable_CQT)
        _register(self, "cqt_kernels_imag", torch.tensor(spectral.imag), trainable_CQT)

        if self.pad_mode == "constant":  # attribute parity (cqt.py:470-473); kernels pad in-flight
            self.padding = nn.ConstantPad1d(self.n_fft // 2, 0)
        elif self.pad_mode == "reflect":
            self.padding = nn.ReflectionPad1d(self.n_fft // 2)
        self._folded = _FoldedBank()
        self._scale = _ScaleCache()

    def _banks(self):
        w_re, w_im, packed = self._folded.get(self, True)
        return [w_re] * self.n_octaves, [w_im] * self.n_octaves, [packed] * self.n_octaves

    def _bank_tensors(self):
        if _has_trainable(self):
            pair = self._folded.differentiable(self, True)
        else:
            pair = self._folded.get(self, True)[:2]
        return [pair] * self.n_octaves

    def forward(self, x, output_format=None, normalization_type="librosa"):
        output_format = output_format or self.output_format
        _check_format_and_norm(output_format, normalization_type)
        x = broadcast_dim(x)
        return _pyramid_forward(self, x, output_format, self._normalization(normalization_type))

    def _normalization(self, normalization_type):
        """(per-bin scale or None, global factor, sqrt eps) of the pyramid call (cqt.py:531-532)."""
        scale, scale_all = None, 1.0
        if normalization_type == "librosa":
            scale = self._scale.get(self.lenghts, 1.0 / self.n_fft)
        elif normalization_type == "wrap":
            scale_all = 2.0 / self.n_fft
        return scale, scale_all, 0.0

    def extra_repr(self) -> str:
        return "STFT kernel size = {}, CQT kernel size = {}".format(
            (*self.wcos.shape,), (*self.cqt_kernels_real.shape,)
        )
