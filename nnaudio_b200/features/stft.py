"""``STFT`` — drop-in for ``nnAudio.features.stft.STFT`` (stft.py:68-361).

Same constructor / forward signature, attribute and buffer names
(``wsin``, ``wcos`` ``(F,1,n_fft)``, ``window_mask`` ``(1,n_fft,1)``,
optional ``kernel_sin_inv`` / ``kernel_cos_inv``), but ``forward`` is one call
into ``libnnab.so`` instead of ReflectionPad1d + 2x conv1d + element-wise ops.
"""
from __future__ import annotations

from time import time

import torch
import torch.nn as nn

from .. import _C, design
from ._common import (AdjointBasis, FramedComplexFn, PackedBasis, PerDeviceCache, as_matrix,
                      broadcast_dim,
                      forward_only_guard, pad_mode_id, upcast_16bit, wants_grad)

_FORMATS = {
    "Magnitude": _C.FMT_MAGNITUDE,
    "Complex": _C.FMT_COMPLEX,
    "Phase": _C.FMT_PHASE_ANGLE,
}


class _InverseBasis:
    """Cache of the tensor-core packing of the (n_fft, n_fft) inverse kernels per
    (one-sided?, bins) variant."""

    def __init__(self):
        self._cache = PerDeviceCache()

    def get(self, kc: torch.Tensor, ks: torch.Tensor, f_in: int, onesided: bool):
        key = (kc.data_ptr(), kc._version, ks.data_ptr(), ks._version, f_in, bool(onesided))
        return self._cache.lookup(kc.device, key, lambda: _C.pack_istft_basis(kc, ks, f_in, onesided))


class _InverseAdjoint:
    """Cache of the forward-shaped basis that carries the iSTFT input gradient:
    ``w[f, o] = kernel[o, f] * window[o] / n_fft`` with the Hermitian mirror rows of a one-sided
    spectrum (utils.py:63-70) folded in, plus its tensor-core packing."""

    def __init__(self):
        self._cache = PerDeviceCache()

    def get(self, kc, ks, win, onesided):
        def build():
            n_fft = kc.shape[0]
            w_re = (kc * (win / n_fft)[:, None]).t().contiguous()   # (f, o)
            w_im = (ks * (win / n_fft)[:, None]).t().contiguous()
            if onesided:
                half = n_fft // 2
                lo_re, lo_im = w_re[:half + 1].clone(), w_im[:half + 1].clone()
                mirror = torch.arange(n_fft - 1, half, -1, device=kc.device)  # rows n_fft-f, f=1..half-1
                lo_re[1:half] += w_re[mirror]
                lo_im[1:half] -= w_im[mirror]
                w_re, w_im = lo_re.contiguous(), lo_im.contiguous()
            return w_re, w_im, _C.pack_basis(w_re, w_im)

        key = (kc.data_ptr(), kc._version, ks.data_ptr(), ks._version, win.data_ptr(), win._version,
               bool(onesided))
        return self._cache.lookup(kc.device, key, build)


class _InverseSTFTFn(torch.autograd.Function):
    """iSTFT with a gradient for the spectrogram input (the reference gets it from autograd
    through conv2d + fold, stft.py:15-63)."""

    @staticmethod
    def forward(ctx, X, run, grad_spec):
        ctx.grad_spec = grad_spec
        ctx.T = X.shape[2]
        with torch.no_grad():
            return run(X)

    @staticmethod
    def backward(ctx, gy):
        return ctx.grad_spec(gy.contiguous().float(), ctx.T), None, None


def _inverse_args(mod, f_in, kernel_cos, kernel_sin, window_mask, onesided):
    """(kc, ks, packed, win) of an inverse STFT of ``f_in``-bin spectra, with the reference's exceptions;
    shared by the offline inverse and ``nnaudio_b200.streaming.StreamingInverse``."""
    n_fft = mod.n_fft
    kc = kernel_cos.detach().reshape(kernel_cos.shape[0], -1)
    ks = kernel_sin.detach().reshape(kernel_sin.shape[0], -1)
    _C._dev_f32(kc, "kernel_cos")
    if kc.shape != (n_fft, n_fft) or ks.shape != (n_fft, n_fft):
        raise RuntimeError("inverse kernels must be (n_fft, n_fft)")
    expect = n_fft // 2 + 1 if onesided else n_fft
    if f_in != expect:
        raise RuntimeError(
            f"expected {expect} frequency bins for onesided={onesided} and n_fft={n_fft}, got {f_in}"
        )
    win = window_mask.detach().reshape(-1).float()  # iSTFT keeps scipy's float64 window
    if win.numel() != n_fft:
        raise RuntimeError(
            f"The size of tensor a ({n_fft}) must match the size of tensor b ({win.numel()}) "
            "at non-singleton dimension 1"
        )
    if not hasattr(mod, "_inv_basis"):
        mod._inv_basis = _InverseBasis()
    packed = mod._inv_basis.get(kc.contiguous(), ks.contiguous(), f_in, onesided)
    return kc, ks, packed, win.contiguous()


def _inverse_stft(mod, X, kernel_cos, kernel_sin, window_mask, onesided, length):
    """Shared by ``STFT.inverse`` and ``iSTFT.forward`` (STFTBase.inverse_stft, stft.py:15-63)."""
    n_fft = mod.n_fft
    kc, ks, packed, win = _inverse_args(mod, X.shape[1], kernel_cos, kernel_sin, window_mask, onesided)

    def run(spec):
        return _C.istft_forward(spec, packed, win, n_fft, mod.stride, mod.center, length)

    if not (torch.is_grad_enabled() and X.requires_grad):
        return run(X)
    if not hasattr(mod, "_inv_adjoint"):
        mod._inv_adjoint = _InverseAdjoint()
    w_re, w_im, w_packed = mod._inv_adjoint.get(kc, ks, win, onesided)
    hop, offset = mod.stride, (n_fft // 2 if mod.center else 0)

    def grad_spec(gy, T):
        """Adjoint of the inverse: undo the window-sum-square division, put the waveform gradient
        back at its place in the overlap-add buffer, then one forward framed contraction with the
        transposed, windowed inverse kernels (one-sided mirroring folded into the rows)."""
        ola_len = n_fft + hop * (T - 1)
        wss = torch.nn.functional.fold((win * win)[None, :, None].expand(1, n_fft, T).contiguous(),
                                       (1, ola_len), (1, n_fft), stride=(1, hop)).reshape(-1)
        inv = torch.where(wss > 1e-10, 1.0 / wss, torch.ones_like(wss))
        G = torch.zeros((gy.shape[0], ola_len), dtype=torch.float32, device=gy.device)
        G[:, offset:offset + gy.shape[1]] = gy
        G *= inv
        return _C.cqt1992v2_forward(G, w_re, w_im, w_packed, None, None, hop, False,
                                    _C.PAD_CONSTANT, None, 1.0, _C.FMT_COMPLEX, 0.0)

    return _InverseSTFTFn.apply(X, run, grad_spec)


class STFT(nn.Module):
    """Short-time Fourier transform of ``(L)``, ``(B, L)`` or ``(B, 1, L)``
    waveforms.  Arguments follow the reference (stft.py:153-170).

    Returns ``(B, F, T)`` for ``'Magnitude'`` and ``'Phase'`` and
    ``(B, F, T, 2)`` for ``'Complex'`` (real, imag), ``T = L // hop + 1`` when
    ``center=True``.
    """

    def __init__(
        self,
        n_fft=2048,
        win_length=None,
        freq_bins=None,
        hop_length=None,
        window="hann",
        freq_scale="no",
        center=True,
        pad_mode="reflect",
        iSTFT=False,
        fmin=50,
        fmax=6000,
        sr=22050,
        trainable=False,
        output_format="Complex",
        verbose=True,
    ):
        super().__init__()
        if win_length is None:
            win_length = n_fft
        if hop_length is None:
            hop_length = int(win_length // 4)

        self.output_format = output_format
        self.trainable = trainable
        self.stride = hop_length
        self.center = center
        self.pad_mode = pad_mode
        self.n_fft = n_fft
        self.freq_bins = freq_bins
        self.pad_amount = self.n_fft // 2
        self.window = window
        self.win_length = win_length
        self.iSTFT = iSTFT
        start = time()

        kernel_sin, kernel_cos, self.bins2freq, self.bin_list, window_mask = design.fourier_basis(
            n_fft,
            win_length=win_length,
            freq_bins=freq_bins,
            window=window,
            freq_scale=freq_scale,
            fmin=fmin,
            fmax=fmax,
            sr=sr,
            verbose=verbose,
        )
        kernel_sin = torch.tensor(kernel_sin, dtype=torch.float)
        kernel_cos = torch.tensor(kernel_cos, dtype=torch.float)

        if iSTFT:
            # inverse kernels for STFT.inverse (stft.py:217-223)
            sin_inv = torch.cat((kernel_sin, -kernel_sin[1:-1].flip(0)), 0)
            cos_inv = torch.cat((kernel_cos, kernel_cos[1:-1].flip(0)), 0)
            self.register_buffer("kernel_sin_inv", sin_inv.unsqueeze(-1))
            self.register_buffer("kernel_cos_inv", cos_inv.unsqueeze(-1))

        # window applied in fp32, like stft.py:230-232
        window_mask = torch.tensor(window_mask)
        wsin = kernel_sin * window_mask
        wcos = kernel_cos * window_mask
        if self.trainable:
            self.register_parameter("wsin", nn.Parameter(wsin, requires_grad=True))
            self.register_parameter("wcos", nn.Parameter(wcos, requires_grad=True))
        else:
            self.register_buffer("wsin", wsin)
            self.register_buffer("wcos", wcos)
        self.register_buffer("window_mask", window_mask.unsqueeze(0).unsqueeze(-1))

        self._packed = PackedBasis()
        if verbose:
            print("STFT kernels created, time used = {:.4f} seconds".format(time() - start))

    # ------------------------------------------------------------------ #
    def _checked_input(self, x):
        """Shape / length checks with the reference's exception types
        (utils.py:219-221, stft.py:283-286)."""
        self.num_samples = x.shape[-1]
        x = broadcast_dim(x)
        self._check_length(self.num_samples)
        return x

    def _check_length(self, n):
        """Raise what the reference raises for a clip of ``n`` samples (also the end of a stream)."""
        if self.center and self.pad_mode == "reflect":
            if n < self.pad_amount:
                raise AssertionError(
                    "Signal length shorter than reflect padding length (n_fft // 2)."
                )
            if n == self.pad_amount:
                raise RuntimeError(
                    "Padding size should be less than the corresponding input dimension"
                )
        pad = self.pad_amount if self.center else 0
        if n + 2 * pad < self.n_fft:
            raise RuntimeError("Kernel size can't be greater than actual input size")

    def _bases(self, block_ok=False):
        """``block_ok``: the caller's output format has a block-partial epilogue (all STFT formats,
        power / fused filterbank); the layout is still only used when the module is forward-only, the
        hop fits and the buffers pass ``is_hann_dft``."""
        wcos, wsin = as_matrix(self.wcos), as_matrix(self.wsin)
        if self.freq_bins is not None and self.freq_bins < wcos.shape[0]:
            wcos, wsin = wcos[: self.freq_bins], wsin[: self.freq_bins]
        # block-partial kernel: forward-only modules whose buffers are the periodic-Hann DFT
        block_hop = self.stride if (block_ok and not self.trainable) else 0
        return wcos, wsin, self._packed.get(wcos, wsin, block_hop=block_hop)

    def _infer_args(self, output_format):
        """(name, keyword arguments after ``x``) of the ``_C`` call of the inference path; the streaming
        API (nnaudio_b200.streaming) makes the same call per chunk."""
        wcos, wsin, packed = self._bases(block_ok=True)
        eps = 1e-8 if (self.trainable and output_format == "Magnitude") else 0.0
        return "stft_forward", dict(
            wcos=wcos, wsin=wsin, packed=packed, n_fft=self.n_fft, hop=self.stride, center=self.center,
            pad_mode=pad_mode_id(self.pad_mode), out_format=_FORMATS[output_format], sqrt_eps=eps,
        )

    def _run(self, x, output_format):
        return _C.stft_forward(x, **self._infer_args(output_format)[1])

    def _backward_input(self, g, L):
        wcos, wsin, _ = self._bases()
        if not hasattr(self, "_adjoint"):
            self._adjoint = AdjointBasis()
        return _C.framed_backward_input(g, self._adjoint.get(wcos, wsin), self.n_fft, self.stride,
                                        self.center, pad_mode_id(self.pad_mode), L)

    def _backward_weight(self, g, x):
        return _C.framed_backward_weight(g, x, self.n_fft, self.stride, self.center,
                                         pad_mode_id(self.pad_mode))

    def _complex_diff(self, x):
        """(B, F, T, 2) with gradient paths back to ``x`` and to trainable ``wcos`` / ``wsin``."""
        return FramedComplexFn.apply(x, self.wcos, self.wsin, lambda t: self._run(t, "Complex"),
                                     self._backward_input, self._backward_weight)

    def _magnitude_diff(self, x):
        c = self._complex_diff(x)
        spec = c[..., 0].pow(2) + c[..., 1].pow(2)
        return torch.sqrt(spec + 1e-8) if self.trainable else torch.sqrt(spec)

    def forward(self, x, output_format=None):
        output_format = output_format or self.output_format
        if output_format not in _FORMATS:
            raise ValueError(
                f"output_format must be 'Magnitude', 'Complex' or 'Phase', got {output_format!r}"
            )
        x = self._checked_input(x)
        if wants_grad(self, x):
            # training through the layer: fused complex contraction + dX kernel, the light
            # element-wise tail (stft.py:299-316) composed in torch for autograd
            x = upcast_16bit(x)
            if output_format == "Complex":
                return self._complex_diff(x)
            if output_format == "Magnitude":
                return self._magnitude_diff(x)
            c = self._complex_diff(x)
            return torch.atan2(c[..., 1] + 0.0, c[..., 0])
        return self._run(x, output_format)

    def inverse(self, X, onesided=True, length=None, refresh_win=True):
        """Inverse STFT of a complex spectrogram ``(B, bins, T, 2)`` (stft.py:318-356);
        needs ``iSTFT=True`` at construction.  ``refresh_win`` is accepted for signature
        compatibility: the window sum-square is recomputed on the fly in the kernel."""
        if not (hasattr(self, "kernel_sin_inv") and hasattr(self, "kernel_cos_inv")):
            raise NameError(
                "Please activate the iSTFT module by setting `iSTFT=True` if you want to use `inverse`"
            )
        assert X.dim() == 4, (
            "Inverse iSTFT only works for complex number,"
            "make sure our tensor is in the shape of (batch, freq_bins, timesteps, 2)."
            "\nIf you have a magnitude spectrogram, please consider using Griffin-Lim."
        )
        # only the tensors the inverse actually uses decide (a trainable *forward* STFT may call
        # .inverse() in training mode, as in the reference: trainable STFT -> process -> inverse)
        forward_only_guard(self, X, (self.kernel_cos_inv, self.kernel_sin_inv, self.window_mask))
        return _inverse_stft(self, X, self.kernel_cos_inv, self.kernel_sin_inv, self.window_mask,
                             onesided, length)

    def extra_repr(self) -> str:
        return "n_fft={}, Fourier Kernel size={}, iSTFT={}, trainable={}".format(
            self.n_fft, (*self.wsin.shape,), self.iSTFT, self.trainable
        )


class iSTFT(nn.Module):
    """Inverse STFT module — drop-in for ``nnAudio.features.stft.iSTFT`` (stft.py:364-546).
    Buffers: ``kernel_sin``, ``kernel_cos`` ``(n_fft, 1, n_fft, 1)`` (un-windowed inverse
    kernels) and ``window_mask`` ``(1, win_length, 1)``.  ``forward(X, onesided=False,
    length=None, refresh_win=None)`` takes ``(B, bins, T, 2)`` and returns ``(B, samples)``."""

    def __init__(
        self,
        n_fft=2048,
        win_length=None,
        freq_bins=None,
        hop_length=None,
        window="hann",
        freq_scale="no",
        center=True,
        fmin=50,
        fmax=6000,
        sr=22050,
        trainable_kernels=False,
        trainable_window=False,
        verbose=True,
        refresh_win=True,
    ):
        super().__init__()
        if win_length is None:
            win_length = n_fft
        if hop_length is None:
            hop_length = int(win_length // 4)
        self.n_fft = n_fft
        self.win_length = win_length
        self.stride = hop_length
        self.center = center
        self.pad_amount = self.n_fft // 2
        self.refresh_win = refresh_win
        start = time()

        kernel_sin, kernel_cos, _, _, _ = design.fourier_basis(
            n_fft, win_length=win_length, freq_bins=n_fft, window=window, freq_scale=freq_scale,
            fmin=fmin, fmax=fmax, sr=sr, verbose=False,
        )
        from scipy.signal import get_window

        window_mask = torch.tensor(get_window(window, int(win_length), fftbins=True))
        window_mask = window_mask.unsqueeze(0).unsqueeze(-1)
        kernel_sin = torch.tensor(kernel_sin, dtype=torch.float).unsqueeze(-1)
        kernel_cos = torch.tensor(kernel_cos, dtype=torch.float).unsqueeze(-1)
        if trainable_kernels:
            self.register_parameter("kernel_sin", nn.Parameter(kernel_sin, requires_grad=True))
            self.register_parameter("kernel_cos", nn.Parameter(kernel_cos, requires_grad=True))
        else:
            self.register_buffer("kernel_sin", kernel_sin)
            self.register_buffer("kernel_cos", kernel_cos)
        if trainable_window:
            self.register_parameter("window_mask", nn.Parameter(window_mask, requires_grad=True))
        else:
            self.register_buffer("window_mask", window_mask)
        if verbose:
            print("iSTFT kernels created, time used = {:.4f} seconds".format(time() - start))

    def forward(self, X, onesided=False, length=None, refresh_win=None):
        assert X.dim() == 4, (
            "Inverse iSTFT only works for complex number,"
            "make sure our tensor is in the shape of (batch, freq_bins, timesteps, 2)"
        )
        forward_only_guard(self, X)
        return _inverse_stft(self, X, self.kernel_cos, self.kernel_sin, self.window_mask, onesided,
                             length)
