"""``Gammatonegram`` — drop-in for ``nnAudio.features.gammatone.Gammatonegram``
(gammatone.py:9-194): the Mel pipeline with ``gammatone_basis (n_bins,
n_fft//2+1)`` as the filterbank."""
from __future__ import annotations

from time import time

import torch
import torch.nn as nn

from .. import _C, design
from ._common import FilterbankTable, pad_mode_id, upcast_16bit, wants_grad
from .stft import STFT


class Gammatonegram(nn.Module):
    """``gammatone_basis @ (|STFT(x)| ** power)`` -> ``(B, n_bins, T)``
    (constructor arguments: gammatone.py:93-112)."""

    def __init__(
        self,
        sr=22050,
        n_fft=2048,
        win_length=None,
        n_bins=64,
        hop_length=512,
        window="hann",
        center=True,
        pad_mode="reflect",
        power=2.0,
        htk=False,
        fmin=0.0,
        fmax=None,
        norm=1,
        trainable_bins=False,
        trainable_STFT=False,
        verbose=True,
        **kwargs,
    ):
        super().__init__()
        self.stride = hop_length
        self.center = center
        self.pad_mode = pad_mode
        self.n_fft = n_fft
        self.power = power
        self.trainable_bins = trainable_bins
        self.trainable_STFT = trainable_STFT

        self.stft = STFT(
            n_fft=n_fft,
            win_length=win_length,
            freq_bins=None,
            hop_length=hop_length,
            window=window,
            freq_scale="no",
            center=center,
            pad_mode=pad_mode,
            sr=sr,
            trainable=trainable_STFT,
            output_format="Magnitude",
            verbose=verbose,
            **kwargs,
        )

        start = time()
        basis = torch.tensor(design.gammatone_filterbank(sr, n_fft, n_bins, fmin, fmax))
        if verbose:
            print("STFT filter created, time used = {:.4f} seconds".format(time() - start))
            print("Gammatone filter created, time used = {:.4f} seconds".format(time() - start))
        if trainable_bins:
            self.register_parameter("gammatone_basis", nn.Parameter(basis, requires_grad=True))
        else:
            self.register_buffer("gammatone_basis", basis)
        self._fb_table = FilterbankTable()

    def forward(self, x):
        x = self.stft._checked_input(x)
        if wants_grad(self, x):
            return torch.matmul(self.gammatone_basis, self.stft._magnitude_diff(upcast_16bit(x)) ** self.power)
        return _C.stft_filterbank_forward(x, **self._infer_args()[1])

    def _infer_args(self):
        """(name, keyword arguments after ``x``) of the ``_C`` call of the inference path."""
        wcos, wsin, packed = self.stft._bases(block_ok=True)
        fb = self.gammatone_basis.detach()
        _C._dev_f32(fb, "gammatone_basis")
        fb = fb if fb.is_contiguous() else fb.contiguous()
        eps = 1e-8 if self.stft.trainable else 0.0
        return "stft_filterbank_forward", dict(
            wcos=wcos, wsin=wsin, packed=packed, n_fft=self.n_fft, hop=self.stride, center=self.center,
            pad_mode=pad_mode_id(self.pad_mode), sqrt_eps=eps, power=float(self.power), fb=fb,
            fb_table=self._fb_table.get(fb),
        )

    def extra_repr(self) -> str:
        return "Gammatone filter banks size = {}, trainable_bins={}".format(
            (*self.gammatone_basis.shape,), self.trainable_bins, self.trainable_STFT
        )
