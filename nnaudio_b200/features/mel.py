"""``MelSpectrogram`` and ``MFCC`` — drop-ins for ``nnAudio.features.mel``
(mel.py:9-194, :197-329).  Buffer names / shapes match the reference:
``mel_basis (n_mels, n_fft//2+1)``, ``stft.wsin/wcos/window_mask``;
``amin (1,)``, ``ref (1,)``, ``melspec_layer.*``.
"""
from __future__ import annotations

from time import time

import torch
import torch.nn as nn

from .. import _C, design
from ._common import FilterbankTable, pad_mode_id, upcast_16bit, wants_grad
from .stft import STFT


class MelSpectrogram(nn.Module):
    """``mel_basis @ (|STFT(x)| ** power)`` -> ``(B, n_mels, T)``
    (constructor arguments: mel.py:93-112)."""

    def __init__(
        self,
        sr=22050,
        n_fft=2048,
        win_length=None,
        n_mels=128,
        hop_length=512,
        window="hann",
        center=True,
        pad_mode="reflect",
        power=2.0,
        htk=False,
        fmin=0.0,
        fmax=None,
        norm=1,
        trainable_mel=False,
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
        self.trainable_mel = trainable_mel
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
        mel_basis = torch.tensor(design.mel_filterbank(sr, n_fft, n_mels, fmin, fmax, htk=htk, norm=norm))
        if verbose:
            print("STFT filter created, time used = {:.4f} seconds".format(time() - start))
            print("Mel filter created, time used = {:.4f} seconds".format(time() - start))
        if trainable_mel:
            self.register_parameter("mel_basis", nn.Parameter(mel_basis, requires_grad=True))
        else:
            self.register_buffer("mel_basis", mel_basis)
        self._fb_table = FilterbankTable()

    def _filterbank(self):
        return self.mel_basis

    def forward(self, x):
        x = self.stft._checked_input(x)
        if wants_grad(self, x):  # mel.py:186-188 on top of the differentiable STFT magnitude
            return torch.matmul(self._filterbank(), self.stft._magnitude_diff(upcast_16bit(x)) ** self.power)
        return _C.stft_filterbank_forward(x, **self._infer_args()[1])

    def _infer_args(self):
        """(name, keyword arguments after ``x``) of the ``_C`` call of the inference path."""
        wcos, wsin, packed = self.stft._bases(block_ok=True)
        fb = self._filterbank().detach()
        _C._dev_f32(fb, "filterbank")
        fb = fb if fb.is_contiguous() else fb.contiguous()
        eps = 1e-8 if self.stft.trainable else 0.0
        return "stft_filterbank_forward", dict(
            wcos=wcos, wsin=wsin, packed=packed, n_fft=self.n_fft, hop=self.stride, center=self.center,
            pad_mode=pad_mode_id(self.pad_mode), sqrt_eps=eps, power=float(self.power), fb=fb,
            fb_table=self._fb_table.get(fb),
        )

    def extra_repr(self) -> str:
        return "Mel filter banks size = {}, trainable_mel={}".format(
            (*self.mel_basis.shape,), self.trainable_mel, self.trainable_STFT
        )


class MFCC(nn.Module):
    """Mel-frequency cepstral coefficients ``(B, n_mfcc, T)``:
    mel power spectrogram -> dB with a per-clip ``top_db`` floor -> orthonormal
    DCT-II (mel.py:238-326; only ``norm='ortho'`` is implemented there too)."""

    def __init__(self, sr=22050, n_mfcc=20, norm="ortho", verbose=True, ref=1.0, amin=1e-10,
                 top_db=80.0, **kwargs):
        super().__init__()
        self.melspec_layer = MelSpectrogram(sr=sr, verbose=verbose, **kwargs)
        self.m_mfcc = n_mfcc
        if amin <= 0:
            raise design.ParameterError("amin must be strictly positive")
        self.register_buffer("amin", torch.tensor([amin]))
        self.register_buffer("ref", torch.abs(torch.tensor([ref])))
        self.top_db = top_db
        self.n_mfcc = n_mfcc
        n_mels = self.melspec_layer.mel_basis.shape[0]
        self.register_buffer(
            "_dct_rows", torch.tensor(design.dct2_ortho_matrix(min(n_mfcc, n_mels), n_mels)),
            persistent=False,
        )
        # scalar copies: reading the (1,) buffers back per forward would sync the stream
        self._amin_host = float(amin)
        self._ref_host = abs(float(ref))

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)
        self._amin_host = float(self.amin.detach().cpu()[0])
        self._ref_host = float(self.ref.detach().cpu()[0])

    def forward(self, x):
        if self.top_db is not None and self.top_db < 0:
            raise design.ParameterError("top_db must be non-negative")
        mel = self.melspec_layer
        x = mel.stft._checked_input(x)
        if wants_grad(self, x):  # mel.py:263-279, :281-307 composed in torch for autograd
            S = mel(upcast_16bit(x))
            amin = torch.tensor(self._amin_host, device=S.device)
            log_spec = 10.0 * torch.log10(torch.clamp(S, min=self._amin_host))
            log_spec = log_spec - 10.0 * torch.log10(torch.clamp(amin, min=self._ref_host))
            if self.top_db is not None:
                peak = log_spec.flatten(1).max(1)[0][:, None, None]
                log_spec = torch.max(log_spec, peak - self.top_db)
            return torch.matmul(self._dct_rows, log_spec)
        return _C.mfcc_forward(x, **self._infer_args()[1])

    def _infer_args(self):
        """(name, keyword arguments after ``x``) of the ``_C`` call of the inference path."""
        mel = self.melspec_layer
        wcos, wsin, packed = mel.stft._bases(block_ok=True)
        fb = mel.mel_basis.detach()
        _C._dev_f32(fb, "mel_basis")
        fb = fb if fb.is_contiguous() else fb.contiguous()
        eps = 1e-8 if mel.stft.trainable else 0.0
        return "mfcc_forward", dict(
            wcos=wcos, wsin=wsin, packed=packed, n_fft=mel.n_fft, hop=mel.stride, center=mel.center,
            pad_mode=pad_mode_id(mel.pad_mode), sqrt_eps=eps, power=float(mel.power), mel_basis=fb,
            amin=self._amin_host, ref=self._ref_host, top_db=self.top_db, dct=self._dct_rows,
            fb_table=mel._fb_table.get(fb),
        )

    def extra_repr(self) -> str:
        return "n_mfcc = {}".format((self.n_mfcc))
