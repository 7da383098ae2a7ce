"""Training through the modules: float64 reference graphs and the shape matrix of the training domain.

When a gradient is needed every module leaves its fused inference call and runs a host composition: the STFT family
(STFT, MelSpectrogram, MFCC, Gammatonegram) a ``FramedComplexFn`` contraction with the magnitude, phase, power,
filterbank matmul, dB, ``top_db`` floor and DCT done in torch; CQT1992v2 the un-normalised contraction, then scale and
format in torch; the CQT2010v2 / VQT pyramid an octave loop of FIR decimation stages and contractions; the inverse STFT
(``iSTFT``, ``STFT.inverse``) the window-sum-square adjoint followed by a forward contraction.

``reference(row, mod, x)`` restates each of these graphs in plain float64 torch from the formulas the modules cite
(the reference's conv1d over ``F.pad``, strided FIR conv1d with ``padding=(taps-1)//2``, its octave loop with the
reflect-to-constant fallback, and ``fold`` with the window sum-square for the inverse).  It reads only the module's
buffers and parameters, upcast to float64, so rounding of the bases is not counted as kernel error; it never calls
the module code it checks.  Gradients are float64 autograd of ``L = sum(W * y)`` with ``W`` seeded per row
(``weights``).

Ill-conditioned cells.  ``d|c|/dc = c/|c|`` and ``d angle(c)/dc`` grow without bound where ``|c| -> 0``, and a
``top_db`` floor switches a cell's gradient between the cell and the clip's peak.  A fp32 kernel that is 1e-5 off
near such a cell gives a gradient that is off by far more, whatever the kernel's quality (DESIGN §3.4, conditioning
note).  Rows whose output passes through the magnitude or phase of ``c`` (the trainable ``+1e-8`` bounds ``1/|c|`` only
at 1e4) therefore carry zero loss weight on cells with ``|c|`` below ``MASK_REL[fmt]`` of the clip's largest ``|c|``; MFCC rows take
coloured noise whose mel powers stay within ~60 dB of each frame's peak, and their ``top_db`` rows are checked to keep
every cell at least ``DB_MARGIN`` dB away from the floor and the peak unique by as much (tests/test_train_domain_host.py).
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

MAX_BATCH = 65535
MASK_REL = {"Magnitude": 1e-2, "Phase": 5e-2}   # zero loss weight below this fraction of the clip's max |c|
DB_MARGIN = 1e-3                                # dB between any MFCC cell and its clip's top_db floor / peak

# --------------------------------------------------------------------------------------------------- matrix ----
# name -> dict(family, cls, ctor, fwd (forward kwargs), B, L, sig (input kind), seed, dtype, params (trainable
#               parameter names), env (NNAUDIO_B200_PATH), edge (why the row is here), host (run through the CPU
#               stand-ins), inv (inverse rows: onesided, length, T))
ROWS = {}


def _row(name, family, cls, ctor, edge, B=2, L=8000, fwd=None, sig="noise", seed=None, dtype="float32",
         params=(), env=None, host=True, **extra):
    assert name not in ROWS
    ROWS[name] = dict(family=family, cls=cls, ctor=ctor, fwd=fwd or {}, B=B, L=L, sig=sig,
                      seed=len(ROWS) + 1 if seed is None else seed, dtype=dtype, params=tuple(params), env=env,
                      edge=edge, host=host, **extra)


# ---- STFT
_row("stft_block_complex", "stft", "STFT", dict(n_fft=2048, hop_length=512), "Complex at 2048/512: block-partial route",
     L=16000, fwd=dict(output_format="Complex"))
_row("stft_block_magnitude", "stft", "STFT", dict(n_fft=2048, hop_length=512), "Magnitude at 2048/512 (|c| mask)",
     L=16000, fwd=dict(output_format="Magnitude"))
_row("stft_block_phase", "stft", "STFT", dict(n_fft=2048, hop_length=512), "Phase at 2048/512 (|c| mask)",
     L=16000, fwd=dict(output_format="Phase"))
_row("stft_trainable", "stft", "STFT", dict(n_fft=512, hop_length=128, trainable=True),
     "trainable 512/128: dense route + dW, Magnitude with +1e-8 (|c| mask)", L=6000, fwd=dict(output_format="Magnitude"),
     params=("wsin", "wcos"))
_row("stft_oddhop_constant", "stft", "STFT", dict(n_fft=256, hop_length=99, pad_mode="constant"),
     "odd hop, constant padding: every frame phase", L=3001, fwd=dict(output_format="Complex"))
_row("stft_nocenter_tail", "stft", "STFT", dict(n_fft=512, hop_length=128, center=False),
     "center=False with 77 unread tail samples (x.grad exactly 0 there)", L=512 + 128 * 20 + 77,
     fwd=dict(output_format="Complex"))
_row("stft_gaps", "stft", "STFT", dict(n_fft=256, hop_length=400, center=False),
     "hop > n_fft: gaps between frames (x.grad exactly 0 there)", L=256 + 400 * 15 + 100,
     fwd=dict(output_format="Complex"))
_row("stft_16384_trainable", "stft", "STFT", dict(n_fft=16384, hop_length=4096, trainable=True),
     "n_fft 16384 trainable: split-K forward, chunked dX, split-K dW", B=1, L=16384 * 2,
     fwd=dict(output_format="Complex"), params=("wsin", "wcos"), host=False)
_row("stft_linear_bins", "stft", "STFT",
     dict(n_fft=256, freq_bins=80, freq_scale="linear", fmin=50, fmax=6000, sr=22050, hop_length=64, trainable=True),
     "freq_bins 80, linear scale: non-Hann basis, (80, 1, 256) dW", L=3000, fwd=dict(output_format="Complex"),
     params=("wsin", "wcos"))
_row("stft_log_bins", "stft", "STFT",
     dict(n_fft=256, freq_bins=60, freq_scale="log", fmin=50, fmax=6000, sr=22050, hop_length=64),
     "freq_bins 60, log scale (|c| mask)", L=3000, fwd=dict(output_format="Magnitude"))
_row("stft_hamming_winlen", "stft", "STFT", dict(n_fft=512, win_length=400, window="hamming", hop_length=128),
     "win_length 400 < n_fft 512, Hamming", L=4000, fwd=dict(output_format="Complex"))
_row("stft_simt", "stft", "STFT", dict(n_fft=512, hop_length=128), "forced SIMT path", L=4000,
     fwd=dict(output_format="Complex"), env="simt")
_row("stft_b40", "stft", "STFT", dict(n_fft=1024, hop_length=256), "B = 40", B=40, L=4000,
     fwd=dict(output_format="Complex"))
_row("stft_bf16", "stft", "STFT", dict(n_fft=512, hop_length=128), "bfloat16 waveform", L=4000,
     fwd=dict(output_format="Complex"), dtype="bfloat16")
_row("stft_fp16", "stft", "STFT", dict(n_fft=512, hop_length=128, trainable=True), "float16 waveform, trainable",
     L=4000, fwd=dict(output_format="Complex"), dtype="float16", params=("wsin", "wcos"))
_row("stft_b65536", "stft", "STFT", dict(n_fft=256, hop_length=64, trainable=True),
     "B = 65 536 short clips, trainable: chunked dX and dW", B=65536, L=512, fwd=dict(output_format="Complex"),
     params=("wsin", "wcos"), host=False)

# ---- Mel / Gammatonegram
_row("mel_power2", "mel", "MelSpectrogram", dict(sr=16000, n_fft=512, hop_length=128, n_mels=40), "power 2", L=8000)
_row("mel_power1_trainable_stft", "mel", "MelSpectrogram",
     dict(sr=16000, n_fft=512, hop_length=128, n_mels=40, power=1.0, trainable_STFT=True),
     "power 1, trainable STFT (+1e-8 bounds c/|c|)", L=8000, params=("stft.wsin", "stft.wcos"))
_row("mel_trainable_mel", "mel", "MelSpectrogram",
     dict(sr=16000, n_fft=256, hop_length=64, n_mels=20, trainable_mel=True, trainable_STFT=True),
     "trainable mel and STFT", L=4000, params=("mel_basis", "stft.wsin", "stft.wcos"))
_row("mel_htk_fmax", "mel", "MelSpectrogram",
     dict(sr=22050, n_fft=1024, hop_length=256, n_mels=64, htk=True, fmax=7000.0), "htk, fmax edge", L=11025)
_row("mel_128_2048", "mel", "MelSpectrogram", dict(sr=22050, n_fft=2048, hop_length=512, n_mels=128),
     "128 mels at 2048", L=22050)
_row("gamma_trainable", "mel", "Gammatonegram",
     dict(sr=22050, n_fft=1024, n_bins=33, hop_length=300, trainable_bins=True),
     "trainable gammatone basis, hop 300, 33 bins", L=9000, params=("gammatone_basis",))
_row("mel_bf16", "mel", "MelSpectrogram", dict(sr=16000, n_fft=512, hop_length=128, n_mels=40),
     "bfloat16 waveform", L=8000, dtype="bfloat16")
_row("gamma_fp16", "mel", "Gammatonegram", dict(sr=22050, n_fft=1024, n_bins=33, hop_length=256),
     "float16 waveform", L=9000, dtype="float16")

# ---- MFCC (coloured noise: mel powers within ~60 dB of each frame's peak)
_MF = dict(sr=16000, n_fft=512, hop_length=160, n_mels=40, n_mfcc=13)
_row("mfcc_db80", "mfcc", "MFCC", dict(_MF, top_db=80.0), "top_db 80 (floor inactive), unique per-clip peak",
     L=8000, sig="decay")
_row("mfcc_db10", "mfcc", "MFCC", dict(_MF, top_db=10.0), "top_db 10: floor active on most cells", L=8000,
     sig="decay")
_row("mfcc_nodb", "mfcc", "MFCC", dict(_MF, top_db=None), "top_db=None", L=8000, sig="decay")
_row("mfcc_full", "mfcc", "MFCC", dict(_MF, n_mfcc=40), "n_mfcc == n_mels", L=8000, sig="decay")
_row("mfcc_fp16", "mfcc", "MFCC", dict(_MF), "float16 waveform", L=8000, sig="decay", dtype="float16")
_row("mfcc_bf16", "mfcc", "MFCC", dict(_MF, top_db=None), "bfloat16 waveform", L=8000, sig="decay", dtype="bfloat16")

# ---- CQT1992v2
_C92 = dict(sr=22050, fmin=220, n_bins=48, hop_length=256)
_row("cqt_dense_complex", "cqt", "CQT1992v2", _C92, "dense route, Complex, librosa", L=16000,
     fwd=dict(output_format="Complex"))
_row("cqt_trainable_mag", "cqt", "CQT1992v2", dict(_C92, trainable=True), "trainable: dense route + dW, Magnitude (|c| mask)",
     L=16000, fwd=dict(output_format="Magnitude"), params=("cqt_kernels_real", "cqt_kernels_imag"))
_row("cqt_phase_conv", "cqt", "CQT1992v2", _C92, "Phase, convolutional (|c| mask)", L=16000,
     fwd=dict(output_format="Phase", normalization_type="convolutional"))
_row("cqt_wrap_constant", "cqt", "CQT1992v2", dict(_C92, pad_mode="constant"), "wrap, constant padding", L=16000,
     fwd=dict(output_format="Complex", normalization_type="wrap"))
_row("cqt_long_grouped", "cqt", "CQT1992v2", dict(sr=22050, fmin=32.7, n_bins=84, hop_length=512),
     "long bank, hop 512: grouped layout, tall-A route", B=2, L=44100,
     fwd=dict(output_format="Complex", normalization_type="convolutional"))
_row("cqt_long_dense", "cqt", "CQT1992v2", dict(sr=22050, fmin=32.7, n_bins=84, hop_length=500),
     "long bank, hop 500: dense layout, split-K", B=1, L=44100, fwd=dict(output_format="Magnitude"))
_row("cqt_long_trainable", "cqt", "CQT1992v2", dict(sr=22050, fmin=65.4, n_bins=72, hop_length=512, trainable=True),
     "long trainable bank: dense split-K + dW", B=1, L=30000, fwd=dict(output_format="Complex"),
     params=("cqt_kernels_real", "cqt_kernels_imag"))
_row("cqt_simt", "cqt", "CQT1992v2", _C92, "forced SIMT path", L=16000, fwd=dict(output_format="Complex"), env="simt")
_row("cqt_b40", "cqt", "CQT1992v2", _C92, "B = 40", B=40, L=6000, fwd=dict(output_format="Complex"))
_row("cqt_varn", "cqt", "CQT1992v2", dict(sr=22050, fmin=32.7, n_bins=84, hop_length=520),
     "long bank, hop 520 (a multiple of 8, not of 64): per-K-block-width (VarN) route, split-K", B=2, L=44100,
     fwd=dict(output_format="Complex", normalization_type="convolutional"))
_row("cqt_fp16", "cqt", "CQT1992v2", dict(_C92, trainable=True), "float16 waveform, trainable", L=16000,
     fwd=dict(output_format="Complex"), dtype="float16", params=("cqt_kernels_real", "cqt_kernels_imag"))
_row("cqt_bf16", "cqt", "CQT1992v2", _C92, "bfloat16 waveform", L=16000, fwd=dict(output_format="Complex"),
     dtype="bfloat16")

# ---- CQT2010v2 / VQT pyramid
_row("pyr_early4_complex", "pyramid", "CQT2010v2", dict(sr=44100, n_bins=72, fmin=32.7),
     "early downsampling by 4, Complex, convolutional", B=1, L=65536,
     fwd=dict(output_format="Complex", normalization_type="convolutional"))
_row("pyr_early2_magnitude", "pyramid", "CQT2010v2", dict(sr=22050, n_bins=48, fmin=110),
     "early downsampling by 2, Magnitude (|c| mask)", L=16384, fwd=dict(output_format="Magnitude"))
_row("pyr_noearly_wrap", "pyramid", "CQT2010v2", dict(sr=22050, n_bins=84), "no early downsampling, wrap",
     L=32768, fwd=dict(output_format="Complex", normalization_type="wrap"))
_row("pyr_fallback", "pyramid", "CQT2010v2", dict(sr=22050, n_bins=84), "reflect -> constant fallback, short clip",
     B=1, L=8192, fwd=dict(output_format="Complex"))
_row("pyr_crop", "pyramid", "CQT2010v2", dict(sr=22050, n_bins=30, fmin=220), "n_bins 30 = 2.5 octaves: crop",
     L=16384, fwd=dict(output_format="Complex"))
_row("pyr_24bpo_phase", "pyramid", "CQT2010v2", dict(sr=22050, n_bins=72, bins_per_octave=24, fmin=65),
     "24 bins per octave, Phase (|c| mask)", B=1, L=32768, fwd=dict(output_format="Phase"))
_row("vqt_gamma5", "pyramid", "VQT", dict(sr=22050, gamma=5, n_bins=60), "VQT gamma 5", B=1, L=32768,
     fwd=dict(output_format="Complex"))
_row("vqt_gamma0", "pyramid", "VQT", dict(sr=22050, gamma=0, n_bins=48, fmin=65), "VQT gamma 0", B=1, L=32768,
     fwd=dict(output_format="Complex", normalization_type="convolutional"))
_row("pyr_trainable", "pyramid", "CQT2010v2", dict(sr=22050, n_bins=48, fmin=110, trainable=True),
     "trainable shared bank: dW summed over octaves (|c| mask)", L=16384, fwd=dict(output_format="Magnitude"),
     params=("cqt_kernels_real", "cqt_kernels_imag"))
_row("pyr_fp16", "pyramid", "CQT2010v2", dict(sr=22050, n_bins=48, fmin=110), "float16 waveform", L=16384,
     fwd=dict(output_format="Complex"), dtype="float16")
_row("pyr_bf16", "pyramid", "VQT", dict(sr=22050, gamma=5, n_bins=48, fmin=110), "bfloat16 waveform", L=16384,
     fwd=dict(output_format="Complex"), dtype="bfloat16")

# ---- v1 CQT1992 (one folded time-domain bank) and CQT2010 (the folded bank in every octave)
_V1 = dict(sr=22050, fmin=880, n_bins=24, hop_length=128)
_row("v1_stft_complex", "v1", "CQT1992", dict(_V1, trainable_STFT=True), "trainable_STFT, Complex (negated imag)",
     L=6000, fwd=dict(output_format="Complex"), params=("wsin", "wcos"))
_row("v1_cqt_magnitude", "v1", "CQT1992", dict(_V1, trainable_CQT=True), "trainable_CQT, Magnitude (|c| mask)",
     L=6000, fwd=dict(output_format="Magnitude"), params=("cqt_kernels_real", "cqt_kernels_imag"))
_row("v1_both_phase", "v1", "CQT1992", dict(_V1, trainable_STFT=True, trainable_CQT=True),
     "trainable_STFT and trainable_CQT, Phase (un-negated imag, |c| mask), wrap", L=6000,
     fwd=dict(output_format="Phase", normalization_type="wrap"),
     params=("wsin", "wcos", "cqt_kernels_real", "cqt_kernels_imag"))
_row("v1_cqt_constant_nocenter", "v1", "CQT1992", dict(_V1, trainable_CQT=True, center=False, pad_mode="constant"),
     "trainable_CQT, center False, Complex, convolutional", L=6000,
     fwd=dict(output_format="Complex", normalization_type="convolutional"),
     params=("cqt_kernels_real", "cqt_kernels_imag"))
_V2010 = dict(sr=22050, n_bins=36, fmin=110)
_row("cqt2010_cqt_complex", "pyramid", "CQT2010", dict(_V2010, trainable_CQT=True),
     "CQT2010, trainable_CQT, Complex (un-negated imag, no downsample factor)", L=16384,
     fwd=dict(output_format="Complex"), params=("cqt_kernels_real", "cqt_kernels_imag"))
_row("cqt2010_stft_magnitude", "pyramid", "CQT2010", dict(_V2010, trainable_STFT=True),
     "CQT2010, trainable_STFT, Magnitude (|c| mask), wrap", L=16384,
     fwd=dict(output_format="Magnitude", normalization_type="wrap"), params=("wsin", "wcos"))
_row("cqt2010_phase", "pyramid", "CQT2010", dict(_V2010, earlydownsample=False), "CQT2010, Phase (|c| mask)",
     B=1, L=16384, fwd=dict(output_format="Phase"))

_row("pyr_b65536", "pyramid", "CQT2010v2",
     dict(sr=8000, n_bins=24, fmin=500, hop_length=64, earlydownsample=False),
     "B = 65 536 short clips: chunked FIR stages, dX", B=65536, L=512, fwd=dict(output_format="Complex"), host=False)

# ---- inverse STFT (X: a seeded spectrum (B, f_in, T, 2))
_row("istft_onesided_len", "istft", "STFT", dict(n_fft=512, hop_length=128, iSTFT=True),
     "STFT.inverse, one-sided, length = samples", L=4000, T=32, onesided=True, length=4000)
_row("istft_full_center", "istft", "iSTFT", dict(n_fft=256, hop_length=64), "iSTFT, full spectrum, length None",
     T=40, onesided=False, length=None)
_row("istft_nocenter", "istft", "iSTFT", dict(n_fft=256, hop_length=64, center=False),
     "center False, length None: ends where wss <= 1e-10", T=40, onesided=False, length=None)
_row("istft_short", "istft", "STFT", dict(n_fft=256, hop_length=64, iSTFT=True), "length shorter than the clip",
     T=40, onesided=True, length=1000)
_row("istft_long", "istft", "STFT", dict(n_fft=256, hop_length=64, iSTFT=True), "length past the last frame",
     T=40, onesided=True, length=5000)
_row("istft_hop_half", "istft", "iSTFT", dict(n_fft=512, hop_length=256), "hop n_fft / 2", T=30,
     onesided=True, length=None)
_row("istft_hop_nondiv", "istft", "iSTFT", dict(n_fft=256, hop_length=100, center=False),
     "hop 100 does not divide n_fft; center False", T=30, onesided=True, length=None)
_row("istft_8192", "istft", "STFT", dict(n_fft=8192, hop_length=2048, iSTFT=True), "n_fft 8192: chunked K",
     B=1, T=12, onesided=True, length=None)
_row("istft_b65536", "istft", "iSTFT", dict(n_fft=64, hop_length=16), "B = 65 536 short clips", B=65536, T=4,
     onesided=True, length=None, host=False)

FAMILIES = ("stft", "mel", "mfcc", "cqt", "v1", "pyramid", "istft")


# ------------------------------------------------------------------------------------------------ inputs ----
def make_input(name, B=None):
    """The row's float32 waveform (B, L), or for inverse rows its spectrum (B, f_in, T, 2); float32 on the CPU."""
    r = ROWS[name]
    B = r["B"] if B is None else B
    g = torch.Generator().manual_seed(1000 + r["seed"])
    if r["family"] == "istft":
        n_fft = r["ctor"]["n_fft"]
        f_in = n_fft // 2 + 1 if r["onesided"] else n_fft
        return torch.randn((B, f_in, r["T"], 2), generator=g)
    x = torch.randn((B, r["L"]), generator=g)
    if r["sig"] == "decay":
        # coloured noise (first-order lowpass) under a decaying envelope: 50+ dB of level across the clip and
        # different levels per clip, with no mel band near silence
        x = torch.from_numpy(np.asarray(_onepole(x.numpy().astype(np.float64), 0.6), dtype=np.float32))
        t = torch.linspace(0, 1, r["L"])
        x = x * torch.exp(-6.0 * t)[None, :] * (0.5 ** torch.arange(B, dtype=torch.float32))[:, None]
    return x.contiguous()


def _onepole(x, a):
    from scipy.signal import lfilter
    return lfilter([1.0 - a], [1.0, -a], x, axis=-1)


def weights(name, shape, device="cpu"):
    """The row's loss weights W (float64), seeded per row."""
    g = torch.Generator().manual_seed(7919 * (ROWS[name]["seed"] + 1))
    return torch.randn(tuple(shape), generator=g, dtype=torch.float64).to(device)


# ------------------------------------------------------------------------------------- reference graphs ----
def _d(t):
    return t.detach().double()


def _padded(x, pad, mode):
    """(B, L) -> padded (B, 1, L + 2 pad), the reference's nn.ReflectionPad1d / ConstantPad1d; a reflection pad
    longer than the signal falls back to zeros, as the reference's get_cqt_complex does (utils.py:505-517)."""
    x = x[:, None, :]
    if pad == 0:
        return x
    if mode == "reflect":
        try:
            return F.pad(x, (pad, pad), mode="reflect")
        except RuntimeError:
            pass
    return F.pad(x, (pad, pad))


def framed(x, w_re, w_im, hop, center, mode):
    """(B, L) float64 -> (B, F, T, 2) = (conv1d(x, w_re), -conv1d(x, w_im)) over the padded signal."""
    K = w_re.shape[-1]
    xp = _padded(x, K // 2 if center else 0, mode)
    re = F.conv1d(xp, w_re[:, None, :], stride=hop)
    im = -F.conv1d(xp, w_im[:, None, :], stride=hop)
    return torch.stack((re, im), -1)


def _fir(x, fir, n):
    taps = fir.numel()
    return F.conv1d(x[:, None, :], fir.reshape(1, 1, -1), stride=n, padding=(taps - 1) // 2)[:, 0, :]


def _cqt_format(c, fmt, eps):
    if fmt == "Complex":
        return c
    if fmt == "Magnitude":
        return torch.sqrt(c[..., 0] ** 2 + c[..., 1] ** 2 + eps)
    ang = torch.atan2(c[..., 1], c[..., 0])
    return torch.stack((torch.cos(ang), torch.sin(ang)), -1)


def dct_ortho(n_out, n):
    """Orthonormal DCT-II rows (mel.py:281-307): D[k, i] = sqrt(2/n) cos(pi k (2i + 1) / (2n)), row 0 / sqrt(2)."""
    k = torch.arange(n_out, dtype=torch.float64)[:, None]
    i = torch.arange(n, dtype=torch.float64)[None, :]
    D = math.sqrt(2.0 / n) * torch.cos(math.pi * k * (2 * i + 1) / (2 * n))
    D[0] /= math.sqrt(2.0)
    return D


def _leaves(mod, names, device):
    """Float64 leaf copies of the module's named tensors (upcast), requiring grad where ``names`` lists them."""
    out = {}
    for n, t in list(mod.named_parameters()) + list(mod.named_buffers()):
        if t is None:
            continue
        v = _d(t).to(device)
        if n in names:
            v.requires_grad_(True)
        out[n] = v
    return out


def _stft_complex(P, prefix, st, x):
    return framed(x, _mat2(P[prefix + "wcos"]), _mat2(P[prefix + "wsin"]), st.stride, st.center, st.pad_mode)


def _stft_magnitude(c, trainable):
    spec = c[..., 0] ** 2 + c[..., 1] ** 2
    return torch.sqrt(spec + 1e-8) if trainable else torch.sqrt(spec)


def _mel(P, prefix, mod, x, fb_name):
    st = mod.stft
    c = _stft_complex(P, prefix + "stft.", st, x)
    return torch.matmul(P[prefix + fb_name], _stft_magnitude(c, st.trainable) ** mod.power), c


def _mfcc(P, mod, x):
    S, c = _mel(P, "melspec_layer.", mod.melspec_layer, x, "mel_basis")
    amin, ref = float(mod.amin[0]), float(mod.ref[0])
    db = 10.0 * torch.log10(torch.clamp(S, min=amin)) - 10.0 * math.log10(max(amin, abs(ref)))
    pre = db
    if mod.top_db is not None:
        peak = db.flatten(1).max(1)[0][:, None, None]
        db = torch.max(db, peak - mod.top_db)
    # the module's fp32 DCT rows, like every other basis (tests/test_train_domain_host.py holds them to dct_ortho)
    return torch.matmul(P["_dct_rows"], db), c, pre


def _fp32_scale(lenghts, factor):
    """The per-bin factor sqrt(lenghts) * factor as the fp32 vector the modules hand the kernels (its rounding,
    <= 6e-8, is not kernel error)."""
    s = torch.sqrt(lenghts.detach().float())
    return (s * factor if factor != 1 else s).double()


def _cqt1992v2(P, mod, x, fmt, norm):
    c = framed(x, _mat2(P["cqt_kernels_real"]), _mat2(P["cqt_kernels_imag"]), mod.hop_length, mod.center,
               mod.pad_mode)
    raw = c
    if norm == "librosa":
        c = c * _fp32_scale(mod.lenghts, 1.0).to(x.device).view(1, -1, 1, 1)
    elif norm == "wrap":
        c = c * 2.0
    eps = 1e-8 if (mod.trainable and fmt == "Magnitude") else 0.0
    return _cqt_format(c, fmt, eps), raw


def _mat2(t):
    return t.reshape(t.shape[0], t.shape[-1])


def _v1_octave(P, x, hop, pad, mode):
    """One v1 octave in the reference's two-stage form (cqt.py:205-222, utils.py:524-559): an un-windowed DFT of
    the padded frames (conv1d with wcos / wsin), then complex_mul with the spectral kernels.  (re, im) before the
    per-class sign of the imaginary part."""
    xp = _padded(x, pad, mode)
    fr = F.conv1d(xp, P["wcos"], stride=hop)
    fi = F.conv1d(xp, P["wsin"], stride=hop)
    kr, ki = P["cqt_kernels_real"], P["cqt_kernels_imag"]
    return torch.matmul(kr, fr) - torch.matmul(ki, fi), torch.matmul(kr, fi) + torch.matmul(ki, fr)


def _v1_format(c, re, im, fmt):
    """cqt.py:241-252: Magnitude and Complex from the stacked c, Phase from atan2 of (im, re) as given."""
    if fmt == "Complex":
        return c
    if fmt == "Magnitude":
        return torch.sqrt(c.pow(2).sum(-1))
    ang = torch.atan2(im, re)
    return torch.stack((torch.cos(ang), torch.sin(ang)), -1)


def _cqt1992_v1(P, mod, x, fmt, norm):
    """cqt.py:189-256: Complex / Magnitude stack (re, -im); Phase takes the angle of the un-negated (re, im)."""
    pad = mod.kernel_width // 2 if mod.center else 0
    re, im = _v1_octave(P, x, mod.hop_length, pad, mod.pad_mode)
    c = torch.stack((re, -im), -1)
    raw = c
    s = 1.0
    if norm == "librosa":
        s = _fp32_scale(mod.lenghts, 1.0 / mod.kernel_width).to(x.device).view(1, -1, 1)
    elif norm == "wrap":
        s = 2.0 / mod.kernel_width
    return _v1_format(c * (s[..., None] if torch.is_tensor(s) else s), re * s, im * s, fmt), raw


def _cqt2010_v1(P, mod, x, fmt, norm):
    """cqt.py:481-553: the octave loop of get_cqt_complex2 (stacked (re, im), not negated), crop, then 'librosa' /
    'wrap' divide by n_fft and no early-downsample factor is applied."""
    if mod.earlydownsample:
        x = _fir(x, P["early_downsample_filter"], int(mod.downsample_factor))
    hop = mod.hop_length
    re, im = _v1_octave(P, x, hop, mod.n_fft // 2, mod.pad_mode)
    cur = x
    for _ in range(1, mod.n_octaves):
        hop //= 2
        cur = _fir(cur, P["lowpass_filter"], 2)
        r1, i1 = _v1_octave(P, cur, hop, mod.n_fft // 2, mod.pad_mode)
        re, im = torch.cat((r1, re), 1), torch.cat((i1, im), 1)
    c = torch.stack((re, im), -1)[:, -mod.n_bins:]
    raw = c
    if norm == "librosa":
        c = c * _fp32_scale(mod.lenghts, 1.0 / mod.n_fft).to(x.device).view(1, -1, 1, 1)
    elif norm == "wrap":
        c = c * (2.0 / mod.n_fft)
    return _v1_format(c, c[..., 0], c[..., 1], fmt), raw


def _pyramid(P, mod, x, fmt, norm):
    """cqt.py:1085-1139 / vqt.py:160-215: optional early decimation, top octave first, each lower octave on the
    ÷2-decimated signal at half the hop, octaves concatenated low -> high, the lowest surplus bins cropped."""
    if mod.earlydownsample:
        x = _fir(x, P["early_downsample_filter"], int(mod.downsample_factor))
    hop = mod.hop_length
    lowpass = P["lowpass_filter"]
    if "cqt_kernels_real" in P:
        banks = [(P["cqt_kernels_real"], P["cqt_kernels_imag"])] * mod.n_octaves
    else:
        banks = [(P[f"cqt_kernels_real_{i}"], P[f"cqt_kernels_imag_{i}"]) for i in range(mod.n_octaves)]
    cur = x
    c = framed(cur, _mat2(banks[0][0]), _mat2(banks[0][1]), hop, True, mod.pad_mode)
    for i in range(1, mod.n_octaves):
        hop //= 2
        cur = _fir(cur, lowpass, 2)
        c = torch.cat((framed(cur, _mat2(banks[i][0]), _mat2(banks[i][1]), hop, True, mod.pad_mode), c), 1)
    c = c[:, -mod.n_bins:]
    raw = c
    dsf = float(mod.downsample_factor)
    if norm == "librosa":
        c = c * _fp32_scale(mod.lenghts, dsf).to(x.device).view(1, -1, 1, 1)
    elif norm == "wrap":
        c = c * (2.0 * dsf)
    else:
        c = c * dsf
    eps = 1e-8 if (mod.trainable and fmt == "Magnitude") else 0.0
    return _cqt_format(c, fmt, eps), raw


def _istft(P, mod, X, onesided, length):
    """stft.py:15-63: mirror a one-sided spectrum, real = (kc X_re - ks X_im) * window / n_fft per frame,
    overlap-add with fold, divide by the window sum-square where it exceeds 1e-10, strip the centre padding."""
    n_fft, hop = mod.n_fft, mod.stride
    if "kernel_cos_inv" in P:
        kc, ks = P["kernel_cos_inv"], P["kernel_sin_inv"]
    else:
        kc, ks = P["kernel_cos"], P["kernel_sin"]
    kc, ks = kc.reshape(n_fft, n_fft), ks.reshape(n_fft, n_fft)
    win = P["window_mask"].reshape(-1).float().double()     # the modules' fp32 window
    if onesided:
        up = X[:, 1:-1].flip(1)
        up = torch.stack((up[..., 0], -up[..., 1]), -1)
        X = torch.cat((X, up), 1)
    real = torch.einsum("of,bft->bot", kc, X[..., 0]) - torch.einsum("of,bft->bot", ks, X[..., 1])
    real = real * win[None, :, None] / n_fft
    T = X.shape[2]
    out_len = n_fft + hop * (T - 1)
    ola = F.fold(real, (1, out_len), (1, n_fft), stride=(1, hop)).flatten(1)
    wsum = F.fold((win ** 2)[None, :, None].expand(1, n_fft, T), (1, out_len), (1, n_fft),
                  stride=(1, hop)).flatten()
    nz = wsum > 1e-10
    ola = torch.where(nz[None, :], ola / torch.where(nz, wsum, torch.ones_like(wsum))[None, :], ola)
    pad = n_fft // 2
    if length is None:
        return ola[:, pad:-pad] if mod.center else ola
    return ola[:, pad:pad + length] if mod.center else ola[:, :length]


def reference(name, mod, x):
    """Float64 forward of row ``name`` through ``mod``'s buffers.  Returns (y, leaves, extra): ``leaves`` maps the
    row's trainable parameter names to their float64 leaves (plus ``"x"``), ``extra`` holds the un-normalised
    complex contraction (``"c"``) and, for MFCC, the pre-floor dB (``"db"``)."""
    r = ROWS[name]
    dev = x.device
    P = _leaves(mod, r["params"], dev)
    xd = _d(x).to(dev).requires_grad_(True)
    fam, fmt = r["family"], r["fwd"].get("output_format")
    extra = {}
    if fam == "stft":
        c = _stft_complex(P, "", mod, xd)
        extra["c"] = c
        if fmt == "Complex":
            y = c
        elif fmt == "Magnitude":
            y = _stft_magnitude(c, mod.trainable)
        else:
            y = torch.atan2(c[..., 1] + 0.0, c[..., 0])
    elif fam == "mel":
        fb = "mel_basis" if r["cls"] == "MelSpectrogram" else "gammatone_basis"
        y, extra["c"] = _mel(P, "", mod, xd, fb)
    elif fam == "mfcc":
        y, extra["c"], extra["db"] = _mfcc(P, mod, xd)
    elif fam == "cqt":
        y, extra["c"] = _cqt1992v2(P, mod, xd, fmt, r["fwd"].get("normalization_type", "librosa"))
    elif fam == "v1":
        y, extra["c"] = _cqt1992_v1(P, mod, xd, fmt, r["fwd"].get("normalization_type", "librosa"))
    elif fam == "pyramid" and r["cls"] == "CQT2010":
        y, extra["c"] = _cqt2010_v1(P, mod, xd, fmt, r["fwd"].get("normalization_type", "librosa"))
    elif fam == "pyramid":
        y, extra["c"] = _pyramid(P, mod, xd, fmt, r["fwd"].get("normalization_type", "librosa"))
    else:
        y = _istft(P, mod, xd, r["onesided"], r["length"])
    leaves = {n: P[n] for n in r["params"]}
    leaves["x"] = xd
    return y, leaves, extra


def loss_mask(name, y, extra):
    """Float64 0/1 mask over y's cells (broadcast to y's shape) that keeps the loss off ill-conditioned cells."""
    r = ROWS[name]
    fmt = r["fwd"].get("output_format")
    ones = torch.ones_like(y, dtype=torch.float64)
    if fmt not in MASK_REL or r["family"] not in ("stft", "cqt", "v1", "pyramid"):
        return ones
    c = extra["c"].detach()
    mag = torch.sqrt(c[..., 0] ** 2 + c[..., 1] ** 2)
    peak = mag.flatten(1).max(1)[0].view(-1, 1, 1)
    keep = (mag >= MASK_REL[fmt] * peak).double()
    return keep[..., None].expand_as(y) if y.dim() == 4 else keep


def gradients(name, mod, x):
    """(y, {name: grad}, W, extra) of the float64 graph for ``L = sum(W * mask * y)``."""
    y, leaves, extra = reference(name, mod, x)
    W = weights(name, y.shape, y.device) * loss_mask(name, y, extra)
    (y * W).sum().backward()
    return y.detach(), {n: t.grad for n, t in leaves.items()}, W, extra


def gradients_by_parts(name, mod, x, part=8192):
    """``gradients`` of a large unmasked batch, ``part`` clips per float64 graph (torch's own float64 convolutions
    take no more than 65 535 clips per launch): y and x.grad concatenated, parameter gradients summed."""
    assert not any(ROWS[name]["fwd"].get("output_format") == f for f in MASK_REL)
    with torch.no_grad():
        y0 = reference(name, mod, x[:1])[0]
    W = weights(name, (x.shape[0],) + tuple(y0.shape[1:]), x.device)
    ys, gs = [], {}
    for i in range(0, x.shape[0], part):
        y, leaves, _ = reference(name, mod, x[i:i + part])
        (y * W[i:i + part]).sum().backward()
        ys.append(y.detach())
        for n, t in leaves.items():
            gs.setdefault(n, []).append(t.grad)
    grads = {n: torch.cat(v, 0) if n == "x" else sum(v[1:], v[0]) for n, v in gs.items()}
    return torch.cat(ys, 0), grads, W


def mfcc_margins(name, mod, x):
    """(smallest distance in dB of any cell from its clip's top_db floor, gap between the two largest cells of
    a clip) of an MFCC row, in float64."""
    with torch.no_grad():
        _, _, extra = reference(name, mod, x)
    db = extra["db"].flatten(1)
    top = db.topk(2, dim=1)[0]
    gap = float((top[:, 0] - top[:, 1]).min())
    if mod.top_db is None:
        return math.inf, gap
    floor = top[:, :1] - mod.top_db
    return float((db - floor).abs().min()), gap


# ------------------------------------------------------------------------------------------- launch model ----
# What each row's training forward and backward() launch: the routes they move (("stft" | "cq" | "pyr", route
# constant) -> count, from the offline route counters of nnaudio_b200._C) and the executed MMA flops they add, taken
# from the kernel-domain models (dense_domain.plan for the STFT family's contraction, cqt1992_domain.plan for every
# CQT1992v2-kernel call, ola_domain for the overlap-add GEMMs of dX, dW and the inverse).  The FIR decimation stages
# and their adjoints are CUDA-core kernels: no MMA flops and no PYR_* counter.
def _chunks(B):
    return [min(MAX_BATCH, B - i) for i in range(0, B, MAX_BATCH)]


def _bank_shim(F_, K, hop, center):
    """A stand-in for a CQT1992v2 module with an (F_, K) bank packed dense and no tap support: the layout every
    contraction of the training path that is not a CQT1992v2 module's own passes (octave banks, v1 folded banks,
    the inverse STFT's adjoint)."""
    from types import SimpleNamespace
    return SimpleNamespace(cqt_kernels_real=torch.empty(F_, 1, K), cqt_kernels_imag=torch.empty(F_, 1, K),
                           hop_length=hop, trainable=True, kernel_width=K, center=center)


def _stft_block(ctor, K, F_, hop, trainable):
    """dense_domain.row_geometry's test: the block-partial layout for a forward-only periodic-Hann DFT basis."""
    from nnaudio_b200 import _C
    hann = (ctor.get("window", "hann") == "hann" and ctor.get("win_length", K) in (None, K)
            and ctor.get("freq_scale", "no") == "no" and F_ == K // 2 + 1)
    return hann and not trainable and bool(_C.block_layout_ok(K, hop))


def _framed_frames(L, K, hop, center):
    return (L + 2 * (K // 2 if center else 0) - K) // hop + 1


def _dx_dw(b, L, K, F_, hop, center, dw):
    import ola_domain as od
    T = _framed_frames(L, K, hop, center)
    f = od.ola_exec_flops(*od.dx_operands(b, T, K, F_))
    return f + (od.ola_exec_flops(*od.dw_operands(b, T, K, F_)) if dw else 0.0)


def _cq_call(model, key, mod, b, L, path):
    import cqt1992_domain as cd
    p = cd.plan(mod, b, L, path)
    model[key][("cq", p["route"])] = model[key].get(("cq", p["route"]), 0) + 1
    model[key + "_flops"] += p["flops"]
    return p["route"]


def launch_model(name, mod, B=None):
    """{"fwd": {route: count}, "fwd_flops", "bwd": {route: count}, "bwd_flops"} of row ``name`` through ``mod``."""
    import dense_domain as dd
    import ola_domain as od
    from nnaudio_b200.features.cqt import _decimated_len

    r = ROWS[name]
    B = r["B"] if B is None else B
    path = r["env"] or "auto"
    m = dict(fwd={}, fwd_flops=0.0, bwd={}, bwd_flops=0.0)
    fam = r["family"]
    for b in _chunks(B):
        if fam in ("stft", "mel", "mfcc"):
            st = {"stft": mod, "mel": getattr(mod, "stft", None), "mfcc": None}[fam]
            st = st if st is not None else mod.melspec_layer.stft
            K, F_, hop = st.n_fft, int(st.wcos.shape[0]), st.stride
            ctor = r["ctor"] if fam == "stft" else dict(n_fft=K)
            p = dd.plan(K, F_, hop, b, r["L"], st.center, _stft_block(ctor, K, F_, hop, st.trainable), path)
            for route in p["routes"]:
                m["fwd"][("stft", route)] = m["fwd"].get(("stft", route), 0) + 1
            m["fwd_flops"] += p["flops"]
            m["bwd_flops"] += _dx_dw(b, r["L"], K, F_, hop, st.center, st.trainable)
        elif fam == "cqt":
            _cq_call(m, "fwd", mod, b, r["L"], path)
            m["bwd_flops"] += _dx_dw(b, r["L"], mod.kernel_width, int(mod.cqt_kernels_real.shape[0]),
                                     mod.hop_length, mod.center, mod.trainable)
        elif fam == "v1":
            F_, K = int(mod.cqt_kernels_real.shape[0]), mod.kernel_width
            trainable = any(p.requires_grad for p in mod.parameters())
            _cq_call(m, "fwd", _bank_shim(F_, K, mod.hop_length, mod.center), b, r["L"], path)
            m["bwd_flops"] += _dx_dw(b, r["L"], K, F_, mod.hop_length, mod.center, trainable)
        elif fam == "pyramid":
            trainable = any(p.requires_grad for p in mod.parameters())
            L = r["L"]
            if mod.earlydownsample:
                L = _decimated_len(L, int(mod.downsample_factor))
            hop = mod.hop_length
            if "cqt_kernels_real" in dict(mod.named_buffers()) | dict(mod.named_parameters()):
                widths = [int(mod.cqt_kernels_real.shape[-1])] * mod.n_octaves
                F_ = int(mod.cqt_kernels_real.shape[0])
            else:
                widths = [int(getattr(mod, f"cqt_kernels_real_{i}").shape[-1]) for i in range(mod.n_octaves)]
                F_ = int(mod.cqt_kernels_real_0.shape[0])
            if r["cls"] == "CQT2010":   # the folded bank: n_fft taps
                widths = [mod.n_fft] * mod.n_octaves
            for i, K in enumerate(widths):
                if i > 0:
                    L, hop = _decimated_len(L, 2), hop // 2
                _cq_call(m, "fwd", _bank_shim(F_, K, hop, True), b, L, path)
                m["bwd_flops"] += _dx_dw(b, L, K, F_, hop, True, trainable)
        else:  # inverse STFT: the overlap-add GEMM forward; backward one CQT1992v2 contraction of the adjoint bank
            n_fft, hop, T = mod.n_fft, mod.stride, r["T"]
            f_in = n_fft // 2 + 1 if r["onesided"] else n_fft
            m["fwd_flops"] += od.ola_exec_flops(*od.istft_operands(b, T, n_fft, f_in))
            _cq_call(m, "bwd", _bank_shim(f_in, n_fft, hop, False), b, n_fft + hop * (T - 1), path)
    return m


def route_claims():
    """The forward route each row's edge names: {row: (family, route constant)}."""
    from nnaudio_b200 import _C
    return {
        "stft_block_complex": ("stft", _C.STFT_BLOCK), "stft_block_magnitude": ("stft", _C.STFT_BLOCK),
        "stft_block_phase": ("stft", _C.STFT_BLOCK), "stft_trainable": ("stft", _C.STFT_DENSE),
        "stft_16384_trainable": ("stft", _C.STFT_DENSE_SPLITK), "stft_simt": ("stft", _C.STFT_SIMT),
        "mel_power2": ("stft", _C.STFT_BLOCK), "mel_power1_trainable_stft": ("stft", _C.STFT_DENSE),
        "cqt_dense_complex": ("cq", _C.CQ1992_DENSE), "cqt_trainable_mag": ("cq", _C.CQ1992_DENSE),
        "cqt_long_grouped": ("cq", _C.CQ1992_TALL), "cqt_varn": ("cq", _C.CQ1992_VARN_SPLITK),
        "cqt_long_dense": ("cq", _C.CQ1992_DENSE_SPLITK), "cqt_long_trainable": ("cq", _C.CQ1992_DENSE_SPLITK),
        "cqt_simt": ("cq", _C.CQ1992_SIMT), "pyr_noearly_wrap": ("cq", _C.CQ1992_DENSE),
        "v1_stft_complex": ("cq", _C.CQ1992_DENSE), "cqt2010_cqt_complex": ("cq", _C.CQ1992_DENSE),
    }
