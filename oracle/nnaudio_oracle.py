"""CPU ORACLE — test infrastructure only.  NOT part of the product path.

A plain NumPy restatement of the reference nnAudio *forward* algorithms
(KinWaiCheuk/nnAudio v0.3.3, ``Installation/nnAudio``) for the hot path of
SURVEY.md §8(a).  Only ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` may import this
module, and only as the checker / the CPU arm — never from ``nnaudio_b200``.

Parity pin: every function below is checked in ``tests/test_oracle_golden.py``
against (i) the reference's own golden vectors
(``Installation/tests/ground-truths/*cqt*.npy``, replayed from
``tests/golden/ref_ground_truths.npz``) and (ii) outputs of the unmodified
reference imported in the build container (``tests/golden/make_golden.py`` ->
``tests/golden/ref_outputs.npz``) — this covers STFT, the inverse STFT, Mel,
MFCC, Gammatone, CQT1992v2, CQT2010v2, VQT, the first-generation
``cqt1992`` / ``cqt2010`` and ``cfp`` (fixtures: ``tests/golden/make_golden_cfp.py``).  ONE EXCEPTION, PARITY UNPINNED: ``griffin_lim`` — the
reference module does not execute under torch >= 2.0 (its ``torch.istft`` /
``torch.stft`` calls are rejected), so that function follows the source and the
documented semantics of the two torch calls without reference outputs to check.

All functions take the module's *buffers* (float32 arrays, exactly what
``state_dict()`` holds) plus scalar configuration, and compute in ``dtype``
(float64 for checking, float32 when timed as the CPU baseline).  The framing +
basis contraction the reference performs with ``conv1d(x, basis, stride=hop)``
is done here as strided frames times the basis matrix (BLAS), which is the same
arithmetic.
"""
from __future__ import annotations

import warnings

import numpy as np

__all__ = [
    "broadcast_dim",
    "pad_signal",
    "framed_contraction",
    "stft",
    "melspectrogram",
    "power_to_db",
    "dct_ortho_fft_route",
    "mfcc",
    "cqt1992v2",
    "downsample_by_n",
    "cqt_octave_complex",
    "cqt2010v2",
    "vqt",
    "istft",
    "cqt1992",
    "cqt2010",
    "griffin_lim",
    "torch_stft_restated",
    "torch_istft_restated",
    "cfp",
]


# --------------------------------------------------------------------------- #
# shared helpers
# --------------------------------------------------------------------------- #
def broadcast_dim(x: np.ndarray) -> np.ndarray:
    """utils.py:206-222 — (L)->(1,L), (B,L) pass, (B,1,L)->(B,L) (channel dim
    is squeezed here because every consumer has exactly one input channel)."""
    if x.ndim == 1:
        return x[None, :]
    if x.ndim == 2:
        return x
    if x.ndim == 3:
        return x[:, 0, :]
    raise ValueError("Only support input with shape = (batch, len) or shape = (len)")


def pad_signal(x: np.ndarray, pad: int, mode: str) -> np.ndarray:
    """nn.ReflectionPad1d(pad) / nn.ConstantPad1d(pad, 0) on the last axis
    (stft.py:278-289, cqt.py:740-746).  Reflect requires pad < L like torch."""
    if pad == 0:
        return x
    if mode == "reflect":
        if pad >= x.shape[-1]:
            raise RuntimeError("reflect padding must be smaller than the input length")
        return np.pad(x, ((0, 0), (pad, pad)), mode="reflect")
    if mode == "constant":
        return np.pad(x, ((0, 0), (pad, pad)), mode="constant")
    raise ValueError("unknown pad_mode %r" % (mode,))


def framed_contraction(xp: np.ndarray, basis: np.ndarray, hop: int, max_rows: int = 8192):
    """``conv1d(xp[:,None,:], basis[:,None,:], stride=hop)`` as frames x basis^T.

    xp (B, Lp), basis (N, K)  ->  (B, N, T) with T = (Lp-K)//hop + 1.  Frames of
    several clips are stacked into one GEMM of up to ``max_rows`` rows (what an
    im2col-style conv1d does), so BLAS can use every host core.
    """
    B, Lp = xp.shape
    N, K = basis.shape
    if Lp < K:
        raise RuntimeError("input shorter than the kernel")
    T = (Lp - K) // hop + 1
    out = np.empty((B, N, T), dtype=xp.dtype)
    bt = np.ascontiguousarray(basis.T)
    st = xp.strides[-1]
    if T > max_rows:  # long clips: chunk along time
        for b in range(B):
            frames = np.lib.stride_tricks.as_strided(
                xp[b], shape=(T, K), strides=(hop * st, st), writeable=False)
            for t0 in range(0, T, max_rows):
                t1 = min(T, t0 + max_rows)
                out[b, :, t0:t1] = (np.ascontiguousarray(frames[t0:t1]) @ bt).T
        return out
    nb = max(1, max_rows // T)
    block = np.empty((nb * T, K), dtype=xp.dtype)
    for b0 in range(0, B, nb):
        b1 = min(B, b0 + nb)
        for i, b in enumerate(range(b0, b1)):
            block[i * T:(i + 1) * T] = np.lib.stride_tricks.as_strided(
                xp[b], shape=(T, K), strides=(hop * st, st), writeable=False)
        res = block[: (b1 - b0) * T] @ bt
        out[b0:b1] = res.reshape(b1 - b0, T, N).transpose(0, 2, 1)
    return out


# --------------------------------------------------------------------------- #
# STFT family
# --------------------------------------------------------------------------- #
def stft(
    x,
    wsin,
    wcos,
    hop,
    center=True,
    pad_mode="reflect",
    output_format="Complex",
    trainable=False,
    freq_bins=None,
    dtype=np.float64,
):
    """STFT.forward (stft.py:256-316).

    wsin/wcos: (F, 1, n_fft) windowed bases.  Magnitude -> (B,F,T);
    Complex -> (B,F,T,2) = (real, -imag); Phase -> (B,F,T) =
    atan2(-imag + 0.0, real).
    """
    x = broadcast_dim(np.asarray(x)).astype(dtype)
    ws = np.asarray(wsin)[:, 0, :].astype(dtype)
    wc = np.asarray(wcos)[:, 0, :].astype(dtype)
    n_fft = ws.shape[-1]
    if center:
        if pad_mode == "reflect" and x.shape[-1] < n_fft // 2:
            raise AssertionError("Signal length shorter than reflect padding length (n_fft // 2).")
        x = pad_signal(x, n_fft // 2, pad_mode)
    both = framed_contraction(x, np.concatenate((wc, ws), 0), hop)  # one pass over the frames
    real, imag = both[:, : wc.shape[0]], both[:, wc.shape[0]:]
    if freq_bins is not None:
        real, imag = real[:, :freq_bins], imag[:, :freq_bins]
    if output_format == "Magnitude":
        spec = real ** 2 + imag ** 2
        return np.sqrt(spec + dtype(1e-8)) if trainable else np.sqrt(spec)
    if output_format == "Complex":
        return np.stack((real, -imag), -1)
    if output_format == "Phase":
        return np.arctan2(-imag + 0.0, real)
    raise ValueError("unknown output_format %r" % (output_format,))


def melspectrogram(x, wsin, wcos, fbank, hop, power=2.0, center=True, pad_mode="reflect",
                   trainable_stft=False, dtype=np.float64):
    """MelSpectrogram.forward / Gammatonegram.forward (mel.py:171-189,
    gammatone.py:171-189): ``fbank @ (|STFT| ** power)``; note the reference
    takes sqrt first and then raises to ``power``."""
    mag = stft(x, wsin, wcos, hop, center, pad_mode, "Magnitude", trainable_stft, None, dtype)
    spec = mag ** dtype(power)
    return np.matmul(np.asarray(fbank).astype(dtype), spec)


def power_to_db(S, amin=1e-10, ref=1.0, top_db=80.0):
    """MFCC._power_to_db (mel.py:263-279); the top_db floor is relative to the
    per-clip maximum over (mel, time)."""
    dt = S.dtype.type
    log_spec = dt(10.0) * np.log10(np.maximum(S, dt(amin)))
    log_spec = log_spec - dt(10.0) * np.log10(np.maximum(dt(amin), dt(abs(ref))))
    if top_db is not None:
        if top_db < 0:
            raise ValueError("top_db must be non-negative")
        peak = log_spec.reshape(log_spec.shape[0], -1).max(1)[:, None, None]
        log_spec = np.maximum(log_spec, peak - dt(top_db))
    return log_spec


def dct_ortho_fft_route(x):
    """MFCC._dct(norm='ortho') (mel.py:281-307): DCT-II along axis 1 of
    (B, N, T) via the even/odd re-ordering + FFT + twiddle route."""
    v_in = np.transpose(x, (0, 2, 1))
    N = v_in.shape[-1]
    v = np.concatenate([v_in[:, :, ::2], v_in[:, :, 1::2][:, :, ::-1]], axis=2)
    Vc = np.fft.fft(v, axis=-1)
    k = -np.arange(N, dtype=x.dtype)[None, :] * np.pi / (2 * N)
    V = Vc.real * np.cos(k) - Vc.imag * np.sin(k)
    V[:, :, 0] /= np.sqrt(N) * 2
    V[:, :, 1:] /= np.sqrt(N / 2) * 2
    V = 2 * V
    return np.transpose(V, (0, 2, 1)).astype(x.dtype)


def mfcc(x, wsin, wcos, mel_basis, hop, n_mfcc=20, power=2.0, amin=1e-10, ref=1.0,
         top_db=80.0, center=True, pad_mode="reflect", dtype=np.float64):
    """MFCC.forward (mel.py:309-326)."""
    S = melspectrogram(x, wsin, wcos, mel_basis, hop, power, center, pad_mode, False, dtype)
    db = power_to_db(S, amin, ref, top_db)
    return dct_ortho_fft_route(db)[:, :n_mfcc, :]


# --------------------------------------------------------------------------- #
# CQT family
# --------------------------------------------------------------------------- #
def _cqt_normalise(real, imag, lenghts, normalization_type, dtype):
    if normalization_type == "librosa":
        s = np.sqrt(np.asarray(lenghts).astype(np.float32)).astype(dtype).reshape(-1, 1)
        return real * s, imag * s
    if normalization_type == "convolutional":
        return real, imag
    if normalization_type == "wrap":
        return real * 2, imag * 2
    raise ValueError(
        "The normalization_type %r is not part of our current options." % normalization_type
    )


def _cqt_format(real, imag, output_format, trainable, dtype):
    if output_format == "Magnitude":
        p = real ** 2 + imag ** 2
        return np.sqrt(p + dtype(1e-8)) if trainable else np.sqrt(p)
    if output_format == "Complex":
        return np.stack((real, imag), -1)
    if output_format == "Phase":
        ang = np.arctan2(imag, real)
        return np.stack((np.cos(ang), np.sin(ang)), -1)
    raise ValueError("unknown output_format %r" % (output_format,))


def cqt1992v2(x, kernels_real, kernels_imag, lenghts, hop, center=True, pad_mode="reflect",
              output_format="Magnitude", normalization_type="librosa", trainable=False,
              dtype=np.float64):
    """CQT1992v2.forward (cqt.py:712-780): real = conv(x, Kr), imag = -conv(x, Ki),
    scale, then Magnitude / Complex (re, im) / Phase (cos, sin)."""
    x = broadcast_dim(np.asarray(x)).astype(dtype)
    kr = np.asarray(kernels_real)[:, 0, :].astype(dtype)
    ki = np.asarray(kernels_imag)[:, 0, :].astype(dtype)
    if center:
        x = pad_signal(x, kr.shape[-1] // 2, pad_mode)
    both = framed_contraction(x, np.concatenate((kr, ki), 0), hop, max_rows=512)
    real, imag = both[:, : kr.shape[0]], -both[:, kr.shape[0]:]
    real, imag = _cqt_normalise(real, imag, lenghts, normalization_type, dtype)
    return _cqt_format(real, imag, output_format, trainable, dtype)


def downsample_by_n(x, fir, n):
    """utils.py:73-100: conv1d(x, fir, stride=n, padding=(len(fir)-1)//2), i.e.
    zero padding of 127 on both sides for the 256-tap filters."""
    fir = np.asarray(fir).reshape(1, -1).astype(x.dtype)
    p = (fir.shape[-1] - 1) // 2
    xp = np.pad(x, ((0, 0), (p, p)), mode="constant")
    return framed_contraction(xp, fir, n)[:, 0, :]


def cqt_octave_complex(x, kr, ki, hop, pad, pad_mode):
    """utils.py:498-521 get_cqt_complex: try the module's padding, on failure
    (reflect pad >= length) warn and zero-pad by kernel_width//2."""
    try:
        xp = pad_signal(x, pad, pad_mode)
    except RuntimeError:
        warnings.warn(
            "padding with reflection mode might not be the best choice, try using constant padding",
            UserWarning,
        )
        xp = np.pad(x, ((0, 0), (kr.shape[-1] // 2,) * 2), mode="constant")
    both = framed_contraction(xp, np.concatenate((kr, ki), 0), hop)
    return both[:, : kr.shape[0]], -both[:, kr.shape[0]:]


def _pyramid(x, banks, hop, n_bins, lowpass, pads, pad_mode, early_fir, early_factor, dtype,
             octave_fn=None):
    """Shared octave pyramid of CQT2010v2 (one bank reused) and VQT (one bank
    per octave): top octave on x, then repeatedly halve with the 256-tap FIR
    and halve the hop; octaves are stacked low -> high and the lowest surplus
    bins are dropped (cqt.py:1086-1105, vqt.py:158-189)."""
    x = broadcast_dim(np.asarray(x)).astype(dtype)
    if early_fir is not None:
        x = downsample_by_n(x, early_fir, int(early_factor))
    reals, imags = [], []
    x_down = x
    for i, (kr, ki) in enumerate(banks):
        if i > 0:
            x_down = downsample_by_n(x_down, lowpass, 2)
            hop = hop // 2
        if octave_fn is not None:
            r, im = octave_fn(x_down, kr, ki, hop, pads[i], pad_mode)
        else:
            kr2 = np.asarray(kr)[:, 0, :].astype(dtype)
            ki2 = np.asarray(ki)[:, 0, :].astype(dtype)
            r, im = cqt_octave_complex(x_down, kr2, ki2, hop, pads[i], pad_mode)
        reals.insert(0, r)
        imags.insert(0, im)
    real = np.concatenate(reals, axis=1)[:, -n_bins:, :]
    imag = np.concatenate(imags, axis=1)[:, -n_bins:, :]
    return real, imag


def cqt2010v2(x, kernels_real, kernels_imag, lowpass_filter, lenghts, hop, n_bins, n_octaves,
              pad_mode="reflect", early_downsample_filter=None, downsample_factor=1,
              output_format="Magnitude", normalization_type="librosa", trainable=False,
              dtype=np.float64):
    """CQT2010v2.forward (cqt.py:1070-1139).  ``hop`` is the module's
    post-early-downsample hop_length."""
    width = np.asarray(kernels_real).shape[-1]
    banks = [(kernels_real, kernels_imag)] * n_octaves
    real, imag = _pyramid(x, banks, hop, n_bins, lowpass_filter, [width // 2] * n_octaves,
                          pad_mode, early_downsample_filter, downsample_factor, dtype)
    real, imag = real * downsample_factor, imag * downsample_factor
    if normalization_type == "librosa":
        s = np.sqrt(np.asarray(lenghts).astype(np.float32)).astype(dtype).reshape(-1, 1)
        real, imag = real * s, imag * s
    elif normalization_type == "convolutional":
        pass
    elif normalization_type == "wrap":
        real, imag = real * 2, imag * 2
    else:
        raise ValueError(
            "The normalization_type %r is not part of our current options." % normalization_type
        )
    return _cqt_format(real, imag, output_format, trainable, dtype)


def vqt(x, banks, lowpass_filter, lenghts, hop, n_bins, pad_mode="reflect",
        early_downsample_filter=None, downsample_factor=1, output_format="Magnitude",
        normalization_type="librosa", trainable=False, dtype=np.float64):
    """VQT.forward (vqt.py:143-215): ``banks`` = [(real_i, imag_i)] for octave
    i = 0 (top) .. n_octaves-1; each octave pads by its own bank width // 2."""
    pads = [np.asarray(kr).shape[-1] // 2 for kr, _ in banks]
    real, imag = _pyramid(x, banks, hop, n_bins, lowpass_filter, pads, pad_mode,
                          early_downsample_filter, downsample_factor, dtype)
    real, imag = real * downsample_factor, imag * downsample_factor
    if normalization_type == "librosa":
        s = np.sqrt(np.asarray(lenghts).astype(np.float32)).astype(dtype).reshape(-1, 1)
        real, imag = real * s, imag * s
    elif normalization_type == "convolutional":
        pass
    elif normalization_type == "wrap":
        real, imag = real * 2, imag * 2
    else:
        raise ValueError(
            "The normalization_type %r is not part of our current options." % normalization_type
        )
    return _cqt_format(real, imag, output_format, trainable, dtype)


# --------------------------------------------------------------------------- #
# first-generation, frequency-domain CQTs  (SURVEY.md §8f next #3)
# --------------------------------------------------------------------------- #
def _spectral_cqt(xp, spec_real, spec_imag, wcos, wsin, hop, dtype):
    """The two stages of cqt.py:211-219 / utils.py:551-557 on an already padded signal:
    un-windowed DFT rows (``conv1d`` with wcos / wsin), then ``complex_mul`` (utils.py:175-203)
    with the spectral CQT kernels.  Returns (CQT_real, CQT_imag), each (B, n_bins, T)."""
    wc = np.asarray(wcos)[:, 0, :].astype(dtype)
    ws = np.asarray(wsin)[:, 0, :].astype(dtype)
    both = framed_contraction(xp, np.concatenate((wc, ws), 0), hop, max_rows=512)
    f_re, f_im = both[:, : wc.shape[0]], both[:, wc.shape[0]:]
    kr = np.asarray(spec_real).astype(dtype)
    ki = np.asarray(spec_imag).astype(dtype)
    real = np.einsum("nf,bft->bnt", kr, f_re) - np.einsum("nf,bft->bnt", ki, f_im)
    imag = np.einsum("nf,bft->bnt", kr, f_im) + np.einsum("nf,bft->bnt", ki, f_re)
    return real, imag


def cqt1992(x, spec_real, spec_imag, wcos, wsin, lenghts, hop, center=True, pad_mode="reflect",
            output_format="Magnitude", normalization_type="librosa", dtype=np.float64):
    """CQT1992.forward (cqt.py:189-251).  The stacked result is (real, -imag) (cqt.py:222) but
    'Phase' takes atan2 of the un-negated imaginary part (cqt.py:246-249)."""
    x = broadcast_dim(np.asarray(x)).astype(dtype)
    width = np.asarray(wcos).shape[-1]
    if center:
        x = pad_signal(x, width // 2, pad_mode)
    real, imag = _spectral_cqt(x, spec_real, spec_imag, wcos, wsin, hop, dtype)
    if normalization_type == "librosa":
        s = (np.sqrt(np.asarray(lenghts).astype(np.float32)).astype(dtype) / width).reshape(-1, 1)
    elif normalization_type == "convolutional":
        s = dtype(1.0)
    elif normalization_type == "wrap":
        s = dtype(2.0 / width)
    else:
        raise ValueError(
            "The normalization_type %r is not part of our current options." % normalization_type
        )
    if output_format == "Phase":  # normalisation is positive: it does not move the angle
        ang = np.arctan2(imag, real)
        return np.stack((np.cos(ang), np.sin(ang)), -1)
    return _cqt_format(real * s, -imag * s, output_format, False, dtype)


def cqt2010(x, spec_real, spec_imag, wcos, wsin, lowpass_filter, lenghts, hop, n_bins, n_octaves,
            pad_mode="reflect", early_downsample_filter=None, downsample_factor=1,
            output_format="Magnitude", normalization_type="librosa", dtype=np.float64):
    """CQT2010.forward (cqt.py:475-553): the /2 pyramid with ``get_cqt_complex2``
    (utils.py:524-559) per octave — imaginary part NOT negated, no downsample_factor gain,
    'librosa' / 'wrap' divide by n_fft."""
    n_fft = np.asarray(wcos).shape[-1]

    def octave(x_down, kr, ki, hop_i, pad, mode):
        try:
            xp = pad_signal(x_down, pad, mode)
        except RuntimeError:
            warnings.warn(
                "padding with reflection mode might not be the best choice, try using constant padding",
                UserWarning,
            )
            xp = np.pad(x_down, ((0, 0), (pad, pad)), mode="constant")
        return _spectral_cqt(xp, kr, ki, wcos, wsin, hop_i, dtype)

    banks = [(spec_real, spec_imag)] * n_octaves
    real, imag = _pyramid(x, banks, hop, n_bins, lowpass_filter, [n_fft // 2] * n_octaves,
                          pad_mode, early_downsample_filter, downsample_factor, dtype,
                          octave_fn=octave)
    if normalization_type == "librosa":
        s = (np.sqrt(np.asarray(lenghts).astype(np.float32)).astype(dtype) / n_fft).reshape(-1, 1)
        real, imag = real * s, imag * s
    elif normalization_type == "wrap":
        real, imag = real * (2.0 / n_fft), imag * (2.0 / n_fft)
    elif normalization_type != "convolutional":
        raise ValueError(
            "The normalization_type %r is not part of our current options." % normalization_type
        )
    return _cqt_format(real, imag, output_format, False, dtype)


# --------------------------------------------------------------------------- #
# inverse STFT  (SURVEY.md §8f next #2)
# --------------------------------------------------------------------------- #
def istft(X, kernel_cos, kernel_sin, window_mask, hop, center=True, onesided=True, length=None,
          dtype=np.float64):
    """STFTBase.inverse_stft (stft.py:15-63).

    X (B, F, T, 2); kernel_cos / kernel_sin: the (n_fft, 1, n_fft[, 1]) inverse kernels
    (``kernel_cos_inv`` of STFT(iSTFT=True) or ``kernel_cos`` of the iSTFT module);
    window_mask: (1, n_fft, 1).  Steps: mirror the one-sided spectrum
    (utils.py:63-70), contract with the kernels over the frequency axis, window and
    divide by n_fft, overlap-add with stride ``hop`` (utils.py:52-56), divide by the
    window sum-square where it exceeds 1e-10 (utils.py:43-49), strip the centre padding.
    """
    X = np.asarray(X).astype(dtype)
    kc = np.asarray(kernel_cos).astype(dtype).reshape(kernel_cos.shape[0], -1)
    ks = np.asarray(kernel_sin).astype(dtype).reshape(kernel_sin.shape[0], -1)
    win = np.asarray(window_mask).astype(dtype).reshape(-1)
    n_fft = kc.shape[0]
    if onesided:
        upper = X[:, 1:-1][:, ::-1].copy()
        upper[..., 1] = -upper[..., 1]
        X = np.concatenate((X, upper), axis=1)
    Xr, Xi = X[..., 0], X[..., 1]                      # (B, n_fft, T)
    real = np.einsum("of,bft->bot", kc, Xr) - np.einsum("of,bft->bot", ks, Xi)
    real = real * win[None, :, None] / n_fft
    B, _, T = real.shape
    out_len = n_fft + hop * (T - 1)
    y = np.zeros((B, out_len), dtype=dtype)
    wss = np.zeros(out_len, dtype=dtype)
    for t in range(T):
        y[:, t * hop: t * hop + n_fft] += real[:, :, t]
        wss[t * hop: t * hop + n_fft] += win ** 2
    nz = wss > 1e-10
    y[:, nz] = y[:, nz] / wss[nz]
    pad = n_fft // 2
    if length is None:
        return y[:, pad:-pad] if center else y
    return y[:, pad: pad + length] if center else y[:, :length]


# --------------------------------------------------------------------------- #
# Griffin-Lim  (SURVEY.md §8f next #4)
# --------------------------------------------------------------------------- #
def _padded_window(window, win_length, n_fft, dtype):
    from scipy.signal import get_window

    w = get_window(window, int(win_length), fftbins=True).astype(np.float32).astype(dtype)
    lpad = (n_fft - win_length) // 2
    return np.pad(w, (lpad, n_fft - win_length - lpad))


def torch_istft_restated(X, n_fft, hop, w, center=True):
    """``torch.istft(X, n_fft, hop, win_length, window, center)`` for one-sided complex
    ``X (B, n_fft//2+1, T)`` and a window already padded to n_fft: inverse real DFT, window,
    overlap-add, divide by the overlap-added squared window, trim n_fft//2 when centred.
    Pinned against torch itself in tests/test_griffin_lim.py."""
    B, _, T = X.shape
    frames = np.fft.irfft(X, n=n_fft, axis=1) * w[None, :, None]
    out_len = n_fft + hop * (T - 1)
    y = np.zeros((B, out_len), dtype=frames.dtype)
    wss = np.zeros(out_len, dtype=frames.dtype)
    for t in range(T):
        y[:, t * hop: t * hop + n_fft] += frames[:, :, t]
        wss[t * hop: t * hop + n_fft] += w ** 2
    if center:
        y, wss = y[:, n_fft // 2: out_len - n_fft // 2], wss[n_fft // 2: out_len - n_fft // 2]
    return y / wss


def torch_stft_restated(y, n_fft, hop, w, pad_mode="reflect"):
    """``torch.stft(y, n_fft, hop, win_length, window, center=True, pad_mode, onesided=True)``
    as complex ``(B, n_fft//2+1, T)``.  Pinned against torch itself in tests/test_griffin_lim.py."""
    yp = pad_signal(y, n_fft // 2, pad_mode)
    n_frames = (yp.shape[-1] - n_fft) // hop + 1
    idx = np.arange(n_fft)[:, None] + hop * np.arange(n_frames)[None, :]
    return np.fft.rfft(yp[:, idx] * w[None, :, None], axis=1)


def griffin_lim(S, rand_phase, n_fft, n_iter=32, hop=None, win_length=None, window="hann",
                center=True, pad_mode="reflect", momentum=0.99, dtype=np.float64):
    """Griffin_Lim.forward (griffin_lim.py:89-148) with the initial ``randn`` phase passed in.

    PARITY UNPINNED for the loop as a whole: the reference module does not execute under
    torch >= 2.0 (its real-view ``torch.istft`` / ``torch.stft`` calls are rejected).  The two
    library calls it makes are restated above and pinned against torch; the glue below (initial
    phase, momentum rule griffin_lim.py:129-137, final inverse) follows the source.  In the loop
    ``torch.stft`` runs with its default ``center=True`` (griffin_lim.py:120-127); only the
    inverse honours ``center``."""
    S = np.asarray(S).astype(dtype)
    win_length = n_fft if win_length is None else win_length
    hop = n_fft // 4 if hop is None else hop
    w = _padded_window(window, win_length, n_fft, dtype)

    ph = np.asarray(rand_phase).astype(np.float32).astype(dtype)
    angles = np.cos(2 * np.pi * ph) + 1j * np.sin(2 * np.pi * ph)
    rebuilt = np.zeros_like(angles)
    for _ in range(n_iter):
        tprev = rebuilt
        inverse = torch_istft_restated(S * angles, n_fft, hop, w, center)
        rebuilt = torch_stft_restated(inverse, n_fft, hop, w, pad_mode)
        angles = rebuilt - (momentum / (1 + momentum)) * tprev
        angles = angles / (np.abs(angles) + 1e-16)
    return torch_istft_restated(S * angles, n_fft, hop, w, center)


# --------------------------------------------------------------------------- #
# Combined frequency / periodicity (features/cfp.py)
# --------------------------------------------------------------------------- #
def cfp(x, h, freq2logfreq, quef2logfreq, N, hop, g, tc_idx, fc_idx, high_freq, high_quef,
        drop_edge_frames=False, dtype=np.float64):
    """``Combined_Frequency_Periodicity.forward`` (cfp.py:137-180, ``drop_edge_frames=True``) and
    ``CFP.forward`` (cfp.py:375-418): returns ``(Z, tfrL0, tfrLF, tfrLQ)``, each (B, bands, T).

    Follows the source step by step with full length-N FFTs: ``torch.stft(n_fft=N, win_length=len(h),
    center=True, pad_mode="constant", onesided=False)`` = N//2 zeros either side, the window zero-padded
    to N with ``(N - len(h)) // 2`` zeros in front, frames every ``hop``; magnitude / ``|h|``;
    ``_CFP`` (cfp.py:119-135) with ``nonlinear_func`` (cfp.py:182-193, including ``X[..., -0:] = 0``
    zeroing everything when the cut-off index is 0); the crops and the two matmuls."""
    x = np.asarray(x, dtype=dtype)
    if x.ndim != 2:
        raise IndexError("cfp: the reference's transpose(1, 2) needs a (batch, len) input")
    h = np.asarray(h, dtype=dtype)
    W = h.shape[0]
    B, L = x.shape
    xp = np.pad(x, ((0, 0), (N // 2, N // 2)))
    win = np.zeros(N, dtype=dtype)
    left = (N - W) // 2
    win[left:left + W] = h
    T = 1 + (L + 2 * (N // 2) - N) // hop  # torch.stft's count: one fewer than L // hop + 1 for odd N, L % hop == 0
    idx = np.arange(T)[:, None] * hop + np.arange(N)[None, :]
    spec_c = np.fft.fft(xp[:, idx] * win, axis=-1)                   # (B, T, N)
    tfr0 = (np.abs(spec_c) / np.linalg.norm(h)).astype(dtype)
    if drop_edge_frames:
        tfr0 = tfr0[:, 1:-1]

    def nonlinear(X, gg, cutoff):
        cutoff = int(cutoff)
        X = np.maximum(X, 0)
        if gg != 0:
            X = X.copy()
            X[:, :, :cutoff] = 0
            X[:, :, X.shape[2] - cutoff if cutoff else 0:] = 0
            return X ** gg
        X = np.log(X + 1e-8)
        X[:, :, :cutoff] = 0
        X[:, :, X.shape[2] - cutoff if cutoff else 0:] = 0
        return X

    spec = np.maximum(tfr0, 0) ** g[0]
    ceps = None
    for gc in range(1, int(np.size(g))):
        if gc % 2 == 1:
            ceps = nonlinear(np.fft.fft(spec, axis=-1).real.astype(dtype) / np.sqrt(N), g[gc], tc_idx)
        else:
            spec = nonlinear(np.fft.fft(ceps, axis=-1).real.astype(dtype) / np.sqrt(N), g[gc], fc_idx)
    if ceps is None:
        raise UnboundLocalError("cfp: fewer than two layers leave `ceps` unassigned (cfp.py:135)")
    half = int(round(N / 2))
    tfr0 = tfr0[:, :, :half][:, :, :high_freq]
    tfr = spec[:, :, :half][:, :, :high_freq]
    ceps = ceps[:, :, :half][:, :, :high_quef]
    f2l = np.asarray(freq2logfreq, dtype=dtype)
    q2l = np.asarray(quef2logfreq, dtype=dtype)
    tfrL0 = f2l @ tfr0.transpose(0, 2, 1)
    tfrLF = f2l @ tfr.transpose(0, 2, 1)
    tfrLQ = q2l @ ceps.transpose(0, 2, 1)
    return tfrLF * tfrLQ, tfrL0, tfrLF, tfrLQ
