"""Float64 references and launch model of the overlap-add GEMM (the FMT_OLA route of csrc/tc_kernels.cu) and of the
FIR decimation adjoint, shared by tests/test_ola_domain_host.py (CPU) and tests/test_zz_gpu_ola_domain.py (-m gpu).

One tensor-core GEMM serves three entry points: the input gradient of every framed transform
(``nnab_framed_backward_input``), the gradient of trainable bases (``nnab_framed_backward_weight``) and the inverse
STFT (``nnab_istft_forward``).  The references below are those operations written out for the forward exactly as the
library defines it, Y = (w_re . x_pad, -w_im . x_pad) per frame; ``ola_exec_flops`` restates the MMA flops the launch
adds, so that a test reading the counter proves the GEMM ran at the shape the model says.

The shape matrices name the edge each row is there for."""
import numpy as np
import torch

MAX_WIDTH = 32768  # 128 N tiles of 256 output samples


# ------------------------------------------------------------------------------------------------ framing ----
def _pad(x, pad, pad_mode):
    if pad == 0:
        return x
    return np.pad(x, ((0, 0), (pad, pad)), mode="reflect" if pad_mode == "reflect" else "constant")


def frames_of(L, K, hop, center):
    pad = K // 2 if center else 0
    return (L + 2 * pad - K) // hop + 1


def frame_matrix(x, K, hop, center, pad_mode):
    """(B, T, K) float64 frames of the padded clips."""
    x = np.atleast_2d(np.asarray(x, dtype=np.float64))
    xp = _pad(x, K // 2 if center else 0, pad_mode)
    T = (xp.shape[-1] - K) // hop + 1
    idx = np.arange(K)[None, :] + hop * np.arange(T)[:, None]
    return xp[:, idx]


def hann_dft_bases(n_fft):
    """The STFT module's (wcos, wsin) for freq_scale='no': (n_fft // 2 + 1, n_fft) periodic-Hann DFT rows."""
    n = np.arange(n_fft)
    k = np.arange(n_fft // 2 + 1)
    ang = 2.0 * np.pi * ((k[:, None] * n[None, :]) % n_fft) / n_fft
    win = 0.5 - 0.5 * np.cos(2.0 * np.pi * n / n_fft)
    return np.cos(ang) * win, np.sin(ang) * win


def frame_grad(g, w_re, w_im):
    """(B, F, T, 2) gradient of Y -> (B, T, K) gradient of the frames: g_re . w_re - g_im . w_im.
    ``w_re = w_im = None``: the periodic-Hann DFT bases of n_fft = 2 (F - 1), by a float64 inverse FFT."""
    g = np.asarray(g, dtype=np.float64)
    if w_re is None:
        F = g.shape[1]
        n_fft = 2 * (F - 1)
        Z = g[..., 0] + 1j * g[..., 1]                        # (B, F, T)
        # sum_f Z[f] e^{+2 pi i f n / N} = N ifft(Z zero-padded to N)
        s = np.fft.ifft(Z, n=n_fft, axis=1).real * n_fft      # (B, N, T)
        win = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(n_fft) / n_fft)
        return (s * win[None, :, None]).transpose(0, 2, 1)
    w_re = np.asarray(w_re, dtype=np.float64)
    w_im = np.asarray(w_im, dtype=np.float64)
    return np.einsum("bft,fk->btk", g[..., 0], w_re) - np.einsum("bft,fk->btk", g[..., 1], w_im)


def overlap_add_adjoint(fg, K, hop, center, pad_mode, L):
    """(B, T, K) frame gradients -> (B, L): overlap-add onto the padded clip, then the padding adjoint (the mirror
    margins of reflect padding fold back onto samples 1..pad and L-1-pad..L-2)."""
    B, T, _ = fg.shape
    pad = K // 2 if center else 0
    gp = np.zeros((B, L + 2 * pad))
    for t in range(T):
        gp[:, t * hop:t * hop + K] += fg[:, t]
    dx = gp[:, pad:pad + L].copy()
    if pad and pad_mode == "reflect":
        for i in range(pad):                # xp[i] = x[pad - i]
            dx[:, pad - i] += gp[:, i]
        for m in range(pad):                # xp[pad + L + m] = x[L - 2 - m]
            dx[:, L - 2 - m] += gp[:, pad + L + m]
    return dx


def ref_backward_input(g, w_re, w_im, K, hop, center, pad_mode, L):
    """d loss / d x (B, L) for the upstream gradient g (B, F, T, 2) of Y = (w_re . x_pad, -w_im . x_pad)."""
    return overlap_add_adjoint(frame_grad(g, w_re, w_im), K, hop, center, pad_mode, L)


def read_mask(K, hop, center, pad_mode, L, T):
    """(L,) bool: the samples some frame reads.  The input gradient is exactly zero everywhere else."""
    ones = np.ones((1, T, K))
    return overlap_add_adjoint(ones, K, hop, center, pad_mode, L)[0] > 0


def ref_backward_weight(g, x, K, hop, center, pad_mode):
    """(d loss / d w_re, d loss / d w_im), each (F, K), for the upstream gradient g (B, F, T, 2)."""
    g = np.asarray(g, dtype=np.float64)
    fr = frame_matrix(x, K, hop, center, pad_mode)            # (B, T, K)
    B, F, T, _ = g.shape
    fr = fr.reshape(B * T, K)
    g_re = g[..., 0].transpose(1, 0, 2).reshape(F, B * T)
    g_im = g[..., 1].transpose(1, 0, 2).reshape(F, B * T)
    return g_re @ fr, -(g_im @ fr)


# ---------------------------------------------------------------------------------------------- inverse ----
def inverse_frames(X, win, onesided):
    """Windowed inverse-DFT frames (B, n_fft, T) of a spectrogram X (B, f_in, T, 2), divided by n_fft: what the
    reference computes with its (un-windowed) DFT kernels, by a float64 inverse FFT."""
    X = np.asarray(X, dtype=np.float64)
    win = np.asarray(win, dtype=np.float64).reshape(-1)
    n_fft = win.size
    Z = X[..., 0] + 1j * X[..., 1]
    if onesided:
        Z = np.concatenate((Z, np.conj(Z[:, 1:-1][:, ::-1])), axis=1)
    # real part of sum_f Z[f] e^{+2 pi i f n / N} (kernel_cos . Xr - kernel_sin . Xi), / N
    s = np.fft.ifft(Z, n=n_fft, axis=1).real
    return s * win[None, :, None]


def istft_wss(win, hop, T, center, length):
    """Window sum-square of the output samples (the overlap-add of win ** 2, sliced like the output)."""
    win = np.asarray(win, dtype=np.float64).reshape(-1)
    n_fft = win.size
    wss = np.zeros(n_fft + hop * (T - 1))
    for t in range(T):
        wss[t * hop:t * hop + n_fft] += win ** 2
    return _slice(wss[None], n_fft, center, length)[0]


def _slice(y, n_fft, center, length):
    pad = n_fft // 2
    if length is None:
        return y[:, pad:y.shape[1] - pad] if center else y
    return y[:, pad:pad + length] if center else y[:, :length]


def ref_istft(X, win, hop, center, onesided, length):
    """(y, y_undivided): the inverse STFT of the DFT kernels (oracle.istft's steps, FFT contraction) and the
    overlap-added frames before the window sum-square division, both sliced like the output."""
    fr = inverse_frames(X, win, onesided)
    B, n_fft, T = fr.shape
    ola = np.zeros((B, n_fft + hop * (T - 1)))
    for t in range(T):
        ola[:, t * hop:t * hop + n_fft] += fr[:, :, t]
    wss = istft_wss(win, hop, T, False, None)
    y = ola.copy()
    nz = wss > 1e-10
    y[:, nz] /= wss[nz]
    return _slice(y, n_fft, center, length), _slice(ola, n_fft, center, length)


# ------------------------------------------------------------------------------------------ FIR adjoint ----
def ref_fir_adjoint(g, fir, factor, L):
    """d loss / d x (B, L) of y = conv1d(x, fir, stride=factor, padding=(taps-1)//2), float64 autograd."""
    g = torch.as_tensor(np.asarray(g, dtype=np.float64))
    w = torch.as_tensor(np.asarray(fir, dtype=np.float64)).reshape(1, 1, -1)
    x = torch.zeros((g.shape[0], L), dtype=torch.float64, requires_grad=True)
    y = torch.nn.functional.conv1d(x[:, None, :], w, stride=factor, padding=(w.shape[-1] - 1) // 2)[:, 0]
    (dx,) = torch.autograd.grad(y, x, g)
    return dx.numpy()


def fir_out_len(L, taps, factor):
    return (L + 2 * ((taps - 1) // 2) - taps) // factor + 1


# -------------------------------------------------------------------------------------------- launch model ----
def round_up(v, m):
    return -(-v // m) * m


def istft_bn(F_out):
    """tc_istft_bn: N tile width of the overlap-add GEMM."""
    return 256 if F_out >= 256 else max(32, round_up(F_out, 16))


def ola_exec_flops(M, F_out, K_gemm):
    """MMA flops launch_framed_tc adds for one overlap-add GEMM: three bf16 split terms x 2 x M padded to the
    128-row tile x F_out padded to the N tile x K_gemm padded to 64."""
    bn = istft_bn(F_out)
    return 6 * round_up(M, 128) * round_up(F_out, bn) * round_up(K_gemm, 64)


def dx_operands(B, T, K, F):
    """(M, F_out, K_gemm) of nnab_framed_backward_input."""
    return B * T, K, round_up(2 * F, 64)


def istft_operands(B, T, n_fft, f_in):
    return B * T, n_fft, round_up(2 * f_in, 64)


def dw_gpad(B, T):
    return round_up(B * T, 64)


def dw_operands(B, T, K, F):
    return 2 * F, K, dw_gpad(B, T)


MAX_SPLITS = 64  # the K chunks the three offline callers allow (k_splits_hint)


def ola_k_splits(K_gemm):
    """K chunks of the GEMM: at most 64 k-blocks (4096 products) per fp32 accumulator, at most 64 chunks."""
    return min(-(-round_up(K_gemm, 64) // 4096), MAX_SPLITS)


def dw_k_splits(gpad):
    """K chunks of the weight-gradient GEMM: min(ceil(gpad / 4096), 64, gpad / 64)."""
    return min(-(-gpad // 4096), 64, gpad // 64)


# ------------------------------------------------------------------------------------------ shape matrices ----
# input gradient: basis "hann" (periodic-Hann DFT of n_fft = K), "perturbed" (the same plus noise: a trainable
# STFT after some steps) or ("cqt", n_bins) (a CQT1992v2 bank; K is the module's kernel width)
DX_ROWS = {
    "hann_512_128": dict(basis="hann", K=512, hop=128, B=2, L=8000, center=True, pad="reflect",
                         edge="baseline: four frames overlap every sample"),
    "hann_256_100_constant": dict(basis="hann", K=256, hop=100, B=2, L=5001, center=True, pad="constant",
                                  edge="odd hop, constant padding"),
    "hann_1024_1024_no_center": dict(basis="hann", K=1024, hop=1024, B=2, L=10000, center=False, pad="reflect",
                                     edge="hop == n_fft: frames never overlap; 784 tail samples no frame reads"),
    "hann_256_384_gaps": dict(basis="hann", K=256, hop=384, B=2, L=6000, center=False, pad="reflect",
                              edge="hop > n_fft: 128-sample gaps between frames"),
    "hann_512_reflect_L258": dict(basis="hann", K=512, hop=128, B=3, L=258, center=True, pad="reflect",
                                  edge="L = pad + 2: the two mirror ranges of the reflect adjoint overlap"),
    "hann_512_T1": dict(basis="hann", K=512, hop=128, B=2, L=512, center=False, pad="reflect",
                        edge="T = 1: one frame per clip"),
    "hann_256_64_B70": dict(basis="hann", K=256, hop=64, B=70, L=300, center=True, pad="reflect",
                            edge="70 clips of 5 frames: M tiles span clip seams"),
    "hann_24": dict(basis="hann", K=24, hop=6, B=2, L=3000, center=True, pad="reflect",
                    edge="n_fft 24: the narrowest N tile (32)"),
    "hann_100": dict(basis="hann", K=100, hop=25, B=2, L=3000, center=True, pad="reflect",
                     edge="n_fft 100: a narrow N tile (112)"),
    "hann_300": dict(basis="hann", K=300, hop=75, B=2, L=6000, center=True, pad="reflect",
                     edge="n_fft 300: a partial second N tile"),
    "hann_1000": dict(basis="hann", K=1000, hop=250, B=2, L=9000, center=True, pad="constant",
                      edge="n_fft 1000: a partial fourth N tile"),
    "cqt_f32": dict(basis=("cqt", 32), hop=256, B=2, L=12000, center=True, pad="reflect",
                    edge="CQT1992v2 bank, 2F = 64: no K padding (the prep kernel's zero_tail branch)"),
    "cqt_f64": dict(basis=("cqt", 64), hop=256, B=2, L=12000, center=True, pad="reflect",
                    edge="CQT1992v2 bank, 2F = 128: no K padding (zero_tail branch), two k-blocks"),
    "perturbed_256": dict(basis="perturbed", K=256, hop=64, B=2, L=4000, center=True, pad="reflect",
                          edge="trainable STFT bases after updates: no DFT structure"),
    "hann_16384": dict(basis="hann", K=16384, hop=4096, B=1, L=40000, center=True, pad="reflect",
                       edge="n_fft 16384: 64 N tiles, K = 16448"),
    "hann_24576": dict(basis="hann", K=24576, hop=6144, B=1, L=60000, center=True, pad="reflect",
                       edge="n_fft 24576: 96 N tiles, above the forward's 128 tiles of 2F columns"),
}

# the CQT1992v2 banks of the cqt rows (small fmin keeps the reflect padding inside the clip)
CQT_BANK = dict(sr=22050, fmin=220.0, hop_length=256)

# weight gradient: F bins of a random upstream gradient (the basis does not enter dW)
DW_ROWS = {
    "gpad_64": dict(K=256, hop=64, B=1, L=4000, center=True, pad="reflect", F=129,
                    edge="63 frames: gpad = 64, one k-block"),
    "gpad_4096": dict(K=256, hop=64, B=4, L=65500, center=True, pad="reflect", F=129,
                      edge="4096 frames: gpad = 4096, k_splits 1"),
    "gpad_4160": dict(K=256, hop=64, B=4, L=65536, center=True, pad="reflect", F=129,
                      edge="4100 frames: gpad = 4160, k_splits 2"),
    "frames_1e5": dict(K=256, hop=64, B=4, L=1600000, center=True, pad="reflect", F=129,
                       edge="100004 frames: k_splits 25"),
    "frames_275k_cap": dict(K=128, hop=32, B=8, L=1100000, center=True, pad="reflect", F=65,
                            edge="275008 frames: ceil(gpad / 4096) = 68, capped at 64 chunks"),
    "frames_999_no_center": dict(K=512, hop=128, B=3, L=43008, center=False, pad="reflect", F=257,
                                 edge="999 frames (not a multiple of 64), center=False"),
    "gaps_constant": dict(K=256, hop=384, B=2, L=20000, center=True, pad="constant", F=129,
                          edge="hop > n_fft with constant padding: frames skip samples"),
    "freq_bins_1": dict(K=256, hop=64, B=2, L=20000, center=True, pad="reflect", F=1,
                        edge="freq_bins=1: M = 2, one partial M tile"),
}

# inverse STFT: (n_fft, hop, B, T, onesided, center, length, window); length "short" / "long" = 3/4 of / 64
# samples more than the output the frames give
ISTFT_ROWS = {
    "n100_hop25": dict(n_fft=100, hop=25, B=2, T=40, onesided=True, center=True, length=None, window="hann",
                       edge="n_fft 100: narrow N tile (112), f_in 51"),
    "n300_hop150_two_sided": dict(n_fft=300, hop=150, B=2, T=30, onesided=False, center=True, length=None,
                                  window="hann", edge="n_fft 300: partial second N tile; two-sided, 2 f_in = 600"),
    "n512_hop128_hamming": dict(n_fft=512, hop=128, B=3, T=20, onesided=True, center=True, length=None,
                                window="hamming", edge="hop n/4, hamming window"),
    "n512_hop256_no_center": dict(n_fft=512, hop=256, B=2, T=20, onesided=True, center=False, length=None,
                                  window="hann", edge="hop n/2, center=False: wss -> 0 at both ends"),
    "n512_hop512_ones": dict(n_fft=512, hop=512, B=2, T=12, onesided=True, center=True, length=None,
                             window="ones", edge="hop n: no overlap, rectangular window"),
    "n512_hop768_gaps": dict(n_fft=512, hop=768, B=2, T=12, onesided=False, center=False, length=None,
                             window="hann", edge="hop 1.5 n: gaps with wss = 0"),
    "n512_length_short": dict(n_fft=512, hop=128, B=2, T=20, onesided=True, center=True, length="short",
                              window="hann", edge="length shorter than the output"),
    "n512_length_long": dict(n_fft=512, hop=128, B=2, T=20, onesided=True, center=True, length="long",
                             window="hann", edge="length longer than the output: truncated"),
    "n2048_hop441": dict(n_fft=2048, hop=441, B=2, T=12, onesided=True, center=True, length=None, window="hann",
                         edge="hop 441, not a divisor of n_fft"),
    "n2048_hop1024_no_center_length": dict(n_fft=2048, hop=1024, B=1, T=8, onesided=False, center=False,
                                           length="short", window="hamming",
                                           edge="two-sided 2048, center=False with a length"),
    "n256_T1_B70": dict(n_fft=256, hop=64, B=70, T=1, onesided=True, center=False, length=None, window="hann",
                        edge="70 clips of one frame: M tiles span clips"),
    "n16384_hop4096": dict(n_fft=16384, hop=4096, B=1, T=6, onesided=True, center=True, length=None,
                           window="hann", edge="n_fft 16384: 64 N tiles, K = 16448"),
}

# FIR decimation adjoint: (taps, factor, L, B)
FIR_ROWS = {}
for _i, (_taps, _L) in enumerate((t, L) for t in (9, 16, 255, 256) for L in (9, 1023, 1024, 1025, 4099, 100000)):
    FIR_ROWS[f"taps{_taps}_L{_L}"] = dict(taps=_taps, factor=2 + _i % 4, L=_L, B=1 + 2 * (_i % 2),
                                          edge="taps x L grid: block edges at 1024, clips shorter than a block")
FIR_ROWS["taps13000_f2_L4099"] = dict(taps=13000, factor=2, L=4099, B=1,
                                      edge="(taps + g_len) x 4 B > 48 KB: the cudaFuncSetAttribute branch")
FIR_ROWS["taps13001_f2_L30000"] = dict(taps=13001, factor=2, L=30000, B=3,
                                       edge="odd long filter above 48 KB of shared memory, three clips")
FIR_ROWS["taps20000_f5_L9000"] = dict(taps=20000, factor=5, L=9000, B=1,
                                      edge="even long filter at factor 5 above 48 KB of shared memory")


def length_of(row, T):
    """The iSTFT row's `length` argument."""
    n_fft, hop = row["n_fft"], row["hop"]
    out = n_fft + hop * (T - 1) - (2 * (n_fft // 2) if row["center"] else 0)
    if row["length"] == "short":
        return out * 3 // 4
    if row["length"] == "long":
        return out + 64
    return None
