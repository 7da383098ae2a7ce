"""Float64 reference, launch model and shape matrix of the STFT family off the block-partial kernel: the dense
tensor-core kernel (``framed_tc_kernel``, csrc/tc_kernels.cu) with and without split-K, and the CUDA-core kernel
(``framed_cplx_simt_kernel``), for STFT, MelSpectrogram, MFCC and Gammatonegram.  Shared by
tests/test_dense_domain_host.py (CPU) and tests/test_zz_gpu_dense_domain.py (-m gpu).

``ref_stft`` contracts centre-padded frames with the module's own fp32 ``wcos`` / ``wsin`` upcast to float64, so
any window, ``win_length``, ``freq_bins`` / ``freq_scale`` or trained basis has an exact reference.  ``plan``
restates how one offline call picks its routes (``_C.stft_route_count``: the contraction's kernel, and for a
filterbank the way the bank is applied) and what it adds to the executed-MMA-flop counter."""
from math import gcd

import numpy as np

import block_domain as bd
import helpers  # noqa: F401  (puts the repository on sys.path)
from nnaudio_b200 import _C, design

TC_BM = 128            # M tile (frames)
TC_MAX_N_TILES = 128   # tc_supported: dense N tiles
SPLITK_MIN_K = 8192    # tc_splitk_scratch_bytes: the STFT's split-K scratch, long bases only
MAX_SPLITS = 16

ROUTE_NAMES = {_C.STFT_BLOCK: "block", _C.STFT_DENSE: "dense", _C.STFT_DENSE_SPLITK: "dense_splitk",
               _C.STFT_SIMT: "simt", _C.STFT_FB_FUSED: "fb_fused", _C.STFT_FB_PLANES: "fb_planes",
               _C.STFT_FB_GEMM: "fb_gemm"}


def _ceil(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------ reference ----
def frames(x, K, hop, center=True, pad_mode="reflect"):
    """(B, T, K) float64 frames of (B, L) ``x`` after the centre padding of K // 2 (reflect or zeros)."""
    x = np.atleast_2d(np.asarray(x, dtype=np.float64))
    if center:
        p = K // 2
        x = np.pad(x, ((0, 0), (p, p)), mode="reflect" if pad_mode == "reflect" else "constant")
    T = (x.shape[-1] - K) // hop + 1
    return x[:, np.arange(K)[None, :] + hop * np.arange(T)[:, None]]


def ref_stft(x, wcos, wsin, hop, center=True, pad_mode="reflect"):
    """(B, F, T) complex128 X = frames . wcos - i frames . wsin, the bases ((F, K) or (F, 1, K), any dtype)
    upcast to float64.  Complex output = (Re X, Im X), Phase = angle(X), Magnitude = |X|."""
    wc = np.asarray(wcos, dtype=np.float64).reshape(np.shape(wcos)[0], -1)
    ws = np.asarray(wsin, dtype=np.float64).reshape(wc.shape)
    fr = frames(x, wc.shape[1], hop, center, pad_mode)
    return (fr @ wc.T - 1j * (fr @ ws.T)).transpose(0, 2, 1)


def ref_stft_fft(x, window, hop, center=True, pad_mode="reflect"):
    """The same for the full-length windowed DFT basis (bin k = window . exp(-2 pi i k n / K)), by FFT: the
    reference of the long bases the tests build on the device (fp32 rounding of those bases is ~1e-7)."""
    fr = frames(x, len(window), hop, center, pad_mode)
    return np.fft.rfft(fr * np.asarray(window, dtype=np.float64), axis=-1).transpose(0, 2, 1)


def ref_filterbank(X, fb, power, trainable=False):
    """fb @ |X| ** power in float64 (the reference takes the magnitude first; a trainable STFT adds 1e-8 under
    the square root)."""
    mag = np.sqrt(np.abs(X) ** 2 + (1e-8 if trainable else 0.0))
    return np.matmul(np.asarray(fb, dtype=np.float64), mag ** power)


def ref_mfcc(S, n_mfcc, amin, ref, top_db):
    """The oracle's MFCC tail on a float64 mel spectrogram: dB with the per-clip top_db floor, orthonormal DCT."""
    return helpers.oracle.dct_ortho_fft_route(helpers.oracle.power_to_db(S, amin, ref, top_db))[:, :n_mfcc, :]


def window(name, n_fft, win_length=None):
    """design.fourier_basis's window: ``name`` of length win_length, centred in n_fft (float64)."""
    win_length = win_length or n_fft
    w = design._window_dispatch(name, win_length)
    lpad = (n_fft - win_length) // 2
    out = np.zeros(n_fft)
    out[lpad:lpad + win_length] = w
    return out


# ------------------------------------------------------------------------------------------- model ----
choose_bn = bd.choose_bn  # the bounded rule


def choose_bn_unbounded(F):
    """choose_bn before the N-tile bound: the least padded width, whatever its tile count."""
    cols = 2 * F
    if cols <= 256:
        return max(32, _ceil(cols, 16) * 16)
    best, best_total = 256, _ceil(cols, 256) * 256
    for bn in range(240, 127, -16):
        if _ceil(cols, bn) * bn < best_total:
            best, best_total = bn, _ceil(cols, bn) * bn
    return best


def n_tiles(F):
    return _ceil(2 * F, choose_bn(F))


def num_phases(hop):
    """num_phases (tc_kernels.cu): 8 / gcd(hop, 8) interleaved frame phases, each a multiple of 8 samples apart."""
    return 8 // gcd(hop, 8)


def fb_entries(fb):
    """fb_table_kernel: (j0, j1) of each bin, its first two non-zero filters (-1 = none), and the largest
    non-zero count of a bin."""
    fb = np.asarray(fb)
    nz = fb != 0
    ent = []
    for f in range(fb.shape[1]):
        j = np.flatnonzero(nz[:, f])
        ent.append((int(j[0]) if len(j) > 0 else -1, int(j[1]) if len(j) > 1 else -1))
    return ent, int(nz.sum(axis=0).max())


def dense_partial_sums(fb, F=None):
    """Atomic partial sums each filter receives from the dense kernel's fused epilogue (FMT_FBANK): the two
    running sums replayed over the bins of every choose_bn(F) / 2-bin N tile, one per flush."""
    ent, _ = fb_entries(fb)
    F = F or len(ent)
    half = choose_bn(F) // 2
    sums = [0] * np.shape(fb)[0]
    for f0 in range(0, F, half):
        c0 = c1 = -1
        for j0, j1 in ent[f0:min(F, f0 + half)]:
            if j0 != c0:
                if j0 == c1:
                    c0, c1 = c1, c0
                else:
                    if c0 >= 0:
                        sums[c0] += 1
                    c0 = j0
            if j1 != c1:
                if c1 >= 0:
                    sums[c1] += 1
                c1 = j1
        for c in (c0, c1):
            if c >= 0:
                sums[c] += 1
    return sums


def plan(K, F, hop, B, L, center=True, block=False, path="auto", fb=None, passes=3, power=2.0, planes=True):
    """Routes and executed flops of one fp32 offline call: an STFT (``fb`` None) or a filterbank / MFCC
    (``fb``: the (n_fb, F) bank) with a K-tap basis of F bins, hop ``hop`` and (B, L) clips.  ``block``: the
    module packed the block-partial layout; ``passes``: its MMA passes (2 for a bf16 waveform); ``power``: the
    exponent of |X|; ``planes``: NNAB_FB_PLANES (a dense bank on a block basis takes the operand planes).
    Returns a dict with ``routes`` ({STFT_* constant: 1}), ``flops`` and the quantities they were decided on,
    and for the block-partial launch its tile width ``nb``, ``ws`` (1: it runs framed_tcb_ws_kernel, the
    four-phase kernel with separate MMA and epilogue warps, else 0) and ``deterministic`` (two calls are bitwise
    equal)."""
    pad = K // 2 if center else 0
    T = (L + 2 * pad - K) // hop + 1
    n_ph = num_phases(hop)
    hop_eff = hop * n_ph
    t_slots = _ceil(L + 2 * pad, hop_eff)
    bn = choose_bn(F)
    tiles = _ceil(2 * F, bn)
    kpad = _ceil(K, 64) * 64
    p = dict(K=K, F=F, hop=hop, T=T, n_ph=n_ph, hop_eff=hop_eff, rows_mode=int(hop_eff % 64 == 0), bn=bn,
             n_tiles=tiles, kpad=kpad, t_slots=t_slots, launched=min(n_ph, T), ks=1, nb=None, ws=0,
             deterministic=True)
    simt = path == "simt"
    dense_tc = not simt and K >= 16 and L + 2 * pad >= K and tiles <= TC_MAX_N_TILES
    block = block and not simt

    def dense_flops():
        return 6.0 * p["launched"] * _ceil(B * t_slots, TC_BM) * TC_BM * tiles * kpad * bn

    def block_launch(nb, ws_format):
        """the block-partial launch at width nb; ws_format: a format framed_tcb_ws_kernel serves (FMT 5 / 9)"""
        p.update(nb=nb, ws=int(ws_format and bd.poly4(hop) and nb <= bd.WS_NB_MAX))
        return float(bd.block_exec_flops(K, hop, B, L, center, passes, nb=nb))

    def contraction(split_ok):
        if block:
            return _C.STFT_BLOCK, block_launch(bd.bp.choose_nb(bd.basis_bins(K, hop)), False)
        if not dense_tc:
            return _C.STFT_SIMT, 0.0
        nkb = kpad // 64
        ks = min(_ceil(nkb, 64), MAX_SPLITS, nkb) if (split_ok and K >= SPLITK_MIN_K) else 1
        p["ks"] = ks
        return (_C.STFT_DENSE_SPLITK if ks > 1 else _C.STFT_DENSE), dense_flops()

    if fb is None:
        r, flops = contraction(split_ok=True)
        return dict(p, routes={r: 1}, flops=flops)
    n_fb = np.shape(fb)[0]
    _, max_nnz = fb_entries(fb)
    sums = dense_partial_sums(fb, F) if max_nnz <= 2 else None
    p.update(max_nnz=max_nnz, max_sums=max(sums) if sums else None)
    has_table = max_nnz <= 2
    # the dense kernel's fused epilogue: at most two partial sums per filter, and a basis short enough to need no
    # split-K (nnab_filterbank_table_fuses)
    if has_table and not simt and (block or (dense_tc and max(sums) <= 2 and K < SPLITK_MIN_K)):
        r, flops = contraction(split_ok=False)
        if block:  # the fused launch runs at the table's deterministic width, else at the default one
            nb, det = bd.fbank_nb(np.asarray(fb), K, hop)
            flops = block_launch(nb, True)
            # the rolled MelRun epilogue (power != 2) flushes each warp part's sums on its own: the bound of two
            # partial sums per filter, and with it run-to-run identical atomics, holds for the fast path only
            p["deterministic"] = det and power == 2.0
        return dict(p, routes={r: 1, _C.STFT_FB_FUSED: 1}, flops=flops)
    if block and planes and F == K // 2 + 1:
        flops = block_launch(bd.bp.choose_nb(bd.basis_bins(K, hop)), True) + bd.planes_gemm_flops(K, hop, B, T, n_fb)
        return dict(p, routes={_C.STFT_BLOCK: 1, _C.STFT_FB_PLANES: 1}, flops=float(flops))
    r, flops = contraction(split_ok=True)  # the power spectrogram splits a long basis like the STFT
    return dict(p, routes={r: 1, _C.STFT_FB_GEMM: 1}, flops=flops)


# ------------------------------------------------------------------------------------------ the matrix ----
# name -> (class, constructor, (B, L), what the row claims about its plan, options).  Classes with a "direct:"
# prefix build their basis on the device from ``window`` (n_fft >= 8192: a module would build gigabytes of float64
# on the host) and call _C directly.  Options: formats (STFT), path, center / pad_mode, nudge (perturb a trainable
# basis), levels (per-clip gains), power.
STFT_FORMATS = ("Complex", "Magnitude", "Phase")
ONE = dict(formats=("Complex",))
D, DS, S, BLK = _C.STFT_DENSE, _C.STFT_DENSE_SPLITK, _C.STFT_SIMT, _C.STFT_BLOCK
FUSED, PLANES, GEMM = _C.STFT_FB_FUSED, _C.STFT_FB_PLANES, _C.STFT_FB_GEMM
ROWS = {
    # ---- STFT on the dense kernel
    "hamming_rows": ("STFT", dict(n_fft=512, hop_length=128, window="hamming"), (2, 128 * 90 + 77),
                     dict(routes={D: 1}, n_ph=1, rows_mode=1, bn=176, n_tiles=3), dict(formats=STFT_FORMATS)),
    "win_length_400": ("STFT", dict(n_fft=512, hop_length=160, win_length=400), (2, 16001),
                       dict(routes={D: 1}, rows_mode=0), dict(formats=STFT_FORMATS)),
    "speech_400_160": ("STFT", dict(n_fft=400, hop_length=160), (3, 16000),
                       dict(routes={D: 1}, n_ph=1, rows_mode=0), dict(formats=STFT_FORMATS)),
    "phases2_400_100": ("STFT", dict(n_fft=400, hop_length=100), (2, 12345),
                        dict(routes={D: 1}, n_ph=2, hop_eff=200), ONE),
    "phases4_1000_250": ("STFT", dict(n_fft=1000, hop_length=250), (2, 22050),
                         dict(routes={D: 1}, n_ph=4, bn=144, n_tiles=7), dict(formats=STFT_FORMATS)),
    "phases8_T3": ("STFT", dict(n_fft=256, hop_length=37, center=False), (3, 256 + 2 * 37 + 5),
                   dict(routes={D: 1}, n_ph=8, T=3, launched=3), dict(formats=("Complex", "Magnitude"))),
    "hann_r4_hop96": ("STFT", dict(n_fft=384, hop_length=96), (2, 9999), dict(routes={D: 1}, rows_mode=0), ONE),
    "f65_hamming": ("STFT", dict(n_fft=128, hop_length=32, window="hamming"), (2, 5003),
                    dict(routes={D: 1}, bn=144, n_tiles=1), ONE),
    "f128_linear": ("STFT", dict(n_fft=512, hop_length=128, freq_bins=128, freq_scale="linear", sr=16000,
                                 fmin=50, fmax=6000), (2, 16001), dict(routes={D: 1}, F=128, bn=256, n_tiles=1),
                    dict(formats=STFT_FORMATS)),
    "f129_hamming": ("STFT", dict(n_fft=256, hop_length=64, window="hamming"), (2, 8001),
                     dict(routes={D: 1}, bn=144, n_tiles=2), ONE),
    "log_bins": ("STFT", dict(n_fft=1024, hop_length=256, freq_bins=100, freq_scale="log", sr=22050, fmin=55,
                              fmax=10000), (2, 22050), dict(routes={D: 1}, F=100), dict(formats=STFT_FORMATS)),
    "log2_bins": ("STFT", dict(n_fft=2048, hop_length=441, freq_bins=84, freq_scale="log2", sr=44100, fmin=32.7,
                               fmax=16000), (2, 44100), dict(routes={D: 1}, F=84, n_ph=8), ONE),
    "linear_bins": ("STFT", dict(n_fft=1024, hop_length=256, freq_scale="linear", sr=22050, fmin=50, fmax=8000),
                    (2, 22050), dict(routes={D: 1}, F=513), ONE),
    "k6000_phases2": ("STFT", dict(n_fft=6000, hop_length=1500, window="hamming"), (2, 40001),
                      dict(routes={D: 1}, kpad=6016, n_ph=2), dict(formats=("Complex", "Magnitude"))),
    "trained_basis": ("STFT", dict(n_fft=512, hop_length=128, trainable=True), (2, 12001), dict(routes={D: 1}),
                      dict(formats=STFT_FORMATS, nudge=1e-3)),
    "short_clips_reflect": ("STFT", dict(n_fft=256, hop_length=100, window="hamming"), (37, 300),
                            dict(routes={D: 1}, n_ph=2), dict(formats=("Complex", "Magnitude"))),
    "short_clips_no_center": ("STFT", dict(n_fft=256, hop_length=100, window="hamming", center=False), (37, 300),
                              dict(routes={D: 1}, T=1), ONE),
    "short_clips_constant": ("STFT", dict(n_fft=256, hop_length=100, window="hamming", pad_mode="constant"),
                             (37, 300), dict(routes={D: 1}), ONE),
    # ---- long bases: split-K, and the N-tile bound of choose_bn
    "splitk_8192": ("direct:STFT", dict(n_fft=8192, hop_length=2048, window="hamming"), (2, 2048 * 20 + 333),
                    dict(routes={DS: 1}, ks=2), dict(formats=("Complex", "Magnitude"))),
    "splitk_8192_phases4": ("direct:STFT", dict(n_fft=8192, hop_length=2050, window="hamming"), (2, 2050 * 20 + 7),
                            dict(routes={DS: 1}, ks=2, n_ph=4), ONE),
    "splitk_16384": ("direct:STFT", dict(n_fft=16384, hop_length=4096, window="hamming"), (2, 4096 * 12 + 1001),
                     dict(routes={DS: 1}, ks=4), ONE),
    "ntile_bound_24576": ("direct:STFT", dict(n_fft=24576, hop_length=6144, window="hamming"), (1, 6144 * 10 + 77),
                          dict(routes={DS: 1}, ks=6, bn=224, n_tiles=110), dict(formats=("Complex", "Magnitude"))),
    "ntile_bound_20000": ("direct:STFT", dict(n_fft=20000, hop_length=5000, window="hamming"), (1, 5000 * 10 + 9),
                          dict(routes={DS: 1}, ks=5, bn=176, n_tiles=114), ONE),
    "tile_limit_32768": ("direct:STFT", dict(n_fft=32768, hop_length=8192, window="hamming"), (1, 8192 * 8 + 5),
                         dict(routes={S: 1}, bn=256, n_tiles=129), ONE),
    # ---- the block-partial kernel (reached for the counters; tests/test_zz_gpu_block_domain.py holds its domain)
    "hann_block": ("STFT", dict(n_fft=512, hop_length=128), (2, 12001), dict(routes={BLK: 1}), ONE),
    "gammatone_planes": ("Gammatonegram", dict(sr=16000, n_fft=1024, hop_length=256, n_bins=64), (2, 16001),
                         dict(routes={BLK: 1, PLANES: 1}), {}),
    # ---- filterbanks on a dense basis
    "mel_fused_speech": ("MelSpectrogram", dict(sr=16000, n_fft=400, hop_length=160, n_mels=64), (3, 16000),
                         dict(routes={D: 1, FUSED: 1}, max_sums=2), {}),
    "mel_fused_power1": ("MelSpectrogram", dict(sr=16000, n_fft=400, hop_length=160, n_mels=64, power=1.0),
                         (2, 16000), dict(routes={D: 1, FUSED: 1}), {}),
    "mel_fused_power1.5": ("MelSpectrogram", dict(sr=16000, n_fft=400, hop_length=160, n_mels=64, power=1.5),
                           (2, 16000), dict(routes={D: 1, FUSED: 1}), {}),
    "mel_fused_hamming": ("MelSpectrogram", dict(sr=16000, n_fft=512, hop_length=128, n_mels=64,
                                                 window="hamming"), (2, 16000), dict(routes={D: 1, FUSED: 1}), {}),
    "mel_3_sums": ("MelSpectrogram", dict(sr=22050, n_fft=2048, hop_length=256, n_mels=40), (2, 22050),
                   dict(routes={D: 1, GEMM: 1}, max_sums=3), {}),
    "mel_4_sums": ("MelSpectrogram", dict(sr=16000, n_fft=2048, hop_length=300, n_mels=16), (2, 16000),
                   dict(routes={D: 1, GEMM: 1}, max_sums=4), {}),
    "mel_8192": ("direct:MelSpectrogram", dict(sr=16000, n_fft=8192, hop_length=2048, n_mels=128,
                                               window="hamming"), (2, 2048 * 16 + 11), dict(routes={DS: 1, GEMM: 1}),
                 {}),
    "mel_16384": ("direct:MelSpectrogram", dict(sr=44100, n_fft=16384, hop_length=4096, n_mels=128,
                                                window="hamming"), (2, 4096 * 12 + 5),
                  dict(routes={DS: 1, GEMM: 1}, max_sums=8, ks=4), {}),
    "gammatone_16384": ("direct:Gammatonegram", dict(sr=16000, n_fft=16384, hop_length=4096, n_bins=64,
                                                     window="hamming"), (2, 4096 * 12 + 5),
                        dict(routes={DS: 1, GEMM: 1}, ks=4), {}),
    "mfcc_levels": ("MFCC", dict(sr=16000, n_fft=400, hop_length=160, n_mels=40, n_mfcc=13), (3, 16000),
                    dict(routes={D: 1, FUSED: 1}), dict(levels=(1.0, 1e-3, 1e-6))),
    "gammatone_hop300_odd": ("Gammatonegram", dict(sr=16000, n_fft=1024, hop_length=300, n_bins=63), (2, 16000),
                             dict(routes={D: 1, GEMM: 1}, n_ph=2), {}),
    # ---- the CUDA-core kernel
    "simt_f32": ("STFT", dict(n_fft=62, hop_length=16), (2, 4001), dict(routes={S: 1}, F=32),
                 dict(formats=STFT_FORMATS, path="simt")),
    "simt_f257": ("STFT", dict(n_fft=512, hop_length=128, window="hamming"), (2, 12001), dict(routes={S: 1}),
                  dict(formats=STFT_FORMATS, path="simt")),
    "simt_mel": ("MelSpectrogram", dict(sr=16000, n_fft=512, hop_length=128, n_mels=40), (2, 12001),
                 dict(routes={S: 1, GEMM: 1}), dict(path="simt")),
    "simt_mel_band": ("MelSpectrogram", dict(sr=16000, n_fft=512, hop_length=128, n_mels=24, fmin=500.0,
                                             fmax=3000.0), (2, 12001), dict(routes={S: 1, GEMM: 1}),
                      dict(path="simt", zero_edges=True)),
    "simt_mfcc": ("MFCC", dict(sr=16000, n_fft=512, hop_length=128, n_mels=40, n_mfcc=20), (2, 12001),
                  dict(routes={S: 1, GEMM: 1}), dict(path="simt")),
    "simt_gammatone": ("Gammatonegram", dict(sr=16000, n_fft=512, hop_length=128, n_bins=40), (2, 12001),
                       dict(routes={S: 1, GEMM: 1}), dict(path="simt")),
}
DEFAULT_OPTS = dict(formats=("Complex",), path="auto", nudge=0.0, levels=None, zero_edges=False)


def row_options(name):
    return dict(DEFAULT_OPTS, **ROWS[name][4])


def row_geometry(name, row=None):
    """(K, F, hop, center, pad_mode, block, trainable) of a row (``row``: a row of this layout kept elsewhere), from
    its constructor alone (no basis built)."""
    cls, ctor = (row or ROWS[name])[:2]
    K, hop = ctor["n_fft"], ctor["hop_length"]
    F = ctor.get("freq_bins") or K // 2 + 1
    trainable = bool(ctor.get("trainable", False))
    hann_dft = (ctor.get("window", "hann") == "hann" and ctor.get("win_length", K) == K
                and ctor.get("freq_scale", "no") == "no" and F == K // 2 + 1)
    block = (hann_dft and not trainable and not cls.startswith("direct:")
             and bool(_C.block_layout_ok(K, hop)))
    return K, F, hop, ctor.get("center", True), ctor.get("pad_mode", "reflect"), block, trainable


def bank(name):
    """The row's (n_fb, F) float64 filterbank, as the module builds it (None for STFT rows)."""
    cls, ctor = ROWS[name][:2]
    cls = cls.split(":")[-1]
    if cls == "STFT":
        return None
    sr, K = ctor["sr"], ctor["n_fft"]
    if cls == "Gammatonegram":
        return design.gammatone_filterbank(sr, K, ctor["n_bins"])
    return design.mel_filterbank(sr, K, ctor.get("n_mels", 128), ctor.get("fmin", 0.0), ctor.get("fmax"))


def row_plan(name, bank_=None, passes=3):
    """``plan`` for a row: its modelled routes and flops on its (B, L) input (``passes=2``: bf16)."""
    K, F, hop, center, _, block, _ = row_geometry(name)
    B, L = ROWS[name][2]
    fb = bank_ if bank_ is not None else bank(name)
    return plan(K, F, hop, B, L, center, block, row_options(name)["path"], fb, passes)
