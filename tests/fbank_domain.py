"""Bank matrix, float64 references and launch model of the filterbank stage of MelSpectrogram, Gammatonegram and
MFCC: the fused epilogue (FB_FUSED) of the warp-specialised four-phase kernel (``framed_tcb_ws_kernel``, nb <= 88),
of the plain four-phase and one-phase block-partial kernels and of the dense kernel; the operand planes plus a
second GEMM (FB_PLANES); the fp32 power spectrogram plus ``filterbank_kernel`` (FB_GEMM); and the MFCC tail
(``clip_max_kernel`` + ``mfcc_tail_kernel``).  Shared by tests/test_fbank_domain_host.py (CPU) and
tests/test_zz_gpu_fbank_domain.py (-m gpu).

Which route and tile width a call takes depends on the bank, not only on the shape: its support decides whether a
table exists (<= 2 non-zeros per bin), the fused launch's width nb, whether a four-phase launch takes the
warp-specialised kernel, and whether the atomics are run-to-run identical.  ``dense_domain.plan`` models all of
that; this module adds the banks that reach each cell, their properties, and an independent replay of
``fb_steps_kernel``'s range cuts."""
import numpy as np

import block_domain as bd
import dense_domain as dd
import helpers  # noqa: F401  (puts the repository on sys.path)
from nnaudio_b200 import _C, design

FUSED, PLANES, GEMM = _C.STFT_FB_FUSED, _C.STFT_FB_PLANES, _C.STFT_FB_GEMM
BLK, D = _C.STFT_BLOCK, _C.STFT_DENSE

CFG2 = dict(sr=22050, n_fft=2048, hop_length=512, n_mels=128)
CFG5 = dict(sr=16000)  # MFCC: n_fft 2048, hop 512, n_mels 128, n_mfcc 20


# ------------------------------------------------------------------------------------------- bank edits ----
def _bin_with_two(fb):
    """The middle bin among those with exactly two non-zero filters, and those filters."""
    nz = np.asarray(fb) != 0
    ks = np.flatnonzero(nz.sum(axis=0) == 2)
    k = int(ks[len(ks) // 2])
    j0, j1 = np.flatnonzero(nz[:, k])
    return k, int(j0), int(j1)


def negate_odd(fb):
    """Every odd filter negated: the support (and so the table, route and width) is unchanged, the sums signed."""
    fb[1::2] *= -1


def extra_nonzero(fb):
    """One extra non-zero at one bin: a third filter (the next one up) gets the weight of its neighbour there, so
    the bank has 3 non-zeros in that bin and no table."""
    k, _, j1 = _bin_with_two(fb)
    fb[j1 + 1, k] = fb[j1, k]


def zero_rows(fb):
    """Three interior filters zeroed: empty filters inside the bank."""
    m = fb.shape[0] // 2
    fb[m - 1:m + 2] = 0


EDITS = {"negate_odd": negate_odd, "extra_nonzero": extra_nonzero, "zero_rows": zero_rows}


# ------------------------------------------------------------------------------------------- the matrix ----
# name -> (class, constructor, edit, (B, L), claims about the row's plan and bank, options).  ``edit`` names one
# of EDITS, applied in place to the built module's bank.  Options: ``planes`` (NNAB_FB_PLANES), ``levels``
# (per-clip gains; 0 is exact silence), ``switch`` (the edit is applied after a first call on the unedited bank:
# the claims are the edited bank's, ``before`` the unedited one's routes), ``burst`` ((Hz, amplitude, hops): a
# tone added over each clip's last hops).
# Claims: routes, nb, ws, deterministic (plan); empty (filters without a non-zero), unfiltered (bins without a
# filter), max_nnz (non-zeros per bin), max_sums (partial sums per filter at the launched width).
ROWS = {
    # ---- fused, warp-specialised four-phase kernel (nb <= 88)
    "cfg2_bank": ("MelSpectrogram", CFG2, None, (2, 22050), dict(routes={BLK: 1, FUSED: 1}, ws=1, deterministic=True), {}),
    "mel400_2048": ("MelSpectrogram", dict(sr=22050, n_fft=2048, hop_length=512, n_mels=400), None, (2, 30001),
                    dict(routes={BLK: 1, FUSED: 1}, ws=1, deterministic=True), {}),
    "htk_band_1024": ("MelSpectrogram", dict(sr=16000, n_fft=1024, hop_length=256, n_mels=40, htk=True, fmin=300.0,
                                             fmax=3400.0, power=1.5), None, (2, 16001),
                      dict(routes={BLK: 1, FUSED: 1}, ws=1, deterministic=False, unfiltered=315), {}),
    "mel256_512": ("MelSpectrogram", dict(sr=22050, n_fft=512, hop_length=128, n_mels=256, power=1.0), None,
                   (2, 12345), dict(routes={BLK: 1, FUSED: 1}, ws=1, deterministic=False, empty=39), {}),
    "gammatone1_2048": ("Gammatonegram", dict(sr=16000, n_fft=2048, hop_length=512, n_bins=1), None, (2, 20001),
                        dict(routes={BLK: 1, FUSED: 1}, ws=1, deterministic=False, max_nnz=1), {}),
    "gammatone2_2048": ("Gammatonegram", dict(sr=16000, n_fft=2048, hop_length=512, n_bins=2), None, (2, 20001),
                        dict(routes={BLK: 1, FUSED: 1}, ws=1, deterministic=False, max_nnz=2), {}),
    "mel8_2048": ("MelSpectrogram", dict(sr=16000, n_fft=2048, hop_length=512, n_mels=8), None, (2, 20001),
                  dict(routes={BLK: 1, FUSED: 1}, ws=1, deterministic=False), {}),
    # ---- fused, plain four-phase kernel (nb > 88)
    "mel128_4096": ("MelSpectrogram", dict(sr=44100, n_fft=4096, hop_length=1024, n_mels=128), None, (2, 40001),
                    dict(routes={BLK: 1, FUSED: 1}, nb=112, ws=0, deterministic=True), {}),
    "mel128_4096_r2": ("MelSpectrogram", dict(sr=44100, n_fft=4096, hop_length=2048, n_mels=128, power=1.0), None,
                       (2, 40001), dict(routes={BLK: 1, FUSED: 1}, nb=112, ws=0, deterministic=False), {}),
    "mel128_8192": ("MelSpectrogram", dict(sr=44100, n_fft=8192, hop_length=2048, n_mels=128), None, (2, 45001),
                    dict(routes={BLK: 1, FUSED: 1}, nb=96, ws=0, deterministic=False), {}),
    "mel1_8192": ("MelSpectrogram", dict(sr=44100, n_fft=8192, hop_length=2048, n_mels=1), None, (2, 45001),
                  dict(routes={BLK: 1, FUSED: 1}, nb=96, ws=0, deterministic=False), {}),
    "mel512_8192": ("MelSpectrogram", dict(sr=44100, n_fft=8192, hop_length=2048, n_mels=512, power=1.5), None,
                    (2, 45001), dict(routes={BLK: 1, FUSED: 1}, ws=0, deterministic=False), {}),
    "mel2048_8192": ("MelSpectrogram", dict(sr=44100, n_fft=8192, hop_length=2048, n_mels=2048), None, (2, 45001),
                     dict(routes={BLK: 1, FUSED: 1}, ws=0, deterministic=True, empty=160), {}),
    # ---- fused, one-phase kernel
    "mel128_256": ("MelSpectrogram", dict(sr=22050, n_fft=256, hop_length=64, n_mels=128), None, (3, 9001),
                   dict(routes={BLK: 1, FUSED: 1}, ws=0, deterministic=True, empty=20), {}),
    "mel32_384": ("MelSpectrogram", dict(sr=8000, n_fft=384, hop_length=192, n_mels=32), None, (2, 16001),
                  dict(routes={BLK: 1, FUSED: 1}, ws=0, deterministic=True), {}),
    # ---- fused, dense basis: weights ~1 (norm=None) instead of ~1e-3
    "mel_norm_none_dense": ("MelSpectrogram", dict(sr=16000, n_fft=400, hop_length=160, n_mels=64, norm=None),
                            None, (3, 16000), dict(routes={D: 1, FUSED: 1}, max_sums=2, deterministic=True), {}),
    # ---- operand planes, warp-specialised kernel: 1 -> 2 N tiles of the second GEMM
    "gammatone255_2048": ("Gammatonegram", dict(sr=16000, n_fft=2048, hop_length=512, n_bins=255), None,
                          (2, 20001), dict(routes={BLK: 1, PLANES: 1}, ws=1, deterministic=True), {}),
    "gammatone256_2048": ("Gammatonegram", dict(sr=16000, n_fft=2048, hop_length=512, n_bins=256, power=1.0), None,
                          (2, 20001), dict(routes={BLK: 1, PLANES: 1}, ws=1, deterministic=True), {}),
    "gammatone257_2048": ("Gammatonegram", dict(sr=16000, n_fft=2048, hop_length=512, n_bins=257, power=1.5),
                          None, (2, 20001), dict(routes={BLK: 1, PLANES: 1}, ws=1, deterministic=True), {}),
    "gammatone512_2048": ("Gammatonegram", dict(sr=16000, n_fft=2048, hop_length=512, n_bins=512), None,
                          (2, 20001), dict(routes={BLK: 1, PLANES: 1}, ws=1, deterministic=True), {}),
    "gammatone64_256": ("Gammatonegram", dict(sr=16000, n_fft=256, hop_length=128, n_bins=64), None, (2, 12001),
                        dict(routes={BLK: 1, PLANES: 1}, nb=40, ws=1, deterministic=True), {}),
    # ---- operand planes, plain four-phase kernel
    "gammatone64_8192": ("Gammatonegram", dict(sr=16000, n_fft=8192, hop_length=2048, n_bins=64, power=1.5), None,
                         (2, 45001), dict(routes={BLK: 1, PLANES: 1}, nb=96, ws=0, deterministic=True), {}),
    # ---- power spectrogram + filterbank_kernel: 2 / 4 / 8 blockIdx.y tiles of 64 filters
    "gammatone65_gemm": ("Gammatonegram", dict(sr=16000, n_fft=1024, hop_length=300, n_bins=65), None, (2, 16000),
                         dict(routes={D: 1, GEMM: 1}, deterministic=True), {}),
    "gammatone200_gemm": ("Gammatonegram", dict(sr=16000, n_fft=1024, hop_length=300, n_bins=200), None,
                          (2, 16000), dict(routes={D: 1, GEMM: 1}, deterministic=True), {}),
    "gammatone512_gemm": ("Gammatonegram", dict(sr=16000, n_fft=1024, hop_length=300, n_bins=512), None,
                          (2, 16000), dict(routes={D: 1, GEMM: 1}, deterministic=True), {}),
    # a block basis with the operand planes off: the block kernel's FMT_POWER, then filterbank_kernel
    "gammatone64_block_gemm": ("Gammatonegram", dict(sr=16000, n_fft=1024, hop_length=256, n_bins=64), None,
                               (2, 16001), dict(routes={BLK: 1, GEMM: 1}, ws=0, deterministic=True),
                               dict(planes=False)),
    # ---- crafted banks
    "cfg2_negate_odd": ("MelSpectrogram", CFG2, "negate_odd", (2, 22050),
                        dict(routes={BLK: 1, FUSED: 1}, ws=1, deterministic=True), {}),
    "cfg2_extra_nonzero": ("MelSpectrogram", CFG2, "extra_nonzero", (2, 22050),
                           dict(routes={BLK: 1, PLANES: 1}, ws=1, deterministic=True, max_nnz=3),
                           dict(switch=True)),
    "dense_extra_nonzero": ("MelSpectrogram", dict(sr=16000, n_fft=400, hop_length=160, n_mels=64), "extra_nonzero",
                            (3, 16000), dict(routes={D: 1, GEMM: 1}, deterministic=True, max_nnz=3),
                            dict(switch=True)),
    "cfg2_zero_rows": ("MelSpectrogram", CFG2, "zero_rows", (2, 22050),
                       dict(routes={BLK: 1, FUSED: 1}, ws=1, deterministic=True, empty=3), {}),
    # ---- MFCC: the tail on the routes above
    "mfcc_cfg5": ("MFCC", CFG5, None, (2, 16000), dict(routes={BLK: 1, FUSED: 1}, ws=1, deterministic=True), {}),
    "mfcc_n1": ("MFCC", dict(CFG5, n_mfcc=1), None, (2, 16000), dict(routes={BLK: 1, FUSED: 1}), {}),
    "mfcc_n32": ("MFCC", dict(CFG5, n_mfcc=32), None, (2, 16000), dict(routes={BLK: 1, FUSED: 1}), {}),
    "mfcc_n33": ("MFCC", dict(CFG5, n_mfcc=33), None, (2, 16000), dict(routes={BLK: 1, FUSED: 1}), {}),
    "mfcc_n64": ("MFCC", dict(CFG5, n_mfcc=64), None, (2, 16000), dict(routes={BLK: 1, FUSED: 1}), {}),
    "mfcc_n20_mels16": ("MFCC", dict(CFG5, n_mfcc=20, n_mels=16), None, (2, 16000),
                        dict(routes={BLK: 1, FUSED: 1}, deterministic=False), {}),
    # the same n_mfcc > n_mels on a deterministic bank, so the tail's DCT rows meet the fp32 bound on their own
    "mfcc_n20_mels16_det": ("MFCC", dict(sr=16000, n_fft=512, hop_length=128, n_mfcc=20, n_mels=16), None,
                            (2, 16000), dict(routes={BLK: 1, FUSED: 1}, ws=1, deterministic=True), {}),
    "mfcc_mels400": ("MFCC", dict(sr=22050, n_mfcc=40, n_mels=400), None, (2, 30001),
                     dict(routes={BLK: 1, FUSED: 1}, deterministic=True), {}),
    "mfcc_mels1600": ("MFCC", dict(sr=22050, n_fft=8192, hop_length=2048, n_mfcc=40, n_mels=1600), None,
                      (2, 45001), dict(routes={BLK: 1, FUSED: 1}, deterministic=True), {}),
    "mfcc_mels2048": ("MFCC", dict(sr=22050, n_fft=8192, hop_length=2048, n_mfcc=40, n_mels=2048), None,
                      (2, 45001), dict(routes={BLK: 1, FUSED: 1}, deterministic=True), {}),
    "mfcc_top_db_none": ("MFCC", dict(CFG5, top_db=None), None, (2, 16000), dict(routes={BLK: 1, FUSED: 1}), {}),
    "mfcc_top_db_0": ("MFCC", dict(CFG5, top_db=0.0), None, (2, 16000), dict(routes={BLK: 1, FUSED: 1}), {}),
    "mfcc_ref_0.5": ("MFCC", dict(CFG5, ref=0.5), None, (2, 16000), dict(routes={BLK: 1, FUSED: 1}), {}),
    "mfcc_ref_below_amin": ("MFCC", dict(CFG5, ref=1e-12), None, (2, 16000), dict(routes={BLK: 1, FUSED: 1}), {}),
    "mfcc_ref_negative": ("MFCC", dict(CFG5, ref=-2.0), None, (2, 16000), dict(routes={BLK: 1, FUSED: 1}), {}),
    "mfcc_amin_1e-5": ("MFCC", dict(CFG5, amin=1e-5), None, (2, 16000), dict(routes={BLK: 1, FUSED: 1}), {}),
    "mfcc_levels_silent": ("MFCC", CFG5, None, (4, 16000), dict(routes={BLK: 1, FUSED: 1}),
                           dict(levels=(1.0, 1e-3, 1e-6, 0.0))),
    # 1200 frames of 128 mels: more cells per clip than clip_max_kernel's 64 x 2048-cell grid, so it strides.  A
    # loud 7 kHz tone in each clip's last frames puts the clip's peak in a high mel band, at cells past the first
    # CLIP_MAX_CELLS that only the capped grid's later strides read, and top_db 30 makes the floor bind
    "mfcc_long_clip": ("MFCC", dict(CFG5, top_db=30.0), None, (2, 512 * 1199),
                       dict(routes={BLK: 1, FUSED: 1}, T=1200, deterministic=True),
                       dict(burst=(7000.0, 100.0, 4))),
    "mfcc_extra_nonzero": ("MFCC", CFG5, "extra_nonzero", (2, 16000),
                           dict(routes={BLK: 1, PLANES: 1}, max_nnz=3, deterministic=True), dict(switch=True)),
}
DEFAULT_OPTS = dict(planes=True, levels=None, switch=False, burst=None)

# the (route, kernel) cells the matrix must reach: FB_FUSED on the WS, plain four-phase, one-phase and dense
# kernels; FB_PLANES on the WS and plain four-phase kernels; FB_GEMM after a dense and a block contraction
CELLS = {("fused", "ws"), ("fused", "ph4"), ("fused", "ph1"), ("fused", "dense"), ("planes", "ws"),
         ("planes", "ph4"), ("gemm", "dense"), ("gemm", "block")}
# the MFCC tail's chunk of DCT coefficients per launch and mel rows of them staged per shared-memory slice
MFCC_CHUNK, MFCC_MEL_SLICE = 32, 384
CLIP_MAX_CELLS = 64 * 256 * 8  # clip_max_kernel's largest grid (64 blocks) x 256 threads x 8 cells


def row_options(name):
    return dict(DEFAULT_OPTS, **ROWS[name][5])


def module_ctor(name):
    """The row's constructor with the class defaults it relies on made explicit (n_fft, hop, power)."""
    c = dict(ROWS[name][1])
    c.setdefault("n_fft", 2048)
    c.setdefault("hop_length", 512)
    return c


def power_of(name):
    return float(ROWS[name][1].get("power", 2.0))


def bank(name, edited=True):
    """The row's (n_fb, F) float64 bank as the module builds it, with its edit applied (``edited``)."""
    cls, _, edit = ROWS[name][:3]
    c = module_ctor(name)
    sr, K = c["sr"], c["n_fft"]
    if cls == "Gammatonegram":
        fb = design.gammatone_filterbank(sr, K, c.get("n_bins", 64), c.get("fmin", 0.0), c.get("fmax"))
    else:
        fb = design.mel_filterbank(sr, K, c.get("n_mels", 128), c.get("fmin", 0.0), c.get("fmax"),
                                   htk=c.get("htk", False), norm=c.get("norm", 1))
    fb = np.array(fb, dtype=np.float32).astype(np.float64)  # the module's fp32 buffer
    if edit is not None and edited:
        EDITS[edit](fb)
    return fb


def row_plan(name, fb=None, passes=3):
    """dense_domain.plan for a row on its (B, L) input and (edited) bank."""
    c = module_ctor(name)
    K, hop = c["n_fft"], c["hop_length"]
    B, L = ROWS[name][3]
    block = bool(_C.block_layout_ok(K, hop))  # every row: Hann, full DFT, untrained
    fb = bank(name) if fb is None else fb
    return dd.plan(K, K // 2 + 1, hop, B, L, True, block, "auto", fb, passes, power_of(name),
                   row_options(name)["planes"])


def row_input(name):
    """The row's (B, L) fp32 input, as float64: white noise, per-clip gains, and a tone burst at the end."""
    B, L = ROWS[name][3]
    opts = row_options(name)
    x = np.random.RandomState(len(name) * 1000 + B).standard_normal((B, L))
    if opts["levels"] is not None:
        x = x * np.asarray(opts["levels"])[:, None]
    if opts["burst"] is not None:
        hz, amp, hops = opts["burst"]
        n = hops * module_ctor(name)["hop_length"]
        x[:, L - n:] += amp * np.sin(2.0 * np.pi * hz / ROWS[name][1]["sr"] * np.arange(n))
    return x.astype(np.float32).astype(np.float64)


def cell(p):
    """(route, kernel) of a plan."""
    r = p["routes"]
    route = "fused" if FUSED in r else ("planes" if PLANES in r else "gemm")
    if BLK not in r:
        return route, "dense"
    if route == "gemm":
        return route, "block"
    return route, ("ws" if p["ws"] else ("ph4" if bd.poly4(p["hop"]) else "ph1"))


# ---------------------------------------------------------------------------------- bank properties ----
def _one_phase_range(k, nb):
    """fb_steps_kernel's one-phase range index of bin k at width nb: tile k // (nb - 2), then the warp part that
    owns chunk (k % (nb - 2) + 2) // 8."""
    outs, n_chunks = nb - 2, nb // 8
    c = (k % outs + 2) // 8
    part = 0
    while part + 1 < 2 and c >= (n_chunks * (part + 1)) // 2:
        part += 1
    return 2 * (k // outs) + part


def _four_phase_range(k, M, nb):
    """common.cuh poly4_range, restated: the family f of bin k (quarters of 2M + 1 bins; families 1 and 3 run
    downwards from M and 2M), then the tile of its family-local bin kq."""
    f = 0 if k < M // 2 else (1 if k < M else (2 if k < 3 * M // 2 else 3))
    kq = (k, M - k, k - M, 2 * M - k)[f]
    return f * 4096 + kq // (nb - 2)


def _supports(fb):
    """(lo, hi) bins of each filter's support as the table records it (first two non-zeros per bin), None for a
    filter the table never names."""
    ent, _ = dd.fb_entries(fb)
    sup = [None] * fb.shape[0]
    for k, (j0, j1) in enumerate(ent):
        for j in (j0, j1):
            if j >= 0:
                sup[j] = (sup[j][0], k) if sup[j] else (k, k)
    return sup


def replay_widths(fb, n_fft, hop):
    """fb_steps_kernel replayed bin by bin: for each width nb = 32 .. 128 the most partial sums any filter gets
    (1 + the range changes across its support; the one- and four-phase range cuts are restated above from the
    CUDA source, not taken from block_poly_emulation, which block_domain.fbank_nb uses), then the launch's width:
    the cheapest qualifying one (block_choose_nb's cost), else block_choose_nb.  Returns (nb, deterministic,
    {nb: most partial sums})."""
    F = fb.shape[1]
    poly = bd.poly4(hop)
    M = (F - 1) // 2
    worst = {}
    for nb in range(32, 136, 8):
        w = 0
        for s in _supports(fb):
            if s is None:
                continue
            lo, hi = s
            if poly:
                r = [_four_phase_range(k, M, nb) for k in range(lo, hi + 1)]
            else:
                r = [_one_phase_range(k, nb) for k in range(lo, hi + 1)]
            w = max(w, 1 + sum(a != b for a, b in zip(r, r[1:])))
        worst[nb] = w
    Fb = M // 2 + 1 if poly else F
    ok = [nb for nb in worst if worst[nb] <= 2]
    if not ok:
        return bd.bp.choose_nb(bd.basis_bins(n_fft, hop)), False, worst
    best = min(ok, key=lambda nb: (bd.bp.n_tiles_of(Fb, nb) * (nb + 6), nb))
    return best, True, worst


def properties(fb, p):
    """Bank properties of a row: empty filters, bins without a filter, most non-zeros per bin, most partial sums
    a filter receives on the row's route (None off the fused route), and the plan's nb / ws / deterministic."""
    nz = np.asarray(fb) != 0
    _, max_nnz = dd.fb_entries(fb)
    out = dict(empty=int((~nz.any(axis=1)).sum()), unfiltered=int((~nz.any(axis=0)).sum()), max_nnz=max_nnz,
               nb=p["nb"], ws=p["ws"], deterministic=p["deterministic"], max_sums=None)
    if FUSED in p["routes"]:
        if BLK in p["routes"]:
            out["max_sums"] = replay_widths(fb, p["K"], p["hop"])[2][p["nb"]]
        else:
            out["max_sums"] = max(dd.dense_partial_sums(fb, p["F"]))
    return out


# ------------------------------------------------------------------------------------------ references ----
def ref_output(x, fb, n_fft, hop, power):
    """(B, n_fb, T) float64 fb @ |X| ** power of the Hann STFT of ``x`` (every row's basis)."""
    return dd.ref_filterbank(bd.ref_stft(x, n_fft, hop), fb, power)


def db(S, amin, ref, top_db):
    """float64 dB of a (B, n_mels, T) mel spectrogram with the per-clip top_db floor (the reference takes |ref|)."""
    v = 10.0 * np.log10(np.maximum(np.asarray(S, dtype=np.float64), amin)) - 10.0 * np.log10(max(amin, abs(ref)))
    if top_db is not None:
        v = np.maximum(v, v.max(axis=(1, 2), keepdims=True) - top_db)
    return v


def mfcc_tail(S, dct, amin, ref, top_db):
    """The tail in float64 on a given mel spectrogram: dB, top_db floor, the module's (n_mfcc, n_mels) DCT rows.
    Returns (coefficients, dB values)."""
    v = db(S, amin, ref, top_db)
    return np.matmul(np.asarray(dct, dtype=np.float64), v), v


def tail_bound(dct, v):
    """|c_gpu - c_ref| bound of the tail on the same mel input: fp32 accumulation over n_mels terms, plus the
    MUFU.LG2 error of the dB (~1e-6 dB; 2e-5 gives 20x headroom) through the DCT.  The floor clamp and the per-clip
    peak are 1-Lipschitz and add nothing."""
    D = np.abs(np.asarray(dct, dtype=np.float64))
    n_mels = D.shape[1]
    return 4.0 * 2.0 ** -23 * n_mels * np.matmul(D, np.abs(v)) + 2e-5 * D.sum(axis=1)[None, :, None]


def silent_c0(n_mels, amin, ref):
    """c0 of a silent clip: every dB value is 10 log10(amin) - ref_dB, the floor changes nothing."""
    return np.sqrt(n_mels) * (10.0 * np.log10(amin) - 10.0 * np.log10(max(amin, abs(ref))))
