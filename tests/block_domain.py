"""Float64 reference and launch model of the block-partial STFT kernel (csrc/tcb_kernels.cu), shared by
tests/test_block_domain_host.py (CPU) and tests/test_zz_gpu_block_domain.py (-m gpu).

``ref_stft`` is ``np.fft.rfft`` of periodic-Hann-windowed frames, the transform the kernel computes from its
analytically generated basis.  ``block_exec_flops`` restates the executed-MMA-flop count the launch adds
(``launch_framed_tc_block``: passes x 2 x M tiles x N tiles x 128 x 2 nb x Kb), so a test that reads the counter
proves which instance ran: the four-phase instance has a quarter of the one-phase K, and a dense or SIMT
fallback adds a different count or none."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "tools") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "tools"))

import block_poly_emulation as bp  # noqa: E402


def ref_stft(x, n_fft, hop, center=True, pad_mode="reflect"):
    """(B, F, T) complex128 STFT of (B, L) ``x``: periodic Hann window of length n_fft, centre padding by
    n_fft // 2 (reflect or zeros).  Complex output = (re, im) of this, Phase = its angle."""
    x = np.atleast_2d(np.asarray(x, dtype=np.float64))
    if center:
        p = n_fft // 2
        x = np.pad(x, ((0, 0), (p, p)), mode="reflect" if pad_mode == "reflect" else "constant")
    T = (x.shape[-1] - n_fft) // hop + 1
    win = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(n_fft) / n_fft)
    idx = np.arange(n_fft)[None, :] + hop * np.arange(T)[:, None]
    return np.fft.rfft(x[:, idx] * win, axis=-1).transpose(0, 2, 1)


def hann_dft_bases(n_fft):
    """The module's ``wsin`` / ``wcos`` definition (design.fourier_basis, window applied) in float64,
    as (F, 1, n_fft) conv-style buffers."""
    n = np.arange(n_fft)
    k = np.arange(n_fft // 2 + 1)
    ang = 2.0 * np.pi * ((k[:, None] * n[None, :]) % n_fft) / n_fft
    win = 0.5 - 0.5 * np.cos(2.0 * np.pi * n / n_fft)
    return (np.sin(ang) * win)[:, None, :], (np.cos(ang) * win)[:, None, :]


WS_NB_MAX = 88  # TCB_WS_NB_MAX: the widest tile framed_tcb_ws_kernel takes


def poly4(hop):
    """block_poly4: four polyphase rows per block whenever hop % 128 == 0."""
    return hop % 128 == 0


def geometry(n_fft, hop, B, L, center):
    """(t_slots, rows an M tile advances, M tiles) of a launch.  num_phases(hop) == 1 for hop % 8 == 0,
    which every block shape has (hop % 64 == 0)."""
    R = n_fft // hop
    pad = n_fft // 2 if center else 0
    t_slots = -(-(L + 2 * pad) // hop)
    rows = (33 - R) if poly4(hop) else 4 * (33 - R)
    return t_slots, rows, -(-(B * t_slots) // rows)


def basis_bins(n_fft, hop):
    """Packed bins of the GEMM: F' = n_fft / 8 + 1 with four phases, F = n_fft / 2 + 1 with one."""
    return n_fft // 8 + 1 if poly4(hop) else n_fft // 2 + 1


def block_exec_flops(n_fft, hop, B, L, center, passes=3, nb=None):
    """Executed MMA flops ``launch_framed_tc_block`` adds for one launch (nb: the default width unless given)."""
    _, _, m_tiles = geometry(n_fft, hop, B, L, center)
    Fb = basis_bins(n_fft, hop)
    Kb = hop // 4 if poly4(hop) else hop
    nb = nb or bp.choose_nb(Fb)
    return passes * 2 * m_tiles * bp.n_tiles_of(Fb, nb) * 128 * 2 * nb * Kb


def one_phase_fb_width(fb):
    """The one-phase kernel's fused-filterbank width: fb_steps_kernel's nb mask (tile widths under which every
    filter's support meets at most two (tile, warp part) ranges) and the launch's cheapest qualifying width,
    or None (the launch keeps block_choose_nb)."""
    F = fb.shape[1]
    supports = [(r.nonzero()[0].min(), r.nonzero()[0].max()) for r in fb if r.any()]
    best, best_cost = None, 1 << 30
    for nb in range(32, 136, 8):
        outs, n_chunks = nb - 2, nb // 8

        def range_of(k):
            c = (k % outs + 2) // 8
            return 2 * (k // outs) + (1 if c >= n_chunks // 2 else 0)

        if any(range_of(hi) - range_of(lo) + 1 > 2 for lo, hi in supports):
            continue
        cost = bp.n_tiles_of(F, nb) * (nb + 6)
        if cost < best_cost:
            best, best_cost = nb, cost
    return best


def fbank_nb(fb, n_fft, hop):
    """(nb the fused-filterbank launch runs at, whether the table builder found a deterministic width)."""
    nb = bp.choose_poly_tile(fb) if poly4(hop) else one_phase_fb_width(fb)
    return (nb, True) if nb is not None else (bp.choose_nb(basis_bins(n_fft, hop)), False)


def choose_bn(F):
    """choose_bn (tc_kernels.cu): the dense kernel's N tile for F complex rows, the least padded width among those
    that need at most 128 tiles (TC_MAX_N_TILES; 256 when none does)."""
    cols = 2 * F
    if cols <= 256:
        return max(32, -(-cols // 16) * 16)
    best, best_total = 256, -(-cols // 256) * 256
    for bn in range(240, 127, -16):
        if -(-cols // bn) > 128:
            break
        total = -(-cols // bn) * bn
        if total < best_total:
            best, best_total = bn, total
    return best


def planes_gemm_flops(n_fft, hop, B, T, n_fb):
    """Executed MMA flops of the dense filterbank's second launch (nnab_api.cu filterbank_run, FMT_PLANES):
    B x T operand rows of kp columns against the re-indexed bank, fh = ceil(n_fb / 2) complex rows, every K
    block of every N tile (launch_framed_tc)."""
    Fb = basis_bins(n_fft, hop)
    nb = bp.choose_nb(Fb)
    kp = -(-(nb * bp.n_tiles_of(Fb, nb) * (4 if poly4(hop) else 1)) // 64) * 64
    fh = (n_fb + 1) // 2
    bn = choose_bn(fh)
    return 3 * 2 * (-(-(B * T) // 128)) * 128 * (-(-(2 * fh) // bn)) * bn * kp


# The STFT shape matrix: (n_fft, hop, B, L).  Lengths leave the last M tile partial and t_slots not a multiple of
# the frames a warp quarter emits (33 - R), so M tiles straddle clips at varying offsets.
STFT_SHAPES = [
    (128, 64, 3, 64 * 150 + 37),       # R = 2, PH = 1: smallest n_fft
    (384, 192, 2, 192 * 130 + 55),     # R = 2, PH = 1: n_fft not a power of two, 6 K blocks
    (1280, 320, 2, 320 * 120 + 99),    # R = 4, PH = 1 at a larger F
    (256, 128, 3, 128 * 70 + 45),      # R = 2, PH = 4: K = 32 (one K block), one N tile of nb = 40
    (512, 128, 2, 128 * 90 + 77),      # R = 4, PH = 4: K = 32
    (768, 384, 2, 384 * 50 + 101),     # R = 2, PH = 4: M = 192, nb = 104
    (1536, 384, 2, 384 * 60 + 13),     # R = 4, PH = 4: M = 384, nb = 104
    (8192, 2048, 2, 2048 * 30 + 333),  # F' = 1025: nb = 96, 11 N tiles
]
# built from a device basis and called directly (a module would build gigabytes of float64 on the host)
STFT_SHAPES_DIRECT = [
    (16384, 4096, 2, 4096 * 16 + 1001),  # nb = 112, 19 N tiles
    (24576, 6144, 2, 6144 * 14 + 777),   # n_fft not a power of two past the dense kernel's 128 N tiles
    (32768, 8192, 2, 8192 * 12 + 555),   # upper bound: nb = 120, 35 N tiles, K = 2048
]
# the shapes that also run center=False and center=True with zero padding
PAD_SHAPES = [(128, 64), (256, 128), (1536, 384)]
