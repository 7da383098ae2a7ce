"""Host-side checks (no GPU) of what tests/test_zz_gpu_block_domain.py trusts: the float64 STFT reference against
the CPU oracle, the launch model of the block-partial kernel (tile widths, N tiles, K of each instance) against
the figures DESIGN §3.1b quotes, and the shape matrix's geometry (partial last M tiles that straddle clips)."""
import numpy as np
import pytest

import block_domain as bd
from block_domain import bp
from helpers import build, oracle, rel_errors
from nnaudio_b200 import _C
from nnaudio_b200.design import gammatone_filterbank, mel_filterbank

# (n_fft, hop, L, center, pad_mode)
REF_CASES = [(256, 64, 1000, True, "reflect"), (512, 128, 1999, True, "constant"), (384, 192, 1500, False, "reflect")]


def _oracle_formats(x, wsin, wcos, hop, center, pad_mode):
    return {f: oracle.stft(x, wsin, wcos, hop, center, pad_mode, f) for f in ("Complex", "Magnitude", "Phase")}


def _ref_formats(x, n_fft, hop, center, pad_mode):
    X = bd.ref_stft(x, n_fft, hop, center, pad_mode)
    return {"Complex": np.stack((X.real, X.imag), -1), "Magnitude": np.abs(X), "Phase": np.angle(X)}


@pytest.mark.parametrize("n_fft,hop,L,center,pad_mode", REF_CASES)
def test_ref_stft_equals_the_oracle_on_float64_hann_bases(n_fft, hop, L, center, pad_mode):
    """The module's basis definition evaluated in float64: the framing, padding and sign convention of
    ``ref_stft`` are the oracle's to rounding."""
    x = np.random.RandomState(n_fft + L).standard_normal((2, L))
    wsin, wcos = bd.hann_dft_bases(n_fft)
    want = _oracle_formats(x, wsin, wcos, hop, center, pad_mode)
    got = _ref_formats(x, n_fft, hop, center, pad_mode)
    for fmt in ("Complex", "Magnitude"):
        emax, el2 = rel_errors(got[fmt], want[fmt])
        assert emax < 1e-12 and el2 < 1e-12, (fmt, emax, el2)
    # angles as unit vectors (an angle of a real negative bin may sit at +pi or -pi)
    u = lambda a: np.stack((np.cos(a), np.sin(a)), -1)  # noqa: E731
    mask = want["Magnitude"] > 1e-6 * want["Magnitude"].max()
    assert np.abs(u(got["Phase"]) - u(want["Phase"]))[mask].max() < 1e-9


@pytest.mark.parametrize("n_fft,hop,L,center,pad_mode", REF_CASES)
def test_ref_stft_matches_the_oracle_on_the_module_buffers(n_fft, hop, L, center, pad_mode):
    """The module's own float32 buffers carry each basis value to within three float32 roundings (sin / cos,
    window, product: 3 x 2^-24 ~ 1.8e-7 relative), so the oracle evaluated on them sits that close to the
    exact transform; 1e-6 leaves room for the max over many outputs and nothing for a wrong frame or sign."""
    mod = build("STFT", dict(n_fft=n_fft, hop_length=hop, center=center, pad_mode=pad_mode))
    x = np.random.RandomState(n_fft + L + 1).standard_normal((2, L))
    want = _oracle_formats(x, mod.wsin.numpy(), mod.wcos.numpy(), hop, center, pad_mode)
    got = _ref_formats(x, n_fft, hop, center, pad_mode)
    for fmt in ("Complex", "Magnitude"):
        emax, el2 = rel_errors(got[fmt], want[fmt])
        assert emax < 1e-6 and el2 < 1e-6, (fmt, emax, el2)


# (n_fft, hop) -> (nb, N tiles, K of the GEMM, packed bins): DESIGN §3.1b and the shape matrix
LAUNCH = {
    (128, 64): (72, 1, 64, 65),
    (384, 192): (104, 2, 192, 193),
    (256, 128): (40, 1, 32, 33),
    (768, 384): (104, 1, 96, 97),
    (1536, 384): (104, 2, 96, 193),
    (2048, 512): (88, 3, 128, 257),
    (8192, 2048): (96, 11, 512, 1025),
    (16384, 4096): (112, 19, 1024, 2049),
    (32768, 8192): (120, 35, 2048, 4097),
}


@pytest.mark.parametrize("n_fft,hop", sorted(LAUNCH))
def test_launch_model_tile_widths(n_fft, hop):
    nb, n_tiles, K, Fb = LAUNCH[(n_fft, hop)]
    assert bd.basis_bins(n_fft, hop) == Fb
    assert bp.choose_nb(Fb) == nb and bp.n_tiles_of(Fb, nb) == n_tiles
    # Kb: the flop count carries the factor of 4 that tells the two instances apart
    one = bd.block_exec_flops(n_fft, hop, 1, 40 * hop, True)
    assert one == 3 * 2 * bd.geometry(n_fft, hop, 1, 40 * hop, True)[2] * n_tiles * 128 * 2 * nb * K
    assert bd.block_exec_flops(n_fft, hop, 1, 40 * hop, True, passes=2) * 3 == one * 2


@pytest.mark.parametrize("shape", bd.STFT_SHAPES + bd.STFT_SHAPES_DIRECT, ids=lambda s: f"{s[0]}-{s[1]}")
def test_shape_matrix_leaves_partial_m_tiles_across_clips(shape):
    n_fft, hop, B, L = shape
    assert B > 1 and L % hop != 0
    for center in (True, False):
        t_slots, rows, m_tiles = bd.geometry(n_fft, hop, B, L, center)
        assert (B * t_slots) % rows != 0 and t_slots % (33 - n_fft // hop) != 0, (center, t_slots, rows)


def test_short_clip_batches_put_several_clips_in_one_m_tile():
    # 512/128, B = 37, L = 300: t_slots = 7 (T = 3) under 29-row tiles; 256/64, B = 50, L = 200: 8 under 116
    assert bd.geometry(512, 128, 37, 300, True)[:2] == (7, 29)
    assert bd.geometry(256, 64, 50, 200, True)[:2] == (8, 116)


@pytest.mark.parametrize("sr,n_fft,n_mels", [(16000, 2048, 40), (16000, 8192, 64)])
def test_banks_without_a_deterministic_four_phase_width(sr, n_fft, n_mels):
    """The table builder finds no width with <= 2 partial sums per filter: the launch keeps the default nb."""
    fb = mel_filterbank(sr, n_fft, n_mels)
    assert bp.choose_poly_tile(fb) is None
    assert bd.fbank_nb(fb, n_fft, n_fft // 4) == (bp.choose_nb(n_fft // 8 + 1), False)


@pytest.mark.parametrize("sr,n_fft,n_mels", [(16000, 256, 40), (8000, 384, 32)])
def test_one_phase_fused_mel_width_keeps_two_partial_sums(sr, n_fft, n_mels):
    fb = mel_filterbank(sr, n_fft, n_mels)
    nb = bd.one_phase_fb_width(fb)
    assert nb is not None and 32 <= nb <= 128 and nb % 8 == 0
    # every filter support meets at most two (tile, warp part) ranges at that width
    outs = nb - 2
    for r in fb:
        k = r.nonzero()[0]
        parts = {(kk // outs, (kk % outs + 2) // 8 >= (nb // 8) // 2) for kk in range(k.min(), k.max() + 1)}
        assert len(parts) <= 2


def test_planes_gemm_model():
    """Gammatone's second launch: 64 filters -> fh = 32 complex rows (bn = 64, one N tile) over kp columns."""
    fb = gammatone_filterbank(16000, 8192, 64)
    assert fb.shape == (64, 4097)
    # nb = 96, 11 tiles, 4 families: 4224 columns (a multiple of 64)
    assert bd.planes_gemm_flops(8192, 2048, 2, 10, 64) == 6 * 128 * 64 * 4224
    assert bd.choose_bn(32) == 64


@pytest.mark.parametrize("n_fft,hop", [(32768, 16384), (32768, 8192)])
def test_block_shapes_past_the_dense_kernels_n_tile_limit(n_fft, hop):
    """The dense kernel takes at most 128 N tiles (TC_MAX_N_TILES); these block shapes need more at any width, so
    the dispatch must not hold a block-partial basis to that limit (it would run the SIMT kernel instead)."""
    assert _C.block_layout_ok(n_fft, hop)
    F = n_fft // 2 + 1
    assert -(-(2 * F) // bd.choose_bn(F)) > 128
    assert bp.n_tiles_of(bd.basis_bins(n_fft, hop), bp.choose_nb(bd.basis_bins(n_fft, hop))) <= 35
