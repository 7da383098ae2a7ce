"""Host-side checks (no GPU) of the block-partial STFT epilogue's arithmetic (csrc/tcb_kernels.cu,
epilogue_tile_block; tools/block_epilogue_emulation.py): the frame sum before the Hann window, pair-sum shuffles
and the carried columns of a chunk seam, against ``np.fft.rfft`` of Hann-windowed frames in float64, and the
float32 replay's error against the previous per-bin formula's."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import block_epilogue_emulation as be  # noqa: E402
import block_poly_emulation as bp  # noqa: E402
from block_dft_emulation import stft_dense  # noqa: E402


@pytest.mark.parametrize("n_fft,hop", [(2048, 512), (2048, 1024), (1024, 256), (512, 256), (256, 64)])
def test_frame_sum_first_matches_rfft_of_hann_frames(n_fft, hop):
    x = np.random.default_rng(n_fft + hop).standard_normal(hop * 29 + 13)
    want, got = stft_dense(x, n_fft, hop), be.stft_frame_sum_first(x, n_fft, hop)
    assert np.abs(got - want).max() / np.abs(want).max() < 1e-12


def spans(n_fft, hop, nb):
    """(k_tile0, nb) of every quarter the kernel runs: one phase, or the four families (f1, f3 column-reversed by
    the butterfly, so their k_tile0 count down from M) with four phases."""
    R = n_fft // hop
    F = n_fft // 2 + 1
    if hop % 128 == 0:
        M = n_fft // 4
        nt = bp.n_tiles_of(M // 2 + 1, nb)
        return [bp.family_span(n, f, nb, M, F)[0] for n in range(nt) for f in range(4)], R
    return [n * (nb - 2) for n in range(bp.n_tiles_of(F, nb))], R


@pytest.mark.parametrize("n_fft,hop,nb", [(2048, 512, 88), (2048, 1024, 88), (1024, 256, 72), (512, 256, 48),
                                          (256, 64, 32)])
@pytest.mark.parametrize("split", [None, 0])
def test_warp_replay_matches_rfft_in_float64(n_fft, hop, nb, split):
    """Every quarter origin (both phase counts and, with four phases, the reversed families), a warp range that
    starts at a chunk seam (c_begin > 0, seeded carried columns) or at the tile's start, and rows past the end."""
    x = np.random.default_rng(nb).standard_normal(hop * 40 + 5)
    k0s, R = spans(n_fft, hop, nb)
    cut = (nb // 8) // 2 if split is None else 0
    for k0 in k0s[:12]:
        for cb, ce in ((0, cut), (cut, nb // 8)):
            if cb == ce:
                continue
            for m0 in (0, 17):
                got, want = be.quarter_check(x, n_fft, hop, k0, nb, cb, ce, m0)
                if got.size:
                    assert np.abs(got - want).max() / np.abs(want).max() < 1e-12, (k0, cb, m0)


def tone(n, f0, sr, noise_db=None):
    t = np.arange(n)
    x = np.sin(2 * np.pi * f0 / sr * t)
    if noise_db is not None:
        x = x + 10 ** (noise_db / 20) * np.random.default_rng(3).standard_normal(n)
    return x


@pytest.mark.parametrize("n_fft,hop", [(2048, 512), (2048, 1024)])
@pytest.mark.parametrize("signal", ["tone", "tone-100dB", "noise"])
def test_float32_replay_error_within_the_previous_formula(n_fft, hop, signal):
    """The Hann 3-tap cancels hardest on a pure tone: far from the peak the bins are ~1e-7 of it.  The new order
    must not be worse there than the per-bin V-term formula it replaces (stated multiple: 1.5x the old error,
    absolute vs max|ref| and per bin away from the peak)."""
    n = hop * 60
    x = {"tone": tone(n, 440.0, 22050), "tone-100dB": tone(n, 440.0, 22050, -100),
         "noise": np.random.default_rng(5).standard_normal(n)}[signal]
    errs = {}
    for order in ("v", "s"):
        got, want = be.quarter_check(x, n_fft, hop, 0, 88, 0, 11, 7, np.float32, order)
        errs[order] = np.abs(got - want).max() / np.abs(want).max()
        far = np.abs(want) < 1e-3 * np.abs(want).max()
        errs[order + "_far"] = np.abs(got - want)[far].max() / np.abs(want).max() if far.any() else 0.0
    assert errs["s"] <= 1.5 * errs["v"], errs
    assert errs["s_far"] <= 1.5 * errs["v_far"] + 1e-12, errs
    assert errs["s"] < 1e-6, errs
