"""Host-side checks (no GPU) of the four-phase block-partial STFT kernel (csrc/tcb_kernels.cu, PH = 4): the float64
spec and the kernel's index arithmetic (tools/block_poly_emulation.py) against ``np.fft.rfft`` of Hann-windowed
frames, every bin emitted exactly once, the fused-Mel range cuts (at most two partial sums per filter, so the
atomic adds commute), and the FMT_PLANES column order (tile, family, packed column) with the re-indexed bank."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import block_poly_emulation as bp  # noqa: E402
from block_dft_emulation import stft_dense  # noqa: E402

from nnaudio_b200.design import mel_filterbank  # noqa: E402


@pytest.mark.parametrize("n_fft,hop", [(2048, 512), (2048, 1024), (1024, 256), (512, 128), (512, 256), (4096, 1024)])
def test_spec_matches_rfft_of_hann_frames(n_fft, hop):
    x = np.random.default_rng(n_fft + hop).standard_normal(hop * 23 + 17)
    want, got = stft_dense(x, n_fft, hop), bp.stft_poly(x, n_fft, hop)
    assert np.abs(got - want).max() / np.abs(want).max() < 1e-12


@pytest.mark.parametrize("n_fft,hop,B,L,split", [(2048, 512, 2, 512 * 33 + 100, None), (512, 128, 1, 5000, None),
                                                 (1024, 512, 2, 7000, 5), (2048, 1024, 1, 9000, 3)])
def test_kernel_index_replay_matches_rfft_and_writes_each_output_once(n_fft, hop, B, L, split):
    x = np.random.default_rng(L).standard_normal((B, L))
    got, written = bp.emulate(x, n_fft, hop, B, split=split)
    want = np.stack([stft_dense(x[b], n_fft, hop).T for b in range(B)])
    assert np.abs(got - want).max() / np.abs(want).max() < 1e-12
    assert (written == 1).all()


@pytest.mark.parametrize("n_fft", [256, 512, 1024, 2048, 4096, 8192])
def test_families_cover_every_bin_once_for_every_tile_width(n_fft):
    F, M = n_fft // 2 + 1, n_fft // 4
    for nb in range(32, 136, 8):
        seen = np.zeros(F, dtype=int)
        for n in range(bp.n_tiles_of(M // 2 + 1, nb)):
            for f in range(4):
                k0, lo, hi = bp.family_span(n, f, nb, M, F)
                for o in range(nb - 2):
                    if lo <= k0 + o < hi:
                        seen[k0 + o] += 1
        assert (seen == 1).all(), (nb, np.nonzero(seen != 1)[0][:8])


# the banks the fused Mel path runs in the benchmark and the GPU tests (cfg2, cfg5's MFCC, the determinism and
# grid tests); all have hop % 128 == 0, so they take the four-phase kernel
BANKS = [(22050, 2048, 128), (16000, 2048, 128), (16000, 1024, 80), (16000, 1024, 64)]


@pytest.mark.parametrize("sr,n_fft,n_mels", BANKS)
def test_fused_mel_cut_replay_gives_at_most_two_partial_sums(sr, n_fft, n_mels):
    fb = mel_filterbank(sr, n_fft, n_mels)
    nb = bp.choose_poly_tile(fb)
    assert nb is not None, "no tile width keeps the fused Mel sums run-to-run identical"
    assert max(bp.fb_ranges(fb, nb)) <= 2
    assert nb == bp.choose_nb(n_fft // 8 + 1)   # the width the other formats run at: no extra tiles


def test_warp_cuts_would_break_cfg2_determinism():
    """Why the two warp parts of a family quarter hand their open filter sums over in the CTA: had each part
    added its own, a filter of cfg2's bank would get three partial sums for every width and every split."""
    fb = mel_filterbank(22050, 2048, 128)
    M = 512
    supp = [(r.nonzero()[0].min(), r.nonzero()[0].max()) for r in fb]

    def cut_ranges(nb, s):
        def rng(k):
            f, t = bp.poly4_range(k, M, nb)
            kq = (k, M - k, k - M, 2 * M - k)[f]
            o = kq - t * (nb - 2)
            o = nb - 3 - o if f & 1 else o
            return f, t, (o + 2) // 8 >= s
        return max(len({rng(k) for k in range(lo, hi + 1)}) for lo, hi in supp)

    assert all(cut_ranges(nb, s) > 2 for nb in range(32, 136, 8) for s in range(1, nb // 8))


def planes_row(power, nb, n_tiles, kp, M):
    """What the FMT_PLANES epilogue writes for one frame: family f of tile n at columns nb (4 n + f) + i."""
    F = power.shape[0]
    row = np.full(kp, np.nan)
    for n in range(n_tiles):
        for f in range(4):
            k0, lo, hi = bp.family_span(n, f, nb, M, F)
            for i in range(nb):
                k = k0 + i - 2
                row[nb * (4 * n + f) + i] = power[k] if i >= 2 and lo <= k < hi else 0.0
    row[4 * nb * n_tiles:] = 0.0              # the tail the launcher clears
    return row


def tile_bank(fb, nb, n_tiles, kp, M):
    """fb_tile_bank_kernel with four phases."""
    n_fb, F = fb.shape
    fh = (n_fb + 1) // 2
    w_re, w_im = np.zeros((fh, kp)), np.zeros((fh, kp))
    for col in range(kp):
        n, f, i = col // (4 * nb), (col // nb) % 4, col % nb
        k0, lo, hi = bp.family_span(n, f, nb, M, F)
        k = k0 + i - 2
        if n < n_tiles and i >= 2 and lo <= k < hi:
            w_re[:, col] = fb[:fh, k]
            w_im[: n_fb - fh, col] = -fb[fh:, k]
    return w_re, w_im, fh


@pytest.mark.parametrize("n_fft,n_fb", [(2048, 64), (1024, 32), (512, 33), (4096, 96), (256, 1)])
def test_family_ordered_planes_times_reindexed_bank_is_the_filterbank_product(n_fft, n_fb):
    rng = np.random.RandomState(n_fft + n_fb)
    F, M = n_fft // 2 + 1, n_fft // 4
    nb = bp.choose_nb(M // 2 + 1)
    n_tiles = bp.n_tiles_of(M // 2 + 1, nb)
    kp = (4 * nb * n_tiles + 63) // 64 * 64
    power = rng.rand(F)
    fb = rng.standard_normal((n_fb, F))
    row = planes_row(power, nb, n_tiles, kp, M)
    assert np.isfinite(row).all()
    w_re, w_im, fh = tile_bank(fb, nb, n_tiles, kp, M)
    re, im = w_re @ row, -(w_im @ row)
    out = np.concatenate([re, im[: n_fb - fh]])
    np.testing.assert_allclose(out, fb @ power, rtol=1e-12, atol=1e-12)
