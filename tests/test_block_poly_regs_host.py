"""Host-side checks (no GPU) of where the four-phase block-partial kernel keeps its values (csrc/tcb_kernels.cu,
tcb_poly_tile; replayed by tools/block_poly_emulation.py): the A tile's phase-interleaved rows and the wgmma
accumulator fragment give each thread all four phases of one (block row, bin) in registers, the butterfly on those
registers and the family stores fill the accumulator tile the epilogue reads exactly once, every family store
instruction is free of shared-memory bank conflicts under the tile's row XOR, and the launcher's A and B tensor maps
(dims, strides, box, origins; replayed as TMA reads them) land those rows in shared memory, with zeros past the last
block row."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import block_poly_emulation as bp  # noqa: E402

NBS = list(range(32, 136, 8))


def a_row(h, w, p, i):
    """(block row, phase) that slab h row 16 w + 8 p + i holds."""
    return 8 * w + i, 2 * h + p


@pytest.mark.parametrize("nb", NBS)
def test_each_thread_holds_all_four_phases_of_its_bins(nb):
    """Thread `lane` of warp w: register 4 j + 2 s + e of slab h is phase 2 h + s, part e (re, im) of block row
    8 w + lane / 4 and bin 4 j + lane % 4 of its warpgroup's half -- every (block row, phase, bin, part) once."""
    seen = {}
    for h in range(2):
        for w in range(4):
            for lane in range(32):
                for reg in range(nb // 2):
                    j, s, e = reg // 4, (reg // 2) & 1, reg & 1
                    row = 16 * w + lane // 4 + 8 * s                  # wgmma fragment row / column
                    col = 8 * j + 2 * (lane % 4) + e
                    block, phase = a_row(h, row // 16, (row // 8) & 1, row % 8)
                    got = (block, phase, col // 2, col & 1)           # B row 2 c + part: bin c, re | im
                    assert got == (8 * w + lane // 4, 2 * h + s, 4 * j + lane % 4, e)
                    assert got not in seen
                    seen[got] = (w, lane)
    assert len(seen) == 32 * 4 * (nb // 2) * 2


def test_a_tile_rows_follow_the_slab_map():
    blocks = np.arange(32 * 128, dtype=float).reshape(32, 128)      # hop = 128: phases of 32 columns
    rows = bp.a_tile_rows(blocks)
    for h in range(2):
        for w in range(4):
            for p in range(2):
                for i in range(8):
                    g, q = a_row(h, w, p, i)
                    np.testing.assert_array_equal(rows[64 * h + 16 * w + 8 * p + i], blocks[g, 32 * q: 32 * q + 32])


@pytest.mark.parametrize("nb", [32, 40, 88, 128])
def test_register_butterfly_fills_the_family_tile_once(nb):
    """poly_tile against the closed form: quarter f = family f of the 32 block rows, f1 and f3 column-reversed."""
    rng = np.random.default_rng(nb)
    kq = 32
    blocks = rng.standard_normal((32, 4 * kq))
    basis = rng.standard_normal((nb, kq)) + 1j * rng.standard_normal((nb, kq))
    tw = np.exp(-2j * np.pi * rng.random((4, nb)))
    tile, written = bp.poly_tile(blocks, basis, tw)
    assert (written == 1).all()
    Y = [blocks[:, q * kq: (q + 1) * kq] @ basis.T for q in range(4)]
    T = [tw[q][None, :] * Y[q] for q in range(4)]
    A0, A1, B0, B1 = T[0] + T[2], T[0] - T[2], T[1] + T[3], T[1] - T[3]
    fam = [A0 + B0, np.conj(A1 + 1j * B1)[:, ::-1], A1 - 1j * B1, np.conj(A0 - B0)[:, ::-1]]
    for f in range(4):
        np.testing.assert_allclose(tile[32 * f: 32 * f + 32, :nb] + 1j * tile[32 * f: 32 * f + 32, nb:], fam[f],
                                   rtol=1e-12, atol=1e-12)


def acc_chunk_offset(col, row, stride):
    """acc_chunk_smem (tc_ptx.cuh), relative to the tile base: 16-byte chunk c of row r at position c ^ (r & 7)."""
    chunk = col >> 2
    pos = (chunk & ~7) | ((chunk ^ row) & 7)
    return row * stride + pos * 16 + (col & 3) * 4


@pytest.mark.parametrize("nb", NBS)
def test_family_stores_match_the_tile_swizzle_and_are_conflict_free(nb):
    """tcb_store_families: the XOR form of the address is acc_chunk_smem's, and each store instruction of a warp
    (fixed warpgroup, j, family and part) touches 32 distinct banks."""
    stride = (2 * nb + 31) // 32 * 128
    for wg in range(2):
        for w in range(4):
            for j in range(nb // 8):
                for f in range(4):
                    for part in range(2):
                        banks = set()
                        for lane in range(32):
                            r = 8 * w + lane // 4
                            c = wg * nb // 2 + 4 * j + lane % 4
                            col = (nb - 1 - c if f & 1 else c) + part * nb
                            row = 32 * f + r
                            at = r * stride + 32 * f * stride + ((4 * col) ^ ((r & 7) << 4))
                            assert at == acc_chunk_offset(col, row, stride)
                            banks.add((at // 4) % 32)
                        assert len(banks) == 32


@pytest.mark.parametrize("hop,nv,m_tile", [(512, 74, 0), (512, 74, 2), (128, 20, 0), (256, 45, 1)])
def test_a_tensor_map_boxes_land_the_slab_rows_and_zero_past_the_last_block(hop, nv, m_tile):
    """The four-phase A map of launch_framed_tc_block (4-D: k, block row, phase, plane) and tcb_load_block's box
    origins give the shared-memory rows a_tile_rows describes, with zeros for block rows past the plane's last."""
    rows = nv + 5
    plane_stride = (rows * hop + 63) // 64 * 64
    rng = np.random.default_rng(hop + nv)
    planes = rng.standard_normal(2 * plane_stride)
    m0 = 29 * m_tile
    for plane in range(2):
        view = planes[plane * plane_stride: plane * plane_stride + rows * hop].reshape(rows, hop)
        blocks = np.zeros((32, hop))
        have = max(0, min(32, rows - m0))
        blocks[:have] = view[m0: m0 + have]
        want = bp.a_tile_rows(blocks)
        for k0 in range(0, hop // 4, 32):
            got = bp.load_a_stage(planes, hop, rows, plane_stride, m0, k0, plane)
            np.testing.assert_array_equal(got, want[:, k0: k0 + 32])


@pytest.mark.parametrize("nb,n_tile", [(88, 0), (88, 2), (32, 1), (128, 0)])
def test_b_tensor_map_box_is_the_tiles_interleaved_basis(nb, n_tile):
    """The four-phase B map (2 p_rows interleaved rows per plane) and the box origin 2 n0 give b_tile_rows of the
    tile's bins: MMA column 2 c + part is (re, im) of tile bin c."""
    kq, Fp = 64, 3 * 86 + 1
    p_rows = Fp + 2 + 128
    rng = np.random.default_rng(nb + n_tile)
    basis = rng.standard_normal((p_rows, kq)) + 1j * rng.standard_normal((p_rows, kq))
    packed = bp.pack_basis_pairs(basis)
    n0 = n_tile * (nb - 2)
    want = bp.b_tile_rows(basis[n0: n0 + nb])
    for k0 in range(0, kq, 32):
        np.testing.assert_array_equal(bp.load_b_stage(packed, kq, p_rows, nb, n0, k0, 0), want[:, k0: k0 + 32])
