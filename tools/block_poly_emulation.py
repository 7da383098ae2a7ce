#!/usr/bin/env python
"""Executable spec (float64, CPU) of the four-phase block-partial STFT kernel, and a replay of its index
arithmetic (csrc/tcb_kernels.cu, PH = 4; csrc/common.cuh block_family_span / poly4_range).

The block DFT of tools/block_dft_emulation.py, Z_g[k] = sum_{n < hop} x[g hop + n] e^{-2 pi i k n / N}, has only
hop = N / R non-zero samples, so it splits by decimation in time.  With M = N / 4 and the polyphase rows
x_q[m] = x[g hop + 4 m + q], m < hop / 4:

    Y_q(k') = sum_m x_q[m] e^{-2 pi i k' m / M}                  k' = -1 .. M/2 + 1, K = hop / 4, one basis
    T_q     = e^{-2 pi i k' q / N} Y_q(k')
    A0 = T0 + T2, A1 = T0 - T2, B0 = T1 + T3, B1 = T1 - T3
    Z[k'] = A0 + B0     Z[M + k'] = A1 - i B1     Z[M - k'] = conj(A1 + i B1)     Z[2M - k'] = conj(A0 - B0)

The four "families" cover bins f0 [0, M/2), f1 [M/2, M), f2 [M, 3M/2), f3 [3M/2, 2M] once each; the Hann 3-tap
filter and the R-block frame sum of the one-phase kernel then run unchanged on every family.
"""
import numpy as np

from block_dft_emulation import stft_dense


def choose_nb(F):
    """block_choose_nb (tcb_kernels.cu)."""
    best, best_cost = 32, 1 << 30
    for nb in range(128, 31, -8):
        cost = ((F + nb - 3) // (nb - 2)) * (nb + 6)
        if cost < best_cost:
            best, best_cost = nb, cost
    return best


def n_tiles_of(F, nb):
    return (F + nb - 3) // (nb - 2)


def family_span(n, f, nb, M, F):
    """block_family_span: output o of family f in tile n is bin k0 + o, emitted iff in [lo, hi)."""
    kq0 = n * (nb - 2)
    if M == 0:
        return kq0, 0, F
    k0 = (kq0, M - kq0 - (nb - 3), M + kq0, 2 * M - kq0 - (nb - 3))[f]
    hi = 2 * M + 1 if f == 3 else (f + 1) * (M // 2)
    return k0, f * (M // 2), min(hi, F)


def poly4_range(k, M, nb):
    """poly4_range: the (family, tile) whose epilogue emits bin k (its two warp parts hand the filter sums open
    at their cut over inside the CTA, so a range adds one partial sum to a filter)."""
    f = 0 if k < M // 2 else (1 if k < M else (2 if k < 3 * M // 2 else 3))
    kq = (k, M - k, k - M, 2 * M - k)[f]
    return (f, kq // (nb - 2))


def block_dft_poly(blocks, n_fft):
    """Z_g[k] for k = -1 .. N/2 + 1 from the four phases (rows = blocks g)."""
    hop = blocks.shape[1]
    M = n_fft // 4
    kp = np.arange(-1, M // 2 + 2)
    m = np.arange(hop // 4)
    basis = np.exp(-2j * np.pi * np.outer(kp, m) / M)                 # (M/2 + 3, hop / 4), un-windowed
    Y = [blocks[:, q::4] @ basis.T for q in range(4)]
    T = [np.exp(-2j * np.pi * kp * q / n_fft)[None, :] * Y[q] for q in range(4)]
    A0, A1, B0, B1 = T[0] + T[2], T[0] - T[2], T[1] + T[3], T[1] - T[3]
    Z = {}
    for bins, val in ((kp, A0 + B0), (M - kp, np.conj(A1 + 1j * B1)), (M + kp, A1 - 1j * B1),
                      (2 * M - kp, np.conj(A0 - B0))):
        for i, b in enumerate(bins.tolist()):
            Z.setdefault(b, val[:, i])
    return np.stack([Z[k] for k in range(-1, n_fft // 2 + 2)], axis=1)


def stft_poly(x, n_fft, hop):
    """The spec: block DFT by the four phases, then the one-phase kernel's window filter and frame sum."""
    R = n_fft // hop
    pad = n_fft // 2
    xp = np.pad(x, pad, mode="reflect")
    T = (len(xp) - n_fft) // hop + 1
    blocks = xp[: (T + R - 1) * hop].reshape(T + R - 1, hop)
    Z = block_dft_poly(blocks, n_fft)
    F = n_fft // 2 + 1
    Z0, Zm, Zp = Z[:, 1:-1], Z[:, :-2], Z[:, 2:]
    w = np.exp(2j * np.pi / R)
    c = np.exp(-2j * np.pi * np.arange(F) / R)
    X = np.zeros((T, F), dtype=complex)
    for j in range(R):
        X += (c ** j)[None, :] * (0.5 * Z0 - 0.25 * w ** j * Zm - 0.25 * w ** (-j) * Zp)[j: j + T]
    return X


def tma_box(mem, elem_strides, dims, box, coords):
    """A tiled TMA load: the box at `coords` of the map (dims, element strides; dimension 0 contiguous) over the
    flat array `mem`, in shared-memory order (dimension 0 fastest), elements outside `dims` read as zero."""
    out = np.zeros(int(np.prod(box)))
    for n, idx in enumerate(np.ndindex(*box[::-1])):
        c = [coords[d] + idx[::-1][d] for d in range(len(box))]
        if all(0 <= c[d] < dims[d] for d in range(len(dims))):
            out[n] = mem[sum(c[d] * elem_strides[d] for d in range(len(dims)))]
    return out


def a_map(hop, rows, plane_stride):
    """launch_framed_tc_block's four-phase A map: (dims, element strides, box) of (k, block row, phase, plane)."""
    return (hop // 4, rows, 4, 2), (1, hop, hop // 4, plane_stride), (32, 8, 2, 1)


def b_map(kq, p_rows):
    """launch_framed_tc_block's four-phase B map: (dims, element strides, box rows) of (k, row, plane), rows
    2 p + part of the interleaved basis."""
    return (kq, 2 * p_rows, 2), (1, kq, 2 * p_rows * kq)


def load_a_stage(planes, hop, rows, plane_stride, m0, k0, plane):
    """tcb_load_block's eight A boxes of one plane: the 128 x 32 shared-memory rows of K block k0 .. k0 + 31."""
    dims, strides, box = a_map(hop, rows, plane_stride)
    out = np.zeros((128, 32))
    for h in range(2):
        for w in range(4):
            out[64 * h + 16 * w: 64 * h + 16 * w + 16] = tma_box(
                planes, strides, dims, box, (k0, m0 + 8 * w, 2 * h, plane)).reshape(16, 32)
    return out


def load_b_stage(packed, kq, p_rows, nb, n0, k0, plane):
    """tcb_load_block's B box of one plane: 2 nb shared-memory rows of K block k0 .. k0 + 31."""
    dims, strides = b_map(kq, p_rows)
    return tma_box(packed, strides, dims, (32, 2 * nb, 1), (k0, 2 * n0, plane)).reshape(2 * nb, 32)


def pack_basis_pairs(basis_rows):
    """pack_block_basis_kernel with four phases, as float64 (the hi plane exact, lo zero): packed[plane][2 p + part]."""
    p_rows, kq = basis_rows.shape
    packed = np.zeros((2, 2 * p_rows, kq))
    packed[0, 0::2], packed[0, 1::2] = basis_rows.real, basis_rows.imag
    return packed.ravel()


def a_tile_rows(blocks):
    """The A operand of one M tile in shared memory (tcb_load_block, four phases): slab h row 16 w + 8 p + i holds
    phase 2 h + p of block row 8 w + i.  blocks: the tile's 32 block rows in polyphase order (hop columns)."""
    kq = blocks.shape[1] // 4
    rows = np.zeros((128, kq))
    for h in range(2):
        for w in range(4):
            for p in range(2):
                q = 2 * h + p
                rows[64 * h + 16 * w + 8 * p: 64 * h + 16 * w + 8 * p + 8] = blocks[8 * w: 8 * w + 8, q * kq: (q + 1) * kq]
    return rows


def b_tile_rows(basis_rows):
    """The B operand of one N tile (pack_block_basis_kernel with four phases): row 2 c + part = (re, im) of bin c."""
    rows = np.zeros((2 * basis_rows.shape[0], basis_rows.shape[1]))
    rows[0::2], rows[1::2] = basis_rows.real, basis_rows.imag
    return rows


def fragment(d, w, lane, n):
    """wgmma m64nNk16 accumulator fragment of thread `lane` of warp w: register 4 j + 2 s + e holds row
    16 w + lane / 4 + 8 s, column 8 j + 2 (lane % 4) + e of the warpgroup's 64 x N tile d."""
    regs = np.zeros(n // 2)
    for j in range(n // 8):
        for s in range(2):
            for e in range(2):
                regs[4 * j + 2 * s + e] = d[16 * w + lane // 4 + 8 * s, 8 * j + 2 * (lane % 4) + e]
    return regs


def poly_tile(blocks, basis_rows, tw_rows):
    """tcb_poly_tile on one (M tile, N tile): both warpgroups' two m64 x nb MMAs, the radix-4 butterfly on each
    thread's registers and the family stores.  tw_rows[q][c]: the twiddle of tile column c.  Returns the
    (128, 2 nb) accumulator tile the epilogue reads (quarter f = family f, f1 / f3 column-reversed; re columns, then
    im) and how many times each of its locations was written."""
    nb = basis_rows.shape[0]
    a, b = a_tile_rows(blocks), b_tile_rows(basis_rows)
    tile = np.zeros((128, 2 * nb))
    written = np.zeros((128, 2 * nb), dtype=int)
    for wg in range(2):
        half = b[wg * nb: (wg + 1) * nb]                     # MMA N = nb: this warpgroup's bins, re / im interleaved
        d = [a[64 * h: 64 * h + 64] @ half.T for h in range(2)]
        for w in range(4):
            for lane in range(32):
                acc = [fragment(d[h], w, lane, nb) for h in range(2)]
                r = 8 * w + lane // 4                        # block row
                for j in range(nb // 8):
                    c = wg * nb // 2 + 4 * j + lane % 4      # tile column (packed bin)
                    y = [acc[q >> 1][4 * j + 2 * (q & 1)] + 1j * acc[q >> 1][4 * j + 2 * (q & 1) + 1] for q in range(4)]
                    t = [y[q] * tw_rows[q][c] for q in range(4)]
                    a0, a1, b0, b1 = t[0] + t[2], t[0] - t[2], t[1] + t[3], t[1] - t[3]
                    fam = (a0 + b0, np.conj(a1 + 1j * b1), a1 - 1j * b1, np.conj(a0 - b0))
                    for f in range(4):
                        col = nb - 1 - c if f & 1 else c
                        tile[32 * f + r, col], tile[32 * f + r, nb + col] = fam[f].real, fam[f].imag
                        written[32 * f + r, col] += 1
                        written[32 * f + r, nb + col] += 1
    return tile, written


def emulate(x, n_fft, hop, B=1, nb=None, split=None):
    """framed_tcb_kernel<.., PH = 4> index by index: polyphase planes, the A tile's phase-interleaved rows, the
    butterfly on each thread's accumulator registers and its stores into family quarters (poly_tile), the
    per-family epilogue windows.  Returns the (B, F, T) STFT and the number of times each (b, bin, frame) was
    written."""
    assert hop % 128 == 0
    R = n_fft // hop
    FW = 33 - R
    F = n_fft // 2 + 1
    M = n_fft // 4
    Fp = M // 2 + 1
    kq = hop // 4
    pad = n_fft // 2
    L = x.shape[-1]
    T = (L + 2 * pad - n_fft) // hop + 1
    t_slots = (L + 2 * pad + hop - 1) // hop
    nv = B * t_slots
    # the pre-pass (TC_SPLIT_POLY4): position q kq + m of a block holds sample 4 m + q
    plane = np.zeros((nv + 40) * hop)
    for b in range(B):
        xp = np.pad(x[b], pad, mode="reflect")
        plane[b * t_slots * hop: b * t_slots * hop + len(xp)] = xp
    rows = plane.reshape(-1, hop)
    perm = np.array([4 * (r % kq) + r // kq for r in range(hop)])
    rows = rows[:, perm]
    nb = nb or choose_nb(Fp)
    split = (nb // 8) // 2 if split is None else split
    n_tiles = n_tiles_of(Fp, nb)
    p_rows = Fp + 2 + 128
    kp = np.arange(p_rows) - 1
    basis = np.exp(-2j * np.pi * np.outer(kp, np.arange(kq)) / M)
    basis[Fp + 2:] = 0
    tw = np.exp(-2j * np.pi * np.outer(np.arange(4), kp) / n_fft)     # [q][p]
    out = np.zeros((B, F, T), dtype=complex)
    written = np.zeros((B, F, T), dtype=int)
    for m_tile in range(-(-nv // FW)):
        m0 = m_tile * FW
        A = rows[m0: m0 + 32]
        for n_tile in range(n_tiles):
            n0 = n_tile * (nb - 2)
            tile, tile_written = poly_tile(A, basis[n0: n0 + nb], tw[:, n0: n0 + nb])
            assert (tile_written == 1).all()
            fam = [tile[32 * f: 32 * f + 32, :nb] + 1j * tile[32 * f: 32 * f + 32, nb:] for f in range(4)]
            for f in range(4):
                k_tile0, lo, hi = family_span(n_tile, f, nb, M, F)
                lo = max(lo, k_tile0)
                tws = [np.exp(-2j * np.pi * ((k_tile0 + 2 + i) % R) / R) for i in range(4)]
                for part, (cb, ce) in enumerate(((0, split), (split, nb // 8))):
                    w = np.zeros((32, 10), dtype=complex)
                    if cb > 0:
                        w[:, 8:10] = fam[f][:, 8 * cb - 2: 8 * cb]
                    for c in range(cb, ce):
                        w[:, 0:2] = w[:, 8:10]
                        w[:, 2:10] = fam[f][:, 8 * c: 8 * c + 8]
                        for e in range(8):
                            kk = k_tile0 + 8 * c - 2 + e
                            if (c == 0 and e < 2) or not lo <= kk < hi:
                                continue
                            assert poly4_range(kk, M, nb) == (f, n_tile)
                            zm, z0, zp = w[:, e], w[:, e + 1], w[:, e + 2]
                            X = np.zeros(32, dtype=complex)
                            for j in range(R):
                                om = np.exp(2j * np.pi * j / R)
                                V = 0.5 * z0 - 0.25 * om * zm - 0.25 / om * zp
                                X += tws[e & 3] ** j * np.concatenate([V[j:], np.zeros(j)])
                            for lane in range(FW):
                                g = m0 + lane
                                b, t = divmod(g, t_slots)
                                if g < nv and t < T:
                                    out[b, kk, t] = X[lane]
                                    written[b, kk, t] += 1
    return out, written


def fb_ranges(fb, nb):
    """Partial sums each filter of the fused filterbank receives at width nb: the number of distinct
    (family, tile) ranges over its support (fb_steps_kernel's replay)."""
    F = fb.shape[1]
    M = (F - 1) // 2
    counts = []
    for row in fb:
        nz = np.nonzero(row)[0]
        if len(nz):
            counts.append(len({poly4_range(k, M, nb) for k in range(nz.min(), nz.max() + 1)}))
    return counts


def choose_poly_tile(fb):
    """fb_steps_kernel's choice of nb for the four-phase kernel, or None: every filter <= 2 partial sums, then
    the fewest packed columns."""
    F = fb.shape[1]
    M = (F - 1) // 2
    best, best_cost = None, 1 << 30
    for nb in range(32, 136, 8):
        if max(fb_ranges(fb, nb), default=0) > 2:
            continue
        cost = n_tiles_of(M // 2 + 1, nb) * (nb + 6)
        if cost < best_cost:
            best, best_cost = nb, cost
    return best


if __name__ == "__main__":
    rng = np.random.default_rng(0)
    for n_fft, hop in ((2048, 512), (2048, 1024), (512, 128), (1024, 256), (4096, 1024)):
        x = rng.standard_normal(hop * 37 + 11)
        a, b = stft_dense(x, n_fft, hop), stft_poly(x, n_fft, hop)
        err = np.abs(a - b).max() / np.abs(a).max()
        print(f"spec  n_fft {n_fft} hop {hop}: max-rel {err:.2e}")
        assert err < 1e-12
    for n_fft, hop, L, B in ((2048, 512, 512 * 40 + 100, 2), (512, 128, 6000, 1), (1024, 512, 9000, 2)):
        x = rng.standard_normal((B, L))
        got, written = emulate(x, n_fft, hop, B)
        want = np.stack([stft_dense(x[b], n_fft, hop).T for b in range(B)])
        err = np.abs(got - want).max() / np.abs(want).max()
        print(f"kernel n_fft {n_fft} hop {hop} B {B}: max-rel {err:.2e}, written once: {(written == 1).all()}")
        assert err < 1e-12 and (written == 1).all()
