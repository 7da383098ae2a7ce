#!/usr/bin/env python
"""Line-by-line CPU emulation (float64) of framed_tcb_kernel's data flow: packed-bin tiles with a
2-bin overlap, 32-row warp quarters whose row origins are 33-R apart, the sliding 10-column window
of the epilogue, the per-tile twiddle tables and the lane shuffles.  Checked against the dense STFT."""
import numpy as np

from block_dft_emulation import stft_dense


def choose_nb(F):
    best, best_cost = 32, 1 << 30
    for nb in range(128, 31, -8):
        tiles = (F + nb - 3) // (nb - 2)
        cost = tiles * (nb + 6)
        if cost < best_cost:
            best, best_cost = nb, cost
    return best


def emulate(x, n_fft, hop, B=1):
    R = n_fft // hop
    FW = 33 - R
    F = n_fft // 2 + 1
    pad = n_fft // 2
    L = x.shape[-1]
    T = (L + 2 * pad - n_fft) // hop + 1
    t_slots = (L + 2 * pad + hop - 1) // hop
    nv = B * t_slots
    # split-signal plane viewed as (rows x hop)
    plane = np.zeros((nv + R + 2) * hop + 130 * hop)
    for b in range(B):
        xp = np.pad(x[b], pad, mode="reflect")
        plane[b * t_slots * hop: b * t_slots * hop + len(xp)] = xp
    rows = plane.reshape(-1, hop)
    nb = choose_nb(F)
    n_tiles = (F + nb - 3) // (nb - 2)
    p_rows = (n_tiles - 1) * (nb - 2) + nb
    k = np.arange(p_rows) - 1
    basis = np.exp(-2j * np.pi * np.outer(k, np.arange(hop)) / n_fft)
    basis[F + 2:] = 0
    out = np.zeros((B, F, T), dtype=complex)
    written = np.zeros((B, F, T), dtype=int)
    cta_tiles = -(-nv // (4 * FW))
    for ct in range(cta_tiles):
        for n_tile in range(n_tiles):
            n0 = n_tile * (nb - 2)
            k_tile0 = n0
            for quarter in range(4):
                m0 = ct * 4 * FW + quarter * FW
                A = rows[m0: m0 + 32]                       # one 32-row TMA box
                acc = A @ basis[n0: n0 + nb].T                # (32 rows, nb) accumulator columns (re + i im)
                tw = [np.exp(-2j * np.pi * ((k_tile0 + 2 + i) % R) / R) for i in range(4)]
                w = np.zeros((32, 10), dtype=complex)
                for c in range(nb // 8):
                    w[:, 0:2] = w[:, 8:10]
                    w[:, 2:10] = acc[:, 8 * c: 8 * c + 8]
                    for e in range(8):
                        if c == 0 and e < 2:
                            continue
                        kk = k_tile0 + 8 * c - 2 + e
                        zm, z0, zp = w[:, e], w[:, e + 1], w[:, e + 2]
                        X = np.zeros(32, dtype=complex)
                        for j in range(R):
                            omega = np.exp(2j * np.pi * j / R)
                            V = 0.5 * z0 - 0.25 * omega * zm - 0.25 / omega * zp
                            Vs = np.concatenate([V[j:], np.zeros(j)])      # shfl_down by j
                            X += tw[e & 3] ** j * Vs
                        if kk < F:
                            for lane in range(FW):
                                g = m0 + lane
                                b, t = divmod(g, t_slots)
                                if g < nv and t < T:
                                    out[b, kk, t] = X[lane]
                                    written[b, kk, t] += 1
    assert (written == 1).all(), (written.min(), written.max())
    return out


if __name__ == "__main__":
    rng = np.random.default_rng(0)
    for n_fft, hop, L, B in ((2048, 512, 512 * 70 + 100, 2), (512, 256, 16000, 1), (256, 64, 4000, 3),
                             (1024, 512, 30000, 2)):
        x = rng.standard_normal((B, L))
        got = emulate(x, n_fft, hop, B)
        want = np.stack([stft_dense(x[b], n_fft, hop).T for b in range(B)])
        err = np.abs(got - want).max() / np.abs(want).max()
        print(f"n_fft {n_fft} hop {hop} B {B} L {L}: nb {choose_nb(n_fft // 2 + 1)} max-rel {err:.2e}")
        assert err < 1e-12
