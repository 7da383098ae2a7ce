#!/usr/bin/env python
"""Executable spec of the block-partial STFT kernel's epilogue arithmetic (csrc/tcb_kernels.cu,
epilogue_tile_block), in float64 and replayed in float32 lane by lane.

tools/block_dft_emulation.py writes the frame as  X_t[k] = sum_{j<R} c_k^j V_j(Z_{t+j})[k]  with the Hann 3-tap
V_j(Z)[k] = 1/2 Z[k] - 1/4 w^j Z[k-1] - 1/4 w^-j Z[k+1].  Since c_k w = c_{k-1} and c_k / w = c_{k+1}, the same sum is

    S_t[k] = sum_{j<R} c_k^j Z_{t+j}[k]                   (the rectangular-window frame DFT)
    X_t[k] = 1/2 S_t[k] - 1/4 (S_t[k-1] + S_t[k+1])       (the Hann window as one 3-tap pass over S)

so the kernel sums frames once per packed column (each S feeds three output bins), with the twiddle of that
column's own bin.  R = 4 uses pair sums, Q_t = Z_t + c Z_{t+1} and S_t = Q_t + c^2 Q_{t+2}: 4 shuffles and 6 FMAs
per column.  The kernel keeps 2X = S[k] - 1/2 (S[k-1] + S[k+1]) and applies the exact 1/2 (1/4 on the power) in the
format tails.

`replay` follows one epilogue warp: 32 block rows (lanes) of a quarter's packed columns, 8-column chunks
[c_begin, c_end), the S of the last two columns carried into the next chunk, `__shfl_down_sync` with lanes past
31 reading their own value.  `order="v"` replays the previous kernel's per-bin V-term formula for comparison.
"""
import numpy as np

from block_dft_emulation import stft_dense


def stft_frame_sum_first(x, n_fft, hop):
    """The spec in float64: Z per block, S per bin, then the window on S."""
    R = n_fft // hop
    pad = n_fft // 2
    xp = np.pad(x, pad, mode="reflect")
    T = (len(xp) - n_fft) // hop + 1
    F = n_fft // 2 + 1
    k = np.arange(-1, F + 1)
    blocks = xp[: (T + R - 1) * hop].reshape(T + R - 1, hop)
    Z = blocks @ np.exp(-2j * np.pi * np.outer(k, np.arange(hop)) / n_fft).T
    c = np.exp(-2j * np.pi * k / R)
    S = sum((c ** j)[None, :] * Z[j: j + T] for j in range(R))
    return 0.5 * S[:, 1:-1] - 0.25 * (S[:, :-2] + S[:, 2:])


def block_dft(blocks, n_fft, bins):
    """Z_g[k] of hop-sized blocks at arbitrary integer bins k (float64)."""
    hop = blocks.shape[1]
    return blocks @ np.exp(-2j * np.pi * np.outer(bins, np.arange(hop)) / n_fft).T


def _twiddle(k, R):
    """c_k = e^{-2 pi i k / R} exactly: (-i)^k for R = 4, (-1)^k for R = 2."""
    m = k % R
    if R == 4:
        return (1.0, 0.0, -1.0, 0.0)[m], (0.0, -1.0, 0.0, 1.0)[m]
    return (1.0, -1.0)[m], 0.0


def replay(zq, k_tile0, c_begin, c_end, R, dtype=np.float64, order="s"):
    """One epilogue warp over a quarter: zq is (32, nb) complex, column j = bin k_tile0 + j - 1.  Returns
    {bin: X of the 32 lanes} for the outputs the chunks [c_begin, c_end) produce (lanes >= 33 - R are garbage)."""
    ft = np.dtype(dtype).type
    rnd = (lambda v: np.asarray(v, dtype=np.float64).astype(dtype).astype(np.float64))
    # fp32 arithmetic: every operation rounds once (an FMA's product is exact in float64)
    add = lambda a, b: rnd(a + b)                    # noqa: E731
    fma = lambda a, b, c: rnd(a * b + c)             # noqa: E731
    mul = lambda a, b: rnd(a * b)                    # noqa: E731

    def shfl(v, d):
        return np.concatenate([v[d:], v[32 - d:]]) if d else v  # lanes past 31 keep their own value

    zr = rnd(zq.real.astype(ft))
    zi = rnd(zq.imag.astype(ft))
    out = {}

    def frame_sum(j):
        cr, ci = _twiddle(k_tile0 + j - 1, R)
        c2 = 1.0 if (k_tile0 + j - 1) % 2 == 0 else -1.0
        ar, ai = zr[:, j], zi[:, j]
        z1r, z1i = shfl(ar, 1), shfl(ai, 1)
        if R == 4:
            qr = fma(cr, z1r, fma(-ci, z1i, ar))
            qi = fma(cr, z1i, fma(ci, z1r, ai))
            return fma(c2, shfl(qr, 2), qr), fma(c2, shfl(qi, 2), qi)
        return fma(c2, z1r, ar), fma(c2, z1i, ai)

    for c in range(c_begin, c_end):
        for e in range(8):
            o = 8 * c - 2 + e
            if c == 0 and e < 2:
                continue
            k = k_tile0 + o
            m, z0, p = o, o + 1, o + 2     # packed columns of bins k - 1, k, k + 1
            if order == "s":
                # the carried columns of a range's first chunk are seeded the same way (c_begin > 0)
                sm, s0, sp = frame_sum(m), frame_sum(z0), frame_sum(p)
                yr = fma(-0.5, add(sm[0], sp[0]), s0[0])
                yi = fma(-0.5, add(sm[1], sp[1]), s0[1])
                out[k] = 0.5 * (yr + 1j * yi)
            else:
                zmr, zmi = zr[:, m], zi[:, m]
                z0r, z0i = zr[:, z0], zi[:, z0]
                zpr, zpi = zr[:, p], zi[:, p]
                sr, si = add(zmr, zpr), add(zmi, zpi)
                ar, ai = mul(0.5, z0r), mul(0.5, z0i)
                qr, qi = _twiddle(k, R)
                q2 = 1.0 if k % 2 == 0 else -1.0
                v0r, v0i = fma(-0.25, sr, ar), fma(-0.25, si, ai)
                if R == 4:
                    dr, di = add(zmr, -zpr), add(zmi, -zpi)
                    v2r, v2i = shfl(fma(0.25, sr, ar), 2), shfl(fma(0.25, si, ai), 2)
                    v1r, v1i = shfl(fma(0.25, di, ar), 1), shfl(fma(-0.25, dr, ai), 1)
                    v3r, v3i = shfl(fma(-0.25, di, ar), 3), shfl(fma(0.25, dr, ai), 3)
                    t1r = add(mul(qr, v1r), -mul(qi, v1i))
                    t1i = add(mul(qr, v1i), mul(qi, v1r))
                    t3r = add(mul(qr, v3r), mul(qi, v3i))
                    t3i = add(mul(qr, v3i), -mul(qi, v3r))
                    xr = add(add(add(v0r, t1r), mul(q2, v2r)), t3r)
                    xi = add(add(add(v0i, t1i), mul(q2, v2i)), t3i)
                else:
                    v1r, v1i = shfl(fma(0.25, sr, ar), 1), shfl(fma(0.25, si, ai), 1)
                    xr, xi = fma(q2, v1r, v0r), fma(q2, v1i, v0i)
                out[k] = xr + 1j * xi
    return out


def frames_of(x, n_fft, hop):
    """Hop-sized blocks of the reflect-padded signal (zeros past its end, as in the kernel's planes), frames T."""
    pad = n_fft // 2
    xp = np.pad(x, pad, mode="reflect")
    T = (len(xp) - n_fft) // hop + 1
    n = -(-len(xp) // hop) + 32
    return np.pad(xp, (0, n * hop - len(xp))).reshape(n, hop), T


def quarter_check(x, n_fft, hop, k_tile0, nb, c_begin, c_end, m0, dtype=np.float64, order="s"):
    """Replay one warp on block rows m0 .. m0 + 31 and return (got, want) over its valid lanes and bins in [0, F)."""
    R = n_fft // hop
    blocks, T = frames_of(x, n_fft, hop)
    F = n_fft // 2 + 1
    zq = block_dft(blocks[m0: m0 + 32], n_fft, k_tile0 - 1 + np.arange(nb))
    got = replay(zq, k_tile0, c_begin, c_end, R, dtype, order)
    want = stft_dense(x, n_fft, hop)            # (T, F)
    lanes = [t for t in range(33 - R) if m0 + t < T]
    bins = sorted(k for k in got if 0 <= k < F)
    g = np.array([[got[k][t] for k in bins] for t in lanes])
    w = np.array([[want[m0 + t, k] for k in bins] for t in lanes])
    return g, w


if __name__ == "__main__":
    rng = np.random.default_rng(0)
    for n_fft, hop in ((2048, 512), (2048, 1024), (512, 128), (256, 64)):
        x = rng.standard_normal(hop * 37 + 11)
        a, b = stft_dense(x, n_fft, hop), stft_frame_sum_first(x, n_fft, hop)
        err = np.abs(a - b).max() / np.abs(a).max()
        print(f"spec   n_fft {n_fft} hop {hop}: max-rel {err:.2e}")
        assert err < 1e-12
    n_fft, hop, nb = 2048, 512, 88
    t = np.arange(hop * 60)
    x = np.sin(2 * np.pi * 440.0 / 22050 * t)
    for order in ("v", "s"):
        g, w = quarter_check(x, n_fft, hop, 0, nb, 0, nb // 8, 5, np.float32, order)
        print(f"fp32 replay ({order}-order), tone: max|d|/max|ref| {np.abs(g - w).max() / np.abs(w).max():.2e}")
