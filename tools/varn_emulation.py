#!/usr/bin/env python
"""CPU emulation of the per-K-block-width kernel's data flow (branch radix2-wip): the packed row
order of pack_basis_varn_kernel, the REAL host plan (nnab_debug_varn_plan through ctypes), the
mixed-width accumulation into one accumulator tile (garbage = NaN until the first MMA of a tile writes
a column) and the epilogue's column -> bin mapping, against the oracle's CQT1992v2.  Also runs the
split-K variant (chunks accumulate into a zeroed raw buffer).  No wgmma mechanics, only logic."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import nnaudio_oracle as oracle  # noqa: E402
import nnaudio_b200 as nb  # noqa: E402
from nnaudio_b200.features._common import tap_support  # noqa: E402
from varn_plan_check import plan as host_plan  # noqa: E402


def pack_rows(w_re, w_im, F, K):
    rows = 16 * ((F + 7) // 8)
    kpad = (K + 63) // 64 * 64
    packed = np.zeros((rows, kpad))
    for r in range(rows):
        f = (r >> 4) * 8 + (r & 7)
        part = (r >> 3) & 1
        if f < F:
            packed[r, :K] = w_re[f] if part == 0 else -w_im[f]
    return packed


def run(mod_kw, L, chunks):
    mod = nb.CQT1992v2(verbose=False, **mod_kw)
    kr, ki = mod.cqt_kernels_real.numpy()[:, 0].astype(np.float64), mod.cqt_kernels_imag.numpy()[:, 0].astype(np.float64)
    F, K = kr.shape
    kb, ke = tap_support((kr != 0) | (ki != 0))
    order, groups, cb = host_plan(kb, ke, F, K, chunks)
    packed = pack_rows(kr, ki, F, K)
    hop = mod.hop_length
    x = np.random.RandomState(1).standard_normal((1, L)).astype(np.float32)
    xp = oracle.pad_signal(x.astype(np.float64), K // 2, "reflect")[0]
    xp = np.concatenate((xp, np.zeros(64)))
    T = L // hop + 1
    frames = np.stack([xp[t * hop: t * hop + packed.shape[1]] for t in range(T)])     # (T, kpad)
    raw = np.zeros((T, 2, F)) if chunks > 1 else None
    out = np.zeros((T, 2, F))
    for c in range(len(cb) - 1):
        tmem = np.full((T, packed.shape[0]), np.nan)          # uninitialised accumulator columns
        first = True
        for i in range(cb[c], cb[c + 1]):
            n = 16 * groups[i]
            ks = slice(64 * order[i], 64 * order[i] + 64)
            part = frames[:, ks] @ packed[:n, ks].T
            if first:
                tmem[:, :n] = part                            # accumulate = 0: overwrites [0, N)
                first = False
            else:
                tmem[:, :n] += part
        n_groups = groups[cb[c]]                              # epilogue reads the chunk's widest block
        for gi in range(n_groups):
            re, im = tmem[:, 16 * gi: 16 * gi + 8], tmem[:, 16 * gi + 8: 16 * gi + 16]
            for j in range(8):
                f = 8 * gi + j
                if f < F:
                    assert not np.isnan(re[:, j]).any() and not np.isnan(im[:, j]).any(), (c, gi, j)
                    if raw is not None:
                        raw[:, 0, f] += re[:, j]
                        raw[:, 1, f] += im[:, j]
                    else:
                        out[:, 0, f], out[:, 1, f] = re[:, j], im[:, j]
    if raw is not None:
        out = raw
    got = (out[:, 0] + 1j * out[:, 1]).T[None]                 # (1, F, T)
    want = oracle.cqt1992v2(x, mod.cqt_kernels_real.numpy(), mod.cqt_kernels_imag.numpy(), mod.lenghts.numpy(),
                            hop, True, "reflect", "Complex", "convolutional", False, np.float64)
    want = want[..., 0] + 1j * want[..., 1]
    err = np.abs(got - want).max() / np.abs(want).max()
    print(f"{mod_kw} chunks {chunks}: {len(order)} blocks, widths {16 * groups.max()}..{16 * groups.min()}, "
          f"vs oracle {err:.1e}")
    assert err < 1e-12


if __name__ == "__main__":
    run(dict(sr=22050, fmin=220, n_bins=48, hop_length=256), 6000, 1)
    run(dict(sr=22050, fmin=220, n_bins=48, hop_length=256), 6000, 4)
    run(dict(sr=44100, n_bins=84, hop_length=512), 20000, 1)
    run(dict(sr=44100, n_bins=84, hop_length=512), 20000, 6)
