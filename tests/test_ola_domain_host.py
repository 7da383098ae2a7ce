"""CPU checks of tests/ola_domain.py, the float64 references and launch model that hold the overlap-add GEMM (input
gradient, weight gradient, inverse STFT) and the FIR decimation adjoint to account on the GPU
(tests/test_zz_gpu_ola_domain.py):

- the gradient references equal float64 torch autograd through the forward definition the CPU stand-ins use
  (tests/cpu_kernels.py), on scaled-down copies of every row class; the FFT form of the Hann frame gradient equals
  the dense product; the inverse reference equals oracle.istft; the FIR adjoint equals its index formula;
- the library's host plan (nnab_debug_ola_plan) agrees with the model on every row, takes frames up to 32768
  samples wide, refuses 65536, and the weight-gradient rows reach 1, an intermediate and the capped 64 K chunks;
- the entry points refuse frames above the limit on the host, before any device work."""
import ctypes

import numpy as np
import pytest
import torch

import cpu_kernels
import ola_domain as od
from helpers import oracle
from nnaudio_b200 import _C

PAD_IDS = {"reflect": _C.PAD_REFLECT, "constant": _C.PAD_CONSTANT}


def _autograd(x, w_re, w_im, hop, center, pad_mode, g):
    """(dx, d w_re, d w_im) of <g, Y> through cpu_kernels' float64 forward Y = (w_re . x_pad, -w_im . x_pad)."""
    x = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    w_re = torch.tensor(w_re, dtype=torch.float64, requires_grad=True)
    w_im = torch.tensor(w_im, dtype=torch.float64, requires_grad=True)
    y = cpu_kernels._framed(x, w_re, w_im, hop, center, PAD_IDS[pad_mode])
    return [t.numpy() for t in torch.autograd.grad(y, (x, w_re, w_im), torch.as_tensor(g))]


# scaled-down copies of the row classes: (basis, K, hop, B, L, center, pad)
SMALL = {
    "reflect": ("hann", 16, 4, 2, 50, True, "reflect"),
    "constant_odd_hop": ("hann", 16, 5, 2, 51, True, "constant"),
    "no_center_tail": ("hann", 16, 16, 2, 77, False, "reflect"),
    "gaps": ("hann", 16, 24, 2, 90, False, "reflect"),
    "gaps_centered": ("hann", 16, 24, 2, 90, True, "constant"),
    "reflect_overlap_L_pad_plus_2": ("hann", 16, 4, 3, 10, True, "reflect"),
    "reflect_L_pad_plus_1": ("hann", 32, 8, 1, 17, True, "reflect"),
    "T1": ("hann", 16, 4, 2, 16, False, "reflect"),
    "trainable": ("random", 24, 6, 2, 70, True, "reflect"),
    "trainable_gaps": ("random", 12, 20, 2, 70, True, "constant"),
}


@pytest.mark.parametrize("name", sorted(SMALL))
def test_gradient_references_equal_float64_autograd(name):
    basis, K, hop, B, L, center, pad = SMALL[name]
    rng = np.random.RandomState(len(name))
    if basis == "hann":
        w_re, w_im = od.hann_dft_bases(K)
    else:
        w_re, w_im = rng.standard_normal((2, 7, K))
    F = w_re.shape[0]
    T = od.frames_of(L, K, hop, center)
    x = rng.standard_normal((B, L))
    g = rng.standard_normal((B, F, T, 2))
    dx, dre, dim = _autograd(x, w_re, w_im, hop, center, pad, g)
    np.testing.assert_allclose(od.ref_backward_input(g, w_re, w_im, K, hop, center, pad, L), dx,
                               rtol=1e-12, atol=1e-12)
    if basis == "hann":
        np.testing.assert_allclose(od.ref_backward_input(g, None, None, K, hop, center, pad, L), dx,
                                   rtol=1e-10, atol=1e-10)
    want_re, want_im = od.ref_backward_weight(g, x, K, hop, center, pad)
    np.testing.assert_allclose(want_re, dre, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(want_im, dim, rtol=1e-12, atol=1e-12)
    # the samples no frame reads get no gradient from any upstream gradient
    mask = od.read_mask(K, hop, center, pad, L, T)
    assert np.all(dx[:, ~mask] == 0.0)
    if name in ("no_center_tail", "gaps"):
        assert not mask.all(), "the row must leave samples unread"


@pytest.mark.parametrize("n_fft", [8, 24, 100, 256, 300, 512, 2048])
def test_fft_frame_gradient_equals_dense_product(n_fft):
    rng = np.random.RandomState(n_fft)
    F = n_fft // 2 + 1
    g = rng.standard_normal((2, F, 5, 2))
    w_re, w_im = od.hann_dft_bases(n_fft)
    dense = od.frame_grad(g, w_re, w_im)
    fast = od.frame_grad(g, None, None)
    assert fast.shape == dense.shape == (2, 5, n_fft)
    np.testing.assert_allclose(fast, dense, rtol=0, atol=1e-10 * np.abs(dense).max())


def test_hann_bases_are_the_module_buffers():
    import nnaudio_b200 as nb

    for n_fft in (24, 256):
        mod = nb.STFT(n_fft=n_fft, hop_length=n_fft // 4, verbose=False)
        w_re, w_im = od.hann_dft_bases(n_fft)
        np.testing.assert_allclose(mod.wcos[:, 0].numpy(), w_re, atol=2e-7)
        np.testing.assert_allclose(mod.wsin[:, 0].numpy(), w_im, atol=2e-7)


@pytest.mark.parametrize("name", ["n100_hop25", "n300_hop150_two_sided", "n512_hop128_hamming",
                                  "n512_hop256_no_center", "n512_hop512_ones", "n512_hop768_gaps",
                                  "n512_length_short", "n512_length_long", "n256_T1_B70"])
def test_inverse_reference_equals_oracle(name):
    import nnaudio_b200 as nb

    row = od.ISTFT_ROWS[name]
    n_fft, hop, B, T, onesided = row["n_fft"], row["hop"], min(row["B"], 3), row["T"], row["onesided"]
    mod = nb.iSTFT(n_fft=n_fft, hop_length=hop, window=row["window"], center=row["center"], verbose=False)
    f_in = n_fft // 2 + 1 if onesided else n_fft
    X = np.random.RandomState(n_fft + hop).standard_normal((B, f_in, T, 2))
    length = od.length_of(row, T)
    want = oracle.istft(X, mod.kernel_cos.numpy(), mod.kernel_sin.numpy(), mod.window_mask.numpy(), hop,
                        center=row["center"], onesided=onesided, length=length)
    win = mod.window_mask.numpy().reshape(-1)
    y, y_raw = od.ref_istft(X, win, hop, row["center"], onesided, length)
    assert y.shape == want.shape == y_raw.shape
    wss = od.istft_wss(win, hop, T, row["center"], length)
    assert wss.shape == (y.shape[1],)
    # the module's kernels are fp32: agreement to their rounding
    np.testing.assert_allclose(y * wss, want * wss, rtol=0, atol=2e-5 * np.abs(want * wss).max())
    tiny = wss <= 1e-10
    np.testing.assert_allclose(y_raw[:, tiny], want[:, tiny], rtol=0, atol=1e-5)
    if name == "n512_hop768_gaps":
        assert tiny.any(), "the row must have overlap-add positions no frame reaches"


@pytest.mark.parametrize("taps,factor,L", [(9, 2, 9), (16, 3, 1025), (255, 4, 300), (256, 5, 1024),
                                           (1301, 2, 2000)])
def test_fir_adjoint_reference_equals_index_formula(taps, factor, L):
    """dx[i] = sum_j g[j] fir[i + half - factor j]: the formula fir_decimate_adjoint_kernel evaluates."""
    rng = np.random.RandomState(taps)
    fir = rng.standard_normal(taps)
    Ly = od.fir_out_len(L, taps, factor)
    g = rng.standard_normal((2, Ly))
    half = (taps - 1) // 2
    want = np.zeros((2, L))
    for i in range(L):
        for j in range(Ly):
            k = i + half - factor * j
            if 0 <= k < taps:
                want[:, i] += g[:, j] * fir[k]
    np.testing.assert_allclose(od.ref_fir_adjoint(g, fir, factor, L), want, rtol=1e-12, atol=1e-12)


# ----------------------------------------------------------------------------------------- launch model ----
def _cqt_width(n_bins):
    import nnaudio_b200 as nb

    return nb.CQT1992v2(n_bins=n_bins, verbose=False, **od.CQT_BANK).kernel_width


def _dx_operands(row):
    if isinstance(row["basis"], tuple):
        K, F = _cqt_width(row["basis"][1]), row["basis"][1]
    else:
        K, F = row["K"], row["K"] // 2 + 1
    return od.dx_operands(row["B"], od.frames_of(row["L"], K, row["hop"], row["center"]), K, F)


def _plan_rows():
    """(name, M, F_out, K_gemm) of every overlap-add GEMM the GPU matrix launches."""
    out = [("dx:" + n, *_dx_operands(r)) for n, r in od.DX_ROWS.items()]
    for n, r in od.DW_ROWS.items():
        out.append(("dw:" + n, *od.dw_operands(r["B"], od.frames_of(r["L"], r["K"], r["hop"], r["center"]), r["K"],
                                               r["F"])))
    for n, r in od.ISTFT_ROWS.items():
        f_in = r["n_fft"] // 2 + 1 if r["onesided"] else r["n_fft"]
        out.append(("istft:" + n, *od.istft_operands(r["B"], r["T"], r["n_fft"], f_in)))
    return out


def test_host_plan_agrees_with_the_model_on_every_row():
    splits = {}
    for name, M, F_out, K_gemm in _plan_rows():
        p = _C.ola_plan(F_out, K_gemm, M, od.MAX_SPLITS)
        bn = od.istft_bn(F_out)
        assert p["supported"], name
        assert (p["bn"], p["n_tiles"]) == (bn, -(-F_out // bn)), (name, p)
        assert p["exec_flops"] == od.ola_exec_flops(M, F_out, K_gemm), (name, p)
        assert p["k_splits"] == od.ola_k_splits(K_gemm), (name, p)
        if name.startswith("dw:"):
            assert p["k_splits"] == od.dw_k_splits(K_gemm), (name, p)
        splits.setdefault(name.split(":")[0], set()).add(p["k_splits"])
    dw = splits["dw"]
    assert 1 in dw and 64 in dw and any(1 < s < 64 for s in dw), dw
    # frames of 16384 and 24576 samples sum 2F > 4096 products per output: chunked too
    assert max(splits["dx"]) == 7 and max(splits["istft"]) == 5, splits


def test_host_plan_width_limit():
    assert _C.OLA_MAX_WIDTH == od.MAX_WIDTH
    for F_out in (16384, 24576, 32768 - 1, 32768):
        assert _C.ola_plan(F_out, 256, 100)["supported"], F_out
    for F_out in (32768 + 1, 32768 + 256, 65536):
        p = _C.ola_plan(F_out, 256, 100)
        assert not p["supported"] and p["n_tiles"] > 128, (F_out, p)
    # the forward's N-tile bound (2 F columns in tiles of up to 256) would have refused these widths
    assert -(-2 * 24576 // 256) > 128 and -(-2 * 32768 // 256) > 128
    # chunks of at most 64 k-blocks, at most the caller's hint of them (none below 2: one chunk)
    for K_gemm, hint, want in ((64, 64, 1), (4096, 64, 1), (4097, 64, 2), (64 * 65, 64, 2), (64 * 65, 0, 1),
                               (64 * 64 * 70, 64, 64), (64 * 64 * 70, 10, 10), (64 * 64 * 70, 1, 1)):
        assert _C.ola_plan(256, K_gemm, 10, hint)["k_splits"] == want, (K_gemm, hint)


def test_flop_model_by_hand():
    # dX, n_fft 512 / hop 128, 2 clips of 8000: T = 63, M = 126 -> 128; N 512 (two 256 tiles); K = 514 -> 576
    assert od.ola_exec_flops(*_dx_operands(od.DX_ROWS["hann_512_128"])) == 6 * 128 * 512 * 576 == 226492416
    # dX, n_fft 24 / hop 6, 2 clips of 3000: T = 501, M = 1002 -> 1024; one 32-wide tile; K = 26 -> 64
    assert od.ola_exec_flops(*_dx_operands(od.DX_ROWS["hann_24"])) == 6 * 1024 * 32 * 64 == 12582912
    # dW, 4 clips of 65536 at hop 64: 4100 frames -> gpad 4160; M = 2 x 129 = 258 -> 384; N 256
    r = od.DW_ROWS["gpad_4160"]
    ops = od.dw_operands(r["B"], od.frames_of(r["L"], r["K"], r["hop"], r["center"]), r["K"], r["F"])
    assert ops == (258, 256, 4160)
    assert od.ola_exec_flops(*ops) == 6 * 384 * 256 * 4160 == 2453667840
    assert od.dw_k_splits(4160) == 2 and od.dw_k_splits(4096) == 1 and od.dw_k_splits(64) == 1
    # iSTFT two-sided n_fft 300, 2 x 30 frames: M 60 -> 128; N 300 -> 512 (256-wide tiles); K 600 -> 640
    assert od.ola_exec_flops(*od.istft_operands(2, 30, 300, 300)) == 6 * 128 * 512 * 640 == 251658240


def test_entry_points_refuse_wide_frames_on_the_host():
    """Above 32768 output samples per frame the three callers return NNAB_EUNSUPPORTED before any device work
    (here, with no device, a call that passed the check would report a CUDA or architecture error instead)."""
    lib = _C.lib()
    P = ctypes.c_void_p
    p = P(256)  # never dereferenced on the host
    B, L, hop, F = 1, 70000, 512, 84

    def dx(K):
        T = (L + 2 * (K // 2) - K) // hop + 1
        return lib.nnab_framed_backward_input(p, B, F, T, p, K, hop, 1, 0, p, L, p, 1 << 40, None)

    def dw(K):
        T = (L + 2 * (K // 2) - K) // hop + 1
        return lib.nnab_framed_backward_weight(p, p, B, L, L, F, T, K, hop, 1, 0, p, p, 1 << 40, None)

    def istft(n_fft):
        return lib.nnab_istft_forward(p, B, n_fft // 2 + 1, 4, p, p, n_fft, n_fft // 4, 1, -1, p, 0, p, 1 << 40,
                                      None)

    for call in (dx, dw, istft):
        assert call(65536) == _C.EUNSUPPORTED, call.__name__
        assert call(32768 + 16) == _C.EUNSUPPORTED, call.__name__
        if not torch.cuda.is_available():
            assert call(32768) in (-3, -4), call.__name__  # NNAB_EARCH / NNAB_ECUDA: past the width check
