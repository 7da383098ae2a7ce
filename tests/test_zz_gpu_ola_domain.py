"""The overlap-add GEMM (the FMT_OLA route of csrc/tc_kernels.cu) and the FIR decimation adjoint across their shape
domain (-m gpu).  One tensor-core GEMM serves the input gradient of every framed transform
(``_C.framed_backward_input``), the gradient of trainable bases (``_C.framed_backward_weight``) and the inverse STFT
(``_C.istft_forward``); the shape matrices of tests/ola_domain.py name the edge each row is there for: frame
coverage (no overlap, gaps, unread tails), the reflect-padding adjoint, narrow and partial N tiles, M-tile seams,
K padding, split-K chunk counts, frames up to 24576 samples wide, and the CQT1992v2 module at kernel width 32768.

Every result is held to a float64 reference (tests/ola_domain.py, pinned against float64 autograd and the CPU oracle
in tests/test_ola_domain_host.py) globally and row by row, samples no frame reads must be exactly zero, and the
executed-MMA-flop counter of every overlap-add call must equal the launch model: a GEMM of another shape, or none,
gives a different count."""
import gc
import math
import warnings

import numpy as np
import pytest
import torch

import nnaudio_b200 as nb
import ola_domain as od
from conftest import record_error
from helpers import oracle
from nnaudio_b200 import _C

pytestmark = pytest.mark.gpu

PAD_IDS = {"reflect": _C.PAD_REFLECT, "constant": _C.PAD_CONSTANT}
BAR = 1e-4       # max|d| / max|ref| and ||d||_2 / ||ref||_2
ROW_BAR = 1e-3   # per clip (dX, iSTFT, FIR) or per bin (dW): max|d| over the rms of the reference row


def _flops(fn):
    """(fn(), executed MMA flops its launches added); fn may run autograd."""
    _C.profile_read_exec_flops()
    _C.profile_enable(True)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            y = fn()
        torch.cuda.synchronize()
    finally:
        _C.profile_enable(False)
        _C.profile_read()
    return y, _C.profile_read_exec_flops()


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _check(got, want, test, case, rows="clip"):
    """got / want: (R, N) with one row per clip (or bin); global and per-row bars."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (case, got.shape, want.shape)
    d = np.abs(got - want)
    emax = float(d.max() / np.abs(want).max())
    el2 = float(np.linalg.norm(d) / np.linalg.norm(want))
    per_row = d.max(axis=1) / np.sqrt((want ** 2).mean(axis=1))
    record_error(test, case, max_rel=emax, l2_rel=el2, **{f"worst_{rows}_rel": float(per_row.max())})
    assert emax <= BAR and el2 <= BAR, (case, emax, el2)
    assert per_row.max() <= ROW_BAR, (case, rows, int(per_row.argmax()), float(per_row.max()))


def _device_hann_basis(n_fft):
    """(F, n_fft) fp32 periodic-Hann DFT rows (wcos, wsin), built on the device in row blocks."""
    F = n_fft // 2 + 1
    wcos = torch.empty((F, n_fft), dtype=torch.float32, device="cuda")
    wsin = torch.empty_like(wcos)
    n = torch.arange(n_fft, device="cuda")
    hann = 0.5 - 0.5 * torch.cos((2.0 * math.pi / n_fft) * n.double())
    rows = max(1, (1 << 24) // n_fft)
    for k0 in range(0, F, rows):
        k = torch.arange(k0, min(F, k0 + rows), device="cuda")
        ang = (2.0 * math.pi / n_fft) * ((k[:, None] * n[None, :]) % n_fft).double()
        wcos[k0:k0 + rows] = (torch.cos(ang) * hann).float()
        wsin[k0:k0 + rows] = (torch.sin(ang) * hann).float()
    return wcos, wsin


def _dx_basis(row, rng):
    """(packed adjoint basis, K, F, reference bases (None, None for the FFT form of the Hann DFT))."""
    basis = row["basis"]
    if isinstance(basis, tuple):
        mod = nb.CQT1992v2(n_bins=basis[1], verbose=False, **od.CQT_BANK)
        w_re = mod.cqt_kernels_real[:, 0].numpy()
        w_im = mod.cqt_kernels_imag[:, 0].numpy()
        assert (2 * basis[1]) % 64 == 0
    elif basis == "perturbed":
        w_re, w_im = od.hann_dft_bases(row["K"])
        w_re = (w_re + 0.05 * rng.standard_normal(w_re.shape)).astype(np.float32)
        w_im = (w_im + 0.05 * rng.standard_normal(w_im.shape)).astype(np.float32)
    else:
        wcos, wsin = _device_hann_basis(row["K"])
        packed = _C.pack_adjoint_basis(wcos, wsin)
        torch.cuda.synchronize()
        return packed, row["K"], wcos.shape[0], None, None
    packed = _C.pack_adjoint_basis(torch.from_numpy(w_re).cuda(), torch.from_numpy(w_im).cuda())
    torch.cuda.synchronize()
    return packed, w_re.shape[1], w_re.shape[0], w_re, w_im


# ------------------------------------------------------------------------------------ input gradient ----
@pytest.mark.parametrize("name", sorted(od.DX_ROWS))
def test_input_gradient_domain(name):
    row = od.DX_ROWS[name]
    rng = np.random.RandomState(len(name) + 100)
    try:
        packed, K, F, w_re, w_im = _dx_basis(row, rng)
        hop, B, L, center, pad = row["hop"], row["B"], row["L"], row["center"], row["pad"]
        T = od.frames_of(L, K, hop, center)
        g = rng.standard_normal((B, F, T, 2)).astype(np.float32)
        dx, flops = _flops(lambda: _C.framed_backward_input(torch.from_numpy(g).cuda(), packed, K, hop, center,
                                                            PAD_IDS[pad], L))
        assert flops == od.ola_exec_flops(*od.dx_operands(B, T, K, F)), (name, flops)
        dx = dx.cpu().numpy()
        want = od.ref_backward_input(g, w_re, w_im, K, hop, center, pad, L)
        unread = ~od.read_mask(K, hop, center, pad, L, T)
        assert np.all(dx[:, unread] == 0.0), (name, int((dx[:, unread] != 0).sum()))
        _check(dx, want, "ola_domain_dx", f"{name} K{K} hop{hop} B{B} L{L}")
    finally:
        packed = None
        _free()


# ----------------------------------------------------------------------------------- weight gradient ----
@pytest.mark.parametrize("name", sorted(od.DW_ROWS))
def test_weight_gradient_domain(name):
    row = od.DW_ROWS[name]
    K, hop, B, L, center, pad, F = (row[k] for k in ("K", "hop", "B", "L", "center", "pad", "F"))
    rng = np.random.RandomState(len(name) + 200)
    T = od.frames_of(L, K, hop, center)
    x = rng.standard_normal((B, L)).astype(np.float32)
    g = rng.standard_normal((B, F, T, 2)).astype(np.float32)
    try:
        (dre, dim), flops = _flops(lambda: _C.framed_backward_weight(
            torch.from_numpy(g).cuda(), torch.from_numpy(x).cuda(), K, hop, center, PAD_IDS[pad]))
        M, F_out, K_gemm = od.dw_operands(B, T, K, F)
        assert flops == od.ola_exec_flops(M, F_out, K_gemm), (name, flops)
        got = np.concatenate((dre.cpu().numpy(), dim.cpu().numpy()))
        want_re, want_im = od.ref_backward_weight(g, x, K, hop, center, pad)
        _check(got, np.concatenate((want_re, want_im)), "ola_domain_dw",
               f"{name} K{K} hop{hop} B{B} frames{B * T} k_splits{od.dw_k_splits(K_gemm)}", rows="bin")
    finally:
        _free()


# ------------------------------------------------------------------- module regression at K = 32768 ----
def _cqt_module(fmin, width):
    mod = nb.CQT1992v2(sr=44100, fmin=fmin, n_bins=100, trainable=True, verbose=False).cuda()
    assert mod.kernel_width == width
    return mod


def test_cqt1992v2_gradients_at_kernel_width_32768():
    """loss.backward() through a trainable CQT1992v2 whose kernels are 32768 taps wide: x.grad and both kernel
    gradients against float64, one input-gradient and one weight-gradient GEMM."""
    mod = _cqt_module(32.7, 32768)
    K, hop = mod.kernel_width, mod.hop_length
    rng = np.random.RandomState(32768)
    x = rng.standard_normal((1, 44100)).astype(np.float32)
    xd = torch.from_numpy(x).cuda().requires_grad_(True)
    try:
        y = mod(xd, output_format="Complex")
        B, F, T, _ = y.shape
        W = rng.standard_normal(tuple(y.shape)).astype(np.float32)
        loss = (y * torch.from_numpy(W).cuda()).sum()
        _, flops = _flops(lambda: loss.backward())
        want_flops = (od.ola_exec_flops(*od.dx_operands(B, T, K, F))
                      + od.ola_exec_flops(*od.dw_operands(B, T, K, F)))
        assert flops == want_flops, (flops, want_flops)
        scale = mod._infer_args("Complex", "librosa")[1]["scale"].double().cpu().numpy()
        g = W.astype(np.float64) * scale[None, :, None, None]
        k_re = mod.cqt_kernels_real.detach()[:, 0].cpu().numpy()
        k_im = mod.cqt_kernels_imag.detach()[:, 0].cpu().numpy()
        want_dx = od.ref_backward_input(g, k_re, k_im, K, hop, mod.center, mod.pad_mode, x.shape[1])
        _check(xd.grad.cpu().numpy(), want_dx, "ola_domain_module", "CQT1992v2 K32768 x.grad")
        want_re, want_im = od.ref_backward_weight(g, x, K, hop, mod.center, mod.pad_mode)
        _check(mod.cqt_kernels_real.grad[:, 0].cpu().numpy(), want_re, "ola_domain_module",
               "CQT1992v2 K32768 d kernels_real", rows="bin")
        _check(mod.cqt_kernels_imag.grad[:, 0].cpu().numpy(), want_im, "ola_domain_module",
               "CQT1992v2 K32768 d kernels_imag", rows="bin")
    finally:
        del mod, xd
        _free()


def test_cqt1992v2_backward_at_kernel_width_65536_names_the_limit():
    """Kernels 65536 taps wide are beyond the overlap-add GEMM's N tiles: the backward refuses on the host, with
    the limit in the message (the forward runs)."""
    mod = _cqt_module(16.35, 65536)
    xd = torch.from_numpy(np.random.RandomState(65536).standard_normal((1, 70000)).astype(np.float32)).cuda()
    try:
        y = mod(xd.requires_grad_(True), output_format="Complex")
        with pytest.raises(RuntimeError, match=r"kernel width 65536 is above the overlap-add GEMM's limit of 32768"):
            y.sum().backward()
        torch.cuda.synchronize()
    finally:
        del mod, xd
        _free()


# ----------------------------------------------------------------------------------------- inverse STFT ----
def _device_dft_kernels(n_fft):
    """(kernel_cos, kernel_sin) (n_fft, n_fft) fp32: cos / sin(2 pi n f / n_fft), built on the device."""
    kc = torch.empty((n_fft, n_fft), dtype=torch.float32, device="cuda")
    ks = torch.empty_like(kc)
    f = torch.arange(n_fft, device="cuda")
    rows = max(1, (1 << 24) // n_fft)
    for n0 in range(0, n_fft, rows):
        n = torch.arange(n0, min(n_fft, n0 + rows), device="cuda")
        ang = (2.0 * math.pi / n_fft) * ((n[:, None] * f[None, :]) % n_fft).double()
        kc[n0:n0 + rows] = torch.cos(ang).float()
        ks[n0:n0 + rows] = torch.sin(ang).float()
    return kc, ks


@pytest.mark.parametrize("name", sorted(od.ISTFT_ROWS))
def test_istft_domain(name):
    row = od.ISTFT_ROWS[name]
    n_fft, hop, B, T, onesided, center = (row[k] for k in ("n_fft", "hop", "B", "T", "onesided", "center"))
    f_in = n_fft // 2 + 1 if onesided else n_fft
    rng = np.random.RandomState(len(name) + 300)
    X = rng.standard_normal((B, f_in, T, 2)).astype(np.float32)
    Xd = torch.from_numpy(X).cuda()
    length = od.length_of(row, T)
    try:
        if n_fft <= 2048:
            mod = nb.iSTFT(n_fft=n_fft, hop_length=hop, window=row["window"], center=center, verbose=False).cuda()
            win = mod.window_mask.reshape(-1).float().cpu().numpy()
            want = oracle.istft(X, mod.kernel_cos.cpu().numpy(), mod.kernel_sin.cpu().numpy(),
                                mod.window_mask.cpu().numpy(), hop, center=center, onesided=onesided, length=length)
            want_raw = od.ref_istft(X, win, hop, center, onesided, length)[1]

            def run():
                with torch.no_grad():
                    return mod(Xd, onesided=onesided, length=length)
        else:
            # the module's float64 design of (n_fft, n_fft) kernels is too large here: the same kernels are built
            # on the device and the reference is the FFT form of oracle.istft (pinned on the host)
            from scipy.signal import get_window

            win = get_window(row["window"], n_fft, fftbins=True).astype(np.float32)
            kc, ks = _device_dft_kernels(n_fft)
            packed = _C.pack_istft_basis(kc, ks, f_in, onesided)
            torch.cuda.synchronize()
            del kc, ks
            _free()
            wind = torch.from_numpy(win).cuda()
            want, want_raw = od.ref_istft(X, win, hop, center, onesided, length)

            def run():
                return _C.istft_forward(Xd, packed, wind, n_fft, hop, center, length)

        y, flops = _flops(run)
        assert flops == od.ola_exec_flops(*od.istft_operands(B, T, n_fft, f_in)), (name, flops)
        y = y.cpu().numpy().astype(np.float64)
        assert y.shape == want.shape, (name, y.shape, want.shape)
        wss = od.istft_wss(win, hop, T, center, length)
        case = f"{name} n_fft{n_fft} hop{hop} B{B} T{T}"
        # where the window sum-square is tiny the division is ill-conditioned: y itself is compared where it is
        # at least 1e-6 of its maximum, y * wss everywhere, and the undivided cells must equal the reference's
        good = wss >= 1e-6 * wss.max()
        _check(y[:, good], want[:, good], "ola_domain_istft", case)
        _check(y * wss, want * wss, "ola_domain_istft", case + " y*wss")
        tiny = wss <= 1e-10
        if tiny.any():
            d = float(np.abs(y[:, tiny] - want_raw[:, tiny]).max())
            assert d <= BAR * np.abs(want[:, good]).max(), (name, d)
    finally:
        mod = packed = None
        _free()


# ----------------------------------------------------------------------------------------- FIR adjoint ----
@pytest.mark.parametrize("name", sorted(od.FIR_ROWS), ids=str)
def test_fir_decimate_adjoint_domain(name):
    row = od.FIR_ROWS[name]
    taps, factor, L, B = row["taps"], row["factor"], row["L"], row["B"]
    rng = np.random.RandomState(taps + L)
    fir = (rng.standard_normal(taps) / math.sqrt(taps)).astype(np.float32)
    Ly = od.fir_out_len(L, taps, factor)
    g = rng.standard_normal((B, Ly)).astype(np.float32)
    dx, flops = _flops(lambda: _C.fir_decimate_adjoint(torch.from_numpy(g).cuda(), torch.from_numpy(fir).cuda(),
                                                       factor, L))
    assert flops == 0, "the FIR adjoint is a CUDA-core kernel: no tensor-core launch"
    want = od.ref_fir_adjoint(g, fir, factor, L)
    _check(dx.cpu().numpy(), want, "ola_domain_fir_adjoint", f"{name} factor{factor} B{B}")
