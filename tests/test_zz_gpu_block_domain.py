"""The block-partial STFT kernel (csrc/tcb_kernels.cu) across its dispatch domain (-m gpu): R = 2 and 4, the
one-phase (hop % 128 == 64) and four-phase (hop % 128 == 0) instances, n_fft from 128 to 32768, both pad modes and
center=False, fp32 and bf16 waveforms, the fused Mel epilogue (fast path, rolled MelRun path, widths with more
than two partial sums per filter), MFCC, the Gammatone operand planes, and batches of clips shorter than an M tile.

Every STFT output is held to a float64 ``np.fft.rfft`` of Hann-windowed frames (tests/block_domain.py, pinned
against the CPU oracle in tests/test_block_domain_host.py), every (bin, frame) cell must be written (the output
buffer starts as NaN), and the executed-MMA-flop counter must equal what the block-partial launch adds for the
instance the shape belongs to: a dense or SIMT fallback, or the other instance, gives a different count."""
import gc
import math
import warnings

import numpy as np
import pytest
import torch

import block_domain as bd
from conftest import record_error
from helpers import build, rel_errors, run_oracle
from nnaudio_b200 import _C

pytestmark = pytest.mark.gpu

FORMATS = ("Complex", "Magnitude", "Phase")
FMT_IDS = {"Complex": _C.FMT_COMPLEX, "Magnitude": _C.FMT_MAGNITUDE, "Phase": _C.FMT_PHASE_ANGLE}
PAD_IDS = {"reflect": _C.PAD_REFLECT, "constant": _C.PAD_CONSTANT}
# the bars test_gpu_parity.py holds the tensor-core routes to
BAR = 1e-4           # max|d| / max|ref| and ||d||_2 / ||ref||_2
BIN_BAR = 1e-3       # max over (clip, frame) of |d| per bin, over the rms of |ref| in that bin
PHASE_FLOOR = 0.01   # phases compared where |X| > PHASE_FLOOR max|X|
PHASE_BAR = 2e-3


def _flops(fn):
    """(fn(), executed MMA flops its launches added)."""
    _C.profile_read_exec_flops()
    _C.profile_enable(True)
    try:
        with torch.no_grad(), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            y = fn()
        torch.cuda.synchronize()
    finally:
        _C.profile_enable(False)
        _C.profile_read()
    return y, _C.profile_read_exec_flops()


def _noise(seed, B, L):
    return np.random.RandomState(seed).standard_normal((B, L)).astype(np.float32)


def _check_stft(y, X, fmt, test, case):
    """y: the kernel's (B, F, T[, 2]) output; X: the float64 complex reference."""
    y = y.cpu().numpy().astype(np.float64)
    mag = np.abs(X)
    if fmt == "Phase":
        mask = mag > PHASE_FLOOR * mag.max()
        d = np.abs(np.exp(1j * y) - np.exp(1j * np.angle(X)))[mask].max()
        record_error(test, case, phase_unit_max=float(d))
        assert d < PHASE_BAR, (case, d)
        return
    got = y[..., 0] + 1j * y[..., 1] if fmt == "Complex" else y
    want = X if fmt == "Complex" else mag
    d = np.abs(got - want)
    emax = float(d.max() / mag.max())
    el2 = float(np.linalg.norm(d) / np.linalg.norm(mag))
    # per bin: one wrong bin (a seam, a family edge, Nyquist) cannot hide under the global maximum
    per_bin = d.max(axis=(0, 2)) / np.sqrt((mag ** 2).mean(axis=(0, 2)))
    record_error(test, case, max_rel=emax, l2_rel=el2, worst_bin_rel=float(per_bin.max()))
    assert emax <= BAR and el2 <= BAR, (case, emax, el2)
    assert per_bin.max() <= BIN_BAR, (case, int(per_bin.argmax()), float(per_bin.max()))


def _run_stft_shape(run, n_fft, hop, B, L, center, pad_mode, test, seed, formats=FORMATS):
    """Every format of one shape: sentinel-filled output, flop count of the instance, float64 reference; then
    the bf16 waveform against its fp32 upcast (bitwise) at two thirds of the flops."""
    xn = _noise(seed, B, L)
    x = torch.from_numpy(xn).cuda()
    X = bd.ref_stft(xn, n_fft, hop, center, pad_mode)
    want_flops = bd.block_exec_flops(n_fft, hop, B, L, center)
    for fmt in formats:
        case = f"{n_fft}/{hop} B{B} L{L} {'center-' + pad_mode if center else 'no-center'} {fmt}"
        shape = X.shape + ((2,) if fmt == "Complex" else ())
        buf = torch.full(shape, float("nan"), device="cuda")

        def into():
            with _C.output_into(buf):
                return run(x, fmt)

        y, flops = _flops(into)
        assert y.data_ptr() == buf.data_ptr() and tuple(y.shape) == shape
        assert bool(torch.isfinite(y).all()), f"{case}: {int((~torch.isfinite(y)).sum())} cells never written"
        assert flops == want_flops, (case, flops, want_flops)
        _check_stft(y, X, fmt, test, case)

        xb = x.to(torch.bfloat16)
        yb, flops_b = _flops(lambda: run(xb, fmt))
        y32 = _flops(lambda: run(xb.float(), fmt))[0]
        assert torch.equal(yb, y32), (case, float((yb - y32).nan_to_num().abs().max()))
        assert flops_b == bd.block_exec_flops(n_fft, hop, B, L, center, passes=2), (case, flops_b)
        assert flops_b * 3 == want_flops * 2


def _module_run(mod):
    return lambda x, fmt: mod(x, output_format=fmt)


# ---------------------------------------------------------------- STFT shape matrix (modules) ----
@pytest.mark.parametrize("shape", bd.STFT_SHAPES, ids=lambda s: f"{s[0]}-{s[1]}")
def test_stft_block_domain(shape):
    n_fft, hop, B, L = shape
    mod = build("STFT", dict(n_fft=n_fft, hop_length=hop)).cuda()
    _run_stft_shape(_module_run(mod), n_fft, hop, B, L, True, "reflect", "block_domain_stft", seed=n_fft + hop)


@pytest.mark.parametrize("center,pad_mode", [(False, "reflect"), (True, "constant")], ids=["no-center", "constant"])
@pytest.mark.parametrize("n_fft,hop", bd.PAD_SHAPES)
def test_stft_block_domain_pad_modes(n_fft, hop, center, pad_mode):
    B, L = next((s[2], s[3]) for s in bd.STFT_SHAPES if s[:2] == (n_fft, hop))
    mod = build("STFT", dict(n_fft=n_fft, hop_length=hop, center=center, pad_mode=pad_mode)).cuda()
    _run_stft_shape(_module_run(mod), n_fft, hop, B, L, center, pad_mode, "block_domain_stft_pad",
                    seed=n_fft + 7)


# ------------------------------------------------- n_fft 16384 and 32768 (direct library call) ----
def _device_hann_basis(n_fft):
    """Full-size contiguous fp32 (F, n_fft) periodic-Hann DFT planes, built on the device in row blocks.  The
    block kernel reads only its own packed rows; the planes are complete so that no route reads outside them."""
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


@pytest.mark.parametrize("shape", bd.STFT_SHAPES_DIRECT, ids=lambda s: f"{s[0]}-{s[1]}")
def test_stft_block_domain_large_n_fft(shape):
    n_fft, hop, B, L = shape
    wcos, wsin = _device_hann_basis(n_fft)
    try:
        packed = _C.pack_basis_block(wcos, hop)

        def run(x, fmt):
            return _C.stft_forward(x, wcos, wsin, packed, n_fft, hop, True, _C.PAD_REFLECT, FMT_IDS[fmt], 0.0)

        _run_stft_shape(run, n_fft, hop, B, L, True, "reflect", "block_domain_stft_large", seed=n_fft)
    finally:
        del wcos, wsin
        packed = None
        gc.collect()
        torch.cuda.empty_cache()


# --------------------------------------------------------------------- batches of short clips ----
@pytest.mark.parametrize("n_fft,hop,B,L,center", [
    (512, 128, 37, 300, True),    # PH = 4, 29-row tiles, T = 3: every tile spans several clips
    (256, 64, 50, 200, True),     # PH = 1, 116-row tiles, T = 4
    (512, 128, 40, 512, False),   # T = 1
    (256, 64, 40, 256, False),    # T = 1
], ids=["ph4-T3", "ph1-T4", "ph4-T1", "ph1-T1"])
def test_stft_block_short_clip_batches(n_fft, hop, B, L, center):
    mod = build("STFT", dict(n_fft=n_fft, hop_length=hop, center=center)).cuda()
    _run_stft_shape(_module_run(mod), n_fft, hop, B, L, center, "reflect", "block_domain_short_clips",
                    seed=B * L)


# ----------------------------------------------------------------- fused filterbank and planes ----
# (class, constructor, input (B, L)); sr / n_fft / hop / bank per the dispatch branch each reaches
FBANK = {
    # rolled MelRun epilogue at PH = 4 (power != 2: sqrt, powf)
    "mel_ph4_power1": ("MelSpectrogram", dict(sr=16000, n_fft=512, hop_length=128, n_mels=40, power=1.0),
                       (2, 12345)),
    "mel_ph4_power1.5": ("MelSpectrogram", dict(sr=16000, n_fft=512, hop_length=128, n_mels=40, power=1.5),
                         (2, 12345)),
    # no width gives <= 2 partial sums per filter: default nb, fast path, more than two sums per filter
    "mel_ph4_no_width": ("MelSpectrogram", dict(sr=16000, n_fft=2048, hop_length=512, n_mels=40), (2, 40001)),
    # fused Mel on the one-phase instance, R = 4 and R = 2
    "mel_ph1_r4": ("MelSpectrogram", dict(sr=16000, n_fft=256, hop_length=64, n_mels=40), (3, 9001)),
    "mel_ph1_r2": ("MelSpectrogram", dict(sr=8000, n_fft=384, hop_length=192, n_mels=32), (2, 16001)),
    # MFCC tail on both instances
    "mfcc_ph4": ("MFCC", dict(sr=16000, n_fft=512, hop_length=128, n_mels=40, n_mfcc=13), (2, 16077)),
    "mfcc_ph1": ("MFCC", dict(sr=16000, n_fft=256, hop_length=64, n_mels=40, n_mfcc=13), (2, 12003)),
    # FMT_PLANES over 11 N tiles x 4 families, and on the one-phase R = 2 instance
    "gammatone_ph4_many_tiles": ("Gammatonegram", dict(sr=16000, n_fft=8192, hop_length=2048, n_bins=64),
                                 (2, 70001)),
    "gammatone_ph1_r2": ("Gammatonegram", dict(sr=8000, n_fft=384, hop_length=192, n_bins=32), (2, 16001)),
}


def _bank(cls, mod):
    if cls == "MFCC":
        return mod.melspec_layer.mel_basis
    return mod.gammatone_basis if cls == "Gammatonegram" else mod.mel_basis


@pytest.mark.parametrize("name", sorted(FBANK))
def test_filterbank_block_domain(name):
    cls, ctor, (B, L) = FBANK[name]
    n_fft, hop = ctor["n_fft"], ctor["hop_length"]
    mod = build(cls, ctor).cuda()
    xn = _noise(len(name) + L, B, L)
    x = torch.from_numpy(xn).cuda()
    y, flops = _flops(lambda: mod(x))
    fb = _bank(cls, mod).detach().cpu().numpy()
    T = y.shape[-1]
    if cls == "Gammatonegram":
        # the dense bank takes the operand-plane route: the block kernel at its default width writes
        # |X| ** power as bf16 planes, then a dense-kernel GEMM contracts them with the re-indexed bank
        want_flops = (bd.block_exec_flops(n_fft, hop, B, L, True)
                      + bd.planes_gemm_flops(n_fft, hop, B, T, fb.shape[0]))
        deterministic = True  # no atomics on this route
    else:
        nb, deterministic = bd.fbank_nb(fb, n_fft, hop)
        want_flops = bd.block_exec_flops(n_fft, hop, B, L, True, nb=nb)
        power = mod.melspec_layer.power if cls == "MFCC" else mod.power
        # the rolled MelRun path (power != 2) flushes each warp part's sums on its own, so the bound of two
        # partial sums per filter -- and with it run-to-run identical atomics -- holds for the fast path only
        deterministic = deterministic and power == 2.0
    assert flops == want_flops, (name, flops, want_flops)
    emax, el2 = rel_errors(y.cpu().numpy(), run_oracle(cls, mod, xn, {}))
    record_error("block_domain_filterbank", name, max_rel=emax, l2_rel=el2)
    assert emax < BAR and el2 < BAR, (name, emax, el2)
    if deterministic:
        again = _flops(lambda: mod(x))[0]
        assert torch.equal(y, again), name
