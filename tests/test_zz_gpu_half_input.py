"""bfloat16 / float16 waveforms on the GPU (-m gpu).  The tensor-core pre-pass converts every sample to
fp32 exactly before the bf16 hi/lo split, so a 16-bit waveform builds the planes its float32 upcast builds,
and every tensor-core route must return the upcast input's result bit for bit.  The block-partial STFT
kernel runs a bf16 waveform with two MMA passes instead of three (the lo plane is zero): the same
accumulators, two thirds of the executed MMA flops.  The forward wrappers run with ``strict_dtype=True``
here, so an upcast retry on the host cannot hide a route that lacks 16-bit input."""
import functools
import warnings

import numpy as np
import pytest
import torch

from helpers import CASES, build, case_input, rel_errors, run_oracle
from nnaudio_b200 import _C

pytestmark = pytest.mark.gpu

WAVE_CALLS = ("stft_forward", "stft_filterbank_forward", "mfcc_forward", "cqt1992v2_forward",
              "cqt_pyramid_forward")
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}


@pytest.fixture
def strict(monkeypatch):
    for name in WAVE_CALLS:
        monkeypatch.setattr(_C, name, functools.partial(getattr(_C, name), strict_dtype=True))


def _run(mod, x, kw):
    with torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        y = mod(x, **kw)
    torch.cuda.synchronize()
    return y


def _cuda(xn, dtype):
    return torch.from_numpy(np.ascontiguousarray(xn)).cuda().to(dtype)


@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_16bit_waveform_equals_its_float32_upcast_bitwise(case, dtype, strict):
    """Every golden configuration of every waveform module, on the routes auto-selection picks."""
    cid, cls, ctor, inp, fwds = case
    mod = build(cls, ctor).cuda()
    x = _cuda(case_input(cid, inp), DTYPES[dtype])
    for kw in fwds:
        y = _run(mod, x, kw)
        want = _run(mod, x.float(), kw)
        assert y.dtype == torch.float32 and y.shape == want.shape
        assert torch.equal(y, want), (kw, float((y - want).abs().max()))


# block-partial kernel routes: (class, constructor, input shape, forward kwargs)
TCB = {
    "mel_cfg2": ("MelSpectrogram", dict(sr=22050, n_fft=2048, hop_length=512, n_mels=128), (2, 22050), {}),
    "stft_r4_magnitude": ("STFT", dict(n_fft=2048, hop_length=512), (2, 22050), dict(output_format="Magnitude")),
    "stft_r4_complex": ("STFT", dict(n_fft=2048, hop_length=512), (2, 22050), dict(output_format="Complex")),
    "stft_r4_phase": ("STFT", dict(n_fft=2048, hop_length=512), (2, 22050), dict(output_format="Phase")),
    "stft_r2_magnitude": ("STFT", dict(n_fft=512, hop_length=256), (2, 16000), dict(output_format="Magnitude")),
    "stft_r2_complex": ("STFT", dict(n_fft=512, hop_length=256), (2, 16000), dict(output_format="Complex")),
    "stft_r2_phase": ("STFT", dict(n_fft=512, hop_length=256), (2, 16000), dict(output_format="Phase")),
    "mfcc": ("MFCC", dict(sr=16000), (3, 16000), {}),
    "gammatone_planes": ("Gammatonegram", dict(sr=22050, n_fft=2048, hop_length=512, n_bins=64), (5, 30000), {}),
    # 3 x 83 block rows: three M tiles, the last one partial (tests/test_zz_gpu_tcb_grid.py)
    "stft_partial_m_tile": ("STFT", dict(n_fft=1024, hop_length=256, sr=16000), (3, 20000),
                            dict(output_format="Magnitude")),
    "mel_partial_m_tile": ("MelSpectrogram", dict(sr=16000, n_fft=1024, hop_length=256, n_mels=64), (3, 20000), {}),
}


def _flops(mod, x, kw):
    _C.profile_read_exec_flops()
    _C.profile_enable(True)
    try:
        y = _run(mod, x, kw)
    finally:
        _C.profile_enable(False)
        _C.profile_read()
    return y, _C.profile_read_exec_flops()


@pytest.mark.parametrize("name", sorted(TCB))
def test_bf16_runs_two_mma_passes_on_the_block_partial_kernel(name, strict):
    cls, ctor, shape, kw = TCB[name]
    mod = build(cls, ctor).cuda()
    x = _cuda(np.random.RandomState(3).standard_normal(shape).astype(np.float32), torch.bfloat16)
    y, f16 = _flops(mod, x, kw)
    want, f32 = _flops(mod, x.float(), kw)
    assert torch.equal(y, want), float((y - want).abs().max())
    assert f32 > 0
    if cls == "Gammatonegram":
        # its second launch (operand planes x bank) is a dense-kernel GEMM on fp32 planes: 3 passes either way
        assert f16 < f32
    else:
        assert f16 == pytest.approx(f32 * 2.0 / 3.0, rel=1e-12)


# one configuration per module for the oracle check: (class, constructor, input shape, forward kwargs)
ORACLE = [
    ("STFT", dict(n_fft=512, hop_length=256, sr=16000), (1, 16000), dict(output_format="Complex")),
    ("STFT", dict(n_fft=512, win_length=400, hop_length=128, window="hamming"), (2, 4000),
     dict(output_format="Magnitude")),
    ("MelSpectrogram", dict(sr=22050, n_fft=2048, hop_length=512, n_mels=128), (2, 22050), {}),
    ("MFCC", dict(sr=16000), (2, 16000), {}),
    ("Gammatonegram", dict(sr=22050, n_fft=1024, n_bins=32, hop_length=256), (2, 8000), {}),
    ("CQT1992v2", dict(sr=22050, fmin=220, n_bins=48, hop_length=256), (2, 16000), dict(output_format="Complex")),
    ("CQT2010v2", dict(sr=22050, n_bins=84), (1, 32768), dict(output_format="Magnitude")),
    ("CQT2010v2", dict(sr=44100, n_bins=72, fmin=32.7), (1, 40000), dict(output_format="Complex")),
    ("VQT", dict(sr=22050, gamma=5, n_bins=60), (1, 32768), dict(output_format="Complex")),
    ("CQT1992", dict(sr=22050, fmin=220, n_bins=60), (1, 16384), dict(output_format="Magnitude")),
    ("CQT2010", dict(sr=22050, n_bins=84), (1, 32768), dict(output_format="Magnitude")),
]


@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("case", ORACLE, ids=[f"{c[0]}-{i}" for i, c in enumerate(ORACLE)])
def test_16bit_waveform_matches_the_oracle_on_its_samples(case, dtype, strict):
    cls, ctor, shape, kw = case
    mod = build(cls, ctor).cuda()
    x = _cuda(np.random.RandomState(4).standard_normal(shape).astype(np.float32), DTYPES[dtype])
    y = _run(mod, x, kw)
    emax, el2 = rel_errors(y.cpu().numpy(), run_oracle(cls, mod, x.float().cpu().numpy(), kw))
    assert emax < 1e-4 and el2 < 1e-4, (emax, el2)


@pytest.mark.parametrize("cls", ["CFP", "Combined_Frequency_Periodicity"])
def test_cfp_16bit_waveform_equals_its_float32_upcast(cls):
    mod = build(cls, {}).cuda()
    x = _cuda(np.random.RandomState(40).standard_normal((2, 16000)).astype(np.float32), torch.bfloat16)
    y, want = _run(mod, x, {}), _run(mod, x.float(), {})
    for a, b in zip(y if isinstance(y, tuple) else (y,), want if isinstance(want, tuple) else (want,)):
        assert a.dtype == torch.float32 and torch.equal(a, b)


SIMT = [
    ("STFT", dict(n_fft=512, hop_length=128), (2, 4000), dict(output_format="Magnitude")),
    ("MelSpectrogram", dict(sr=16000, n_fft=512, hop_length=128, n_mels=40), (2, 8000), {}),
    ("MFCC", dict(sr=16000), (2, 16000), {}),
    ("CQT1992v2", dict(sr=22050, fmin=220, n_bins=48, hop_length=256), (1, 16000), {}),
    ("CQT2010v2", dict(sr=22050, n_bins=84), (1, 32768), {}),
]


@pytest.mark.parametrize("case", SIMT, ids=[c[0] for c in SIMT])
def test_forced_simt_path_upcasts_a_16bit_waveform(case, monkeypatch):
    """The SIMT kernels read fp32 samples: the library refuses the 16-bit waveform before launching
    anything, the wrapper upcasts and calls again."""
    cls, ctor, shape, kw = case
    monkeypatch.setenv("NNAUDIO_B200_PATH", "simt")
    mod = build(cls, ctor).cuda()
    xn = np.random.RandomState(6).standard_normal(shape).astype(np.float32)
    x = _cuda(xn, torch.float16)
    y = _run(mod, x, kw)
    assert torch.equal(y, _run(mod, x.float(), kw))
    emax, el2 = rel_errors(y.cpu().numpy(), run_oracle(cls, mod, x.float().cpu().numpy(), kw))
    assert emax < 1e-4 and el2 < 1e-4, (emax, el2)
    for name in WAVE_CALLS:
        monkeypatch.setattr(_C, name, functools.partial(getattr(_C, name), strict_dtype=True))
    with pytest.raises(RuntimeError, match=r"status -6"):
        _run(mod, x, kw)


def test_trainable_mel_gradient_of_a_bf16_waveform():
    mod = build("MelSpectrogram", dict(sr=16000, n_fft=512, hop_length=128, n_mels=40, trainable_mel=True)).cuda()
    xn = np.random.RandomState(8).standard_normal((2, 8000)).astype(np.float32)
    xb = _cuda(xn, torch.bfloat16).requires_grad_()
    x32 = xb.detach().float().requires_grad_()
    y = mod(xb)
    w = torch.randn(y.shape, generator=torch.Generator().manual_seed(9)).cuda()
    (y * w).sum().backward()
    (mod(x32) * w).sum().backward()
    assert xb.grad.dtype == torch.bfloat16
    want = x32.grad.to(torch.bfloat16).float()
    got = xb.grad.float()
    # (a one-ulp bf16 rounding difference stays far below the bar in the l2 norm)
    assert float((got - want).norm() / want.norm()) < 1e-4
    assert float((got - want).abs().max()) <= float(want.abs().max()) * 2.0 ** -7
