"""bfloat16 / float16 waveforms on the CPU: which sample type each module hands to the library.  The
forward entry points take a 16-bit waveform as is (include/nnab.h NNAB_DTYPE_*), so on the inference
path every waveform module must pass it on without a float32 copy; the differentiable branches run the
fp32 training kernels and upcast once, so autograd returns ``x.grad`` in the input's dtype; float64 and
integer waveforms are still refused.  The float64 stand-ins of tests/cpu_kernels.py take the place of the
C wrappers, each behind a recorder that keeps the dtype it was given and refuses what the real wrapper
refuses.  The kernels are checked on the GPU by tests/test_zz_gpu_half_input.py."""
import ctypes
import warnings

import numpy as np
import pytest
import torch

from helpers import build
import cpu_kernels

from nnaudio_b200 import _C

WAVE_CALLS = ("stft_forward", "stft_filterbank_forward", "mfcc_forward", "cqt1992v2_forward",
              "cqt_pyramid_forward")

# one small configuration per waveform module: (class, constructor, input shape, forward kwargs)
MODULES = [
    ("STFT", dict(n_fft=512, hop_length=128, sr=16000), (2, 4000), dict(output_format="Complex")),
    ("MelSpectrogram", dict(sr=16000, n_fft=512, hop_length=128, n_mels=40), (2, 4000), {}),
    ("MFCC", dict(sr=16000, n_fft=512, hop_length=160, n_mels=40, n_mfcc=13), (2, 4000), {}),
    ("Gammatonegram", dict(sr=22050, n_fft=1024, n_bins=32, hop_length=256), (1, 5000), {}),
    ("CQT1992v2", dict(sr=22050, fmin=440, n_bins=24, hop_length=256), (1, 6000), dict(output_format="Complex")),
    ("CQT", dict(sr=22050, fmin=440, n_bins=24, hop_length=256), (1, 6000), {}),
    ("CQT2010v2", dict(sr=22050, n_bins=36, fmin=110, earlydownsample=False), (1, 8192), {}),
    ("VQT", dict(sr=22050, gamma=5, n_bins=24, fmin=220), (1, 8192), {}),
    ("CQT1992", dict(sr=16000, fmin=440, n_bins=24, hop_length=256), (1, 6000), {}),
    ("CQT2010", dict(sr=22050, n_bins=24, fmin=220), (1, 8192), {}),
]
IDS = [m[0] for m in MODULES]


@pytest.fixture
def calls(monkeypatch):
    """Install the stand-ins; returns the list of waveform dtypes the forward calls received."""
    cpu_kernels.install(monkeypatch)
    seen = []

    def recorded(fn):
        def call(x, *args, **kwargs):
            if x.dtype not in _C._WAVE_DTYPES:  # what _C._dev_wave refuses
                raise RuntimeError(f"x must be float32, bfloat16 or float16, got {x.dtype}")
            seen.append(x.dtype)
            return fn(x, *args, **kwargs)
        return call

    for name in WAVE_CALLS:
        monkeypatch.setattr(_C, name, recorded(getattr(cpu_kernels, name)))

    def fir_decimate(x, fir, factor):  # the pyramid's training path: fp32 only, like _C._rows
        if x.dtype != torch.float32:
            raise RuntimeError(f"x must be float32, got {x.dtype}")
        return cpu_kernels.fir_decimate(x, fir, factor)

    monkeypatch.setattr(_C, "fir_decimate", fir_decimate)
    return seen


def _module(case, trainable=False):
    cls, ctor, shape, kw = case
    ctor = dict(ctor)
    if trainable:
        ctor[{"STFT": "trainable", "MelSpectrogram": "trainable_mel", "MFCC": "trainable_mel",
              "Gammatonegram": "trainable_bins"}[cls]] = True
    return build(cls, ctor)


def _input(shape, dtype, seed=0):
    return torch.from_numpy(np.random.RandomState(seed).standard_normal(shape).astype(np.float32)).to(dtype)


def _run(mod, x, kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return mod(x, **kw)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("case", MODULES, ids=IDS)
def test_inference_path_hands_the_16bit_waveform_to_the_library(case, dtype, calls):
    mod = _module(case)
    x = _input(case[2], dtype)
    with torch.no_grad():
        y = _run(mod, x, case[3])
        assert calls and set(calls) == {dtype}, calls
        calls.clear()
        want = _run(mod, x.float(), case[3])
    assert set(calls) == {torch.float32}
    assert y.dtype == torch.float32
    assert torch.equal(y, want)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("case", MODULES[:4] + [MODULES[4], MODULES[6], MODULES[8]],
                         ids=IDS[:4] + [IDS[4], IDS[6], IDS[8]])
def test_autograd_path_upcasts_once_and_returns_the_input_dtype_gradient(case, dtype, calls):
    mod = _module(case)
    x = _input(case[2], dtype).requires_grad_()
    y = _run(mod, x, case[3])
    assert calls and set(calls) == {torch.float32}, calls
    w = torch.from_numpy(np.random.RandomState(1).standard_normal(tuple(y.shape)).astype(np.float32))
    (y * w).sum().backward()
    assert x.grad.dtype == dtype

    x32 = x.detach().float().requires_grad_()
    (_run(mod, x32, case[3]) * w).sum().backward()
    assert torch.equal(x.grad, x32.grad.to(dtype))


@pytest.mark.parametrize("case", MODULES[:4], ids=IDS[:4])
def test_trainable_bases_take_the_autograd_path_with_16bit_input(case, calls):
    mod = _module(case, trainable=True)
    y = _run(mod, _input(case[2], torch.bfloat16), case[3])
    assert set(calls) == {torch.float32}
    assert y.dtype == torch.float32 and y.requires_grad


@pytest.mark.parametrize("dtype", [torch.float64, torch.int16], ids=["float64", "int16"])
@pytest.mark.parametrize("case", MODULES, ids=IDS)
def test_other_dtypes_are_still_refused(case, dtype, calls):
    mod = _module(case)
    x = (_input(case[2], torch.float32) * 1000).to(dtype)
    with torch.no_grad(), pytest.raises(RuntimeError, match="float32"):
        _run(mod, x, case[3])
    if dtype.is_floating_point:
        with pytest.raises(RuntimeError, match="float32"):
            _run(mod, x.requires_grad_(), case[3])


@pytest.mark.parametrize("cls", ["CFP", "Combined_Frequency_Periodicity"])
def test_cfp_upcasts_a_16bit_waveform_on_the_host(cls, calls):
    mod = build(cls, dict(fr=3, g=[0.3, 0], window_size=1500))
    x = _input((1, 7000), torch.bfloat16)
    with torch.no_grad():
        y = mod(x)
        want = mod(x.float())
    assert set(calls) == {torch.float32}
    for a, b in zip(y if isinstance(y, tuple) else (y,), want if isinstance(want, tuple) else (want,)):
        assert a.dtype == torch.float32 and torch.equal(a, b)
    with torch.no_grad(), pytest.raises(RuntimeError, match="float32"):
        mod(x.double())


def test_wave_checks_device_and_dtype():
    with pytest.raises(TypeError):
        _C._dev_wave(np.zeros(4, np.float32), "x")
    with pytest.raises(RuntimeError, match="CUDA"):
        _C._dev_wave(torch.zeros(4, dtype=torch.bfloat16), "x")
    assert set(_C._WAVE_DTYPES) == {torch.float32, torch.bfloat16, torch.float16}
    assert [_C._WAVE_DTYPES[t] for t in (torch.float32, torch.bfloat16, torch.float16)] == [
        _C.DTYPE_F32, _C.DTYPE_BF16, _C.DTYPE_F16]


@pytest.mark.parametrize("strict", [False, True])
def test_unsupported_16bit_plan_is_retried_in_float32_unless_strict(strict):
    got = []

    def call(x, pitch, dtype):
        got.append((x.dtype, pitch, dtype))
        return _C.EUNSUPPORTED if dtype != _C.DTYPE_F32 else 0

    x = torch.zeros((3, 100), dtype=torch.bfloat16)[:, :90]  # rows with a pitch of 100 samples
    rc = _C._call_wave(call, x, 100, _C.DTYPE_BF16, strict)
    if strict:
        assert rc == _C.EUNSUPPORTED and got == [(torch.bfloat16, 100, _C.DTYPE_BF16)]
    else:
        assert rc == 0 and got == [(torch.bfloat16, 100, _C.DTYPE_BF16), (torch.float32, 90, _C.DTYPE_F32)]
    got.clear()
    assert _C._call_wave(call, x.float(), 100, _C.DTYPE_F32, strict) == 0  # nothing to retry for fp32
    assert got == [(torch.float32, 100, _C.DTYPE_F32)]


def test_batch_chunking_keeps_the_sample_type(monkeypatch):
    monkeypatch.setattr(_C, "MAX_BATCH", 2)
    seen = []

    @_C._batch_chunked
    def fwd(x, scale):
        seen.append((x.dtype, x.shape[0]))
        return x.float() * scale

    x = _input((5, 16), torch.float16)
    y = fwd(x, 2.0)
    assert seen == [(torch.float16, 2), (torch.float16, 2), (torch.float16, 1)]
    assert torch.equal(y, x.float() * 2.0)


def test_ex_entry_points_reject_an_unknown_sample_type_on_the_host():
    """The *_forward_ex calls take the arguments of *_forward plus x_dtype: a value outside NNAB_DTYPE_*
    is NNAB_EINVAL before any CUDA work, and the same call with a valid dtype gets as far as the device
    (on a GPU-less host: NNAB_EARCH / NNAB_ECUDA; on the GPU it fails on the fake pointers' shapes, never
    with EINVAL from the dtype)."""
    lib = _C.lib()
    P = ctypes.c_void_p
    x = w = out = P(256)  # never dereferenced on the host
    EINVAL = -1
    widths = (ctypes.c_int32 * 1)(512)
    ptrs = (P * 1)(256)

    def calls(dt):
        return {
            "stft": lambda: lib.nnab_stft_forward_ex(x, dt, 4, 4000, 4000, w, w, None, 512, 257, 128, 1, 0, 0,
                                                      0.0, out, 32, None, 0, 1, None),
            "filterbank": lambda: lib.nnab_stft_filterbank_forward_ex(
                x, dt, 4, 4000, 4000, w, w, None, 512, 257, 128, 1, 0, 0.0, 2.0, w, 40, None, out, 32, None, 0,
                1, None),
            "mfcc": lambda: lib.nnab_mfcc_forward_ex(
                x, dt, 4, 4000, 4000, w, w, None, 512, 257, 128, 1, 0, 0.0, 2.0, w, 40, None, 1e-10, 1.0, 80.0,
                w, 13, out, 32, None, 0, 1, None),
            "cqt1992v2": lambda: lib.nnab_cqt1992v2_forward_ex(
                x, dt, 4, 4000, 4000, w, w, None, None, None, 24, 512, 128, 1, 0, None, 1.0, 0, 0.0, out, 32,
                None, 0, 1, None),
            "pyramid": lambda: lib.nnab_cqt_pyramid_forward_ex(
                x, dt, 1, 8192, 8192, 1, ptrs, ptrs, None, widths, 12, w, None, None, None, 1, 512, 0, 12, None,
                1.0, 0, 0.0, out, 17, None, 0, 1, None),
        }

    for name, call in calls(3).items():
        assert call() == EINVAL, name
    for name, call in calls(-1).items():
        assert call() == EINVAL, name
    if not torch.cuda.is_available():
        for dt in (_C.DTYPE_F32, _C.DTYPE_BF16, _C.DTYPE_F16):
            for name, call in calls(dt).items():
                assert call() in (-2, -4), (name, dt)
