"""The CQT pyramid (``nnab_cqt_pyramid_forward``: CQT2010v2, VQT, CQT2010) across its plans and routes (-m gpu).

Each row of tests/pyramid_domain.py's matrix runs on white noise and must
- write every output cell (the output buffer starts as NaN),
- take the route the model predicts: the library's route counters must move by exactly ``expected_routes``,
- match the float64 oracle globally (the parity bars), per octave (so a wrong low octave cannot hide under the
  top octave's peak) and in phase,
- give bit-identical results on a second call, and
- on the fused plans, give a bf16 / fp16 waveform's fp32-upcast result bit for bit; the per-octave plan, which
  reads the waveform as fp32, must refuse a 16-bit waveform under ``strict_dtype``."""
import warnings

import numpy as np
import pytest
import torch

import pyramid_domain as pd
from conftest import record_error
from helpers import build, run_oracle
from nnaudio_b200 import _C
from nnaudio_b200.features.cqt import _pyramid_args, _pyramid_length_plan, _v2_normalization

pytestmark = pytest.mark.gpu

BAR = 1e-4           # max|d| / max|ref| and ||d||_2 / ||ref||_2 (test_gpu_parity.py's bars)
OCTAVE_BAR = 1e-3    # max|d| over an octave's rows, over the rms of |ref| in those rows
PHASE_FLOOR = 0.01   # phases compared where |X| > PHASE_FLOOR max|X|
PHASE_BAR = 2e-3


def _counts():
    return [_C.pyramid_route_count(r) for r in range(_C.PYR_ROUTES)]


def _with_routes(fn):
    """(fn(), {route: counter delta} of the call)."""
    before = _counts()
    with torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter("ignore")  # the reflect-fallback warning of the short rows
        y = fn()
    torch.cuda.synchronize()
    return y, {r: a - b for r, (a, b) in enumerate(zip(_counts(), before)) if a != b}


def _normalization(mod, norm, fmt):
    if hasattr(mod, "_normalization"):  # CQT2010
        return mod._normalization(norm)
    return _v2_normalization(mod, norm, fmt)


def _direct(mod, x, fmt, norm, opts, strict_dtype):
    """``_pyramid_forward``'s C call, with ``strict_dtype`` and, for a row that withholds it, no packed FIR."""
    T, _ = _pyramid_length_plan(mod, x.shape[0], x.shape[-1])
    args = _pyramid_args(mod, fmt, _normalization(mod, norm, fmt))
    if not opts["lowpass_packed"]:
        args["lowpass_packed"] = None
    return _C.cqt_pyramid_forward(x, T=T, strict_dtype=strict_dtype, **args)


def _run(mod, x, fmt, norm, opts, strict_dtype=False):
    if opts["lowpass_packed"] and not strict_dtype:
        return mod(x, output_format=fmt, normalization_type=norm)
    return _direct(mod, x, fmt, norm, opts, strict_dtype)


def _check(y, X, fmt, F, name, case):
    """y: the kernel's output; X: the float64 complex reference (B, n_bins, T)."""
    y = y.cpu().numpy().astype(np.float64)
    mag = np.abs(X)
    if fmt == "Phase":
        mask = mag > PHASE_FLOOR * mag.max()
        d = float(np.abs((y[..., 0] + 1j * y[..., 1]) - X / np.where(mag > 0, mag, 1))[mask].max())
        record_error("pyramid_domain", case, phase_unit_max=d)
        assert d <= PHASE_BAR, (case, d)
        return
    got = y[..., 0] + 1j * y[..., 1] if fmt == "Complex" else y
    want = X if fmt == "Complex" else mag
    d = np.abs(got - want)
    emax = float(d.max() / mag.max())
    el2 = float(np.linalg.norm(d) / np.linalg.norm(mag))
    n_bins = X.shape[1]
    per_octave = []
    for i in range(-(-n_bins // F)):
        rows = slice(max(0, n_bins - F * (i + 1)), n_bins - F * i)
        per_octave.append(float(d[:, rows].max() / np.sqrt((mag[:, rows] ** 2).mean())))
    worst = int(np.argmax(per_octave))
    record_error("pyramid_domain", case, max_rel=emax, l2_rel=el2, worst_octave=worst,
                 worst_octave_rel=per_octave[worst])
    assert emax <= BAR and el2 <= BAR, (case, emax, el2)
    assert per_octave[worst] <= OCTAVE_BAR, (case, worst, per_octave)


@pytest.mark.parametrize("name", sorted(pd.ROWS))
def test_pyramid_domain(name, monkeypatch):
    cls, ctor, B, near = pd.ROWS[name][:4]
    opts = pd.row_options(name)
    if opts["path"] != "auto":
        monkeypatch.setenv("NNAUDIO_B200_PATH", opts["path"])
    mod = build(cls, ctor).cuda()
    F, _ = pd.bank_shapes(mod)
    L = pd.valid_length(mod, near)
    xn = np.random.RandomState(len(name) * 1000 + B).standard_normal((B, L)).astype(np.float32)
    x = torch.from_numpy(xn).cuda()
    want_routes = pd.expected_routes(mod, B, L, "float32", opts["path"], opts["lowpass_packed"])
    lv = pd.levels(mod, L)
    T = (lv[0].len + 2 * lv[0].pad - lv[0].width) // lv[0].hop + 1

    for norm in opts["norms"]:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            c = run_oracle(cls, mod, xn, dict(output_format="Complex", normalization_type=norm), dtype=np.float64)
        X = c[..., 0] + 1j * c[..., 1]
        for fmt in opts["formats"]:
            case = f"{name} B{B} L{L} {norm} {fmt}"
            shape = (B, mod.n_bins, T) + ((2,) if fmt != "Magnitude" else ())
            assert X.shape == shape[:3]
            buf = torch.full(shape, float("nan"), device="cuda")

            def into():
                with _C.output_into(buf):
                    return _run(mod, x, fmt, norm, opts)

            y, routes = _with_routes(into)
            assert y.data_ptr() == buf.data_ptr() and tuple(y.shape) == shape, case
            assert routes == want_routes, (case, routes, want_routes)
            assert bool(torch.isfinite(y).all()), f"{case}: {int((~torch.isfinite(y)).sum())} cells never written"
            _check(y, X, fmt, F, name, case)
            again = _with_routes(lambda: _run(mod, x, fmt, norm, opts))[0]
            assert torch.equal(y, again), f"{case}: two calls differ"

    # 16-bit waveforms: the fused plans read them as is, bit for bit with the fp32 upcast
    fmt, norm = opts["formats"][0], opts["norms"][0]
    for dt in (torch.bfloat16, torch.float16):
        xh = x.to(dt)
        want16 = pd.expected_routes(mod, B, L, str(dt).split(".")[-1], opts["path"], opts["lowpass_packed"])
        if want16 is None:
            with pytest.raises(RuntimeError, match="status -6"):
                _with_routes(lambda: _direct(mod, xh, fmt, norm, opts, True))
            continue
        yh, routes = _with_routes(lambda: _direct(mod, xh, fmt, norm, opts, True))
        assert routes == want16, (name, dt, routes, want16)
        y32 = _with_routes(lambda: _run(mod, xh.float(), fmt, norm, opts))[0]
        assert torch.equal(yh, y32), (name, dt, float((yh - y32).nan_to_num().abs().max()))
