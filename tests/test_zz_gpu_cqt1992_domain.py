"""CQT1992v2 (``nnab_cqt1992v2_forward``) across its kernel routes (-m gpu): the tall-A kernel (static and balanced
schedule), the per-K-block-width kernel with and without split-K, the dense kernel with and without split-K and
over several frame phases, and the SIMT kernel.

Each row of tests/cqt1992_domain.py's matrix runs on white noise and must
- write every output cell (the output buffer starts as NaN),
- take the route the model predicts: the route counters must move by exactly ``expected_route`` and the
  executed-MMA-flop counter by exactly ``expected_exec_flops``,
- match the float64 oracle globally, per 8-bin group (the N granularity of the tall and VarN kernels, so a wrong
  group cannot hide under the peak bins) and in phase,
- give bit-identical results on a second call (the balanced schedule and the split-K finalize sum in a fixed
  order), and
- on the tensor-core routes, give a bf16 / fp16 waveform's fp32-upcast result bit for bit, on the same route with
  the same flops; the SIMT kernel, which reads fp32 samples only, must refuse a 16-bit waveform under
  ``strict_dtype``."""
import warnings

import numpy as np
import pytest
import torch

import cqt1992_domain as cd
from conftest import record_error
from helpers import build, run_oracle
from nnaudio_b200 import _C

pytestmark = pytest.mark.gpu

BAR = 1e-4           # max|d| / max|ref| and ||d||_2 / ||ref||_2 (test_gpu_parity.py's bars)
GROUP_BAR = 1e-3     # max|d| over an 8-bin group, over the rms of |ref| in that group
PHASE_FLOOR = 0.01   # phases compared where |X| > PHASE_FLOOR max|X|
PHASE_BAR = 2e-3


def _counts():
    return [_C.cqt1992v2_route_count(r) for r in range(_C.CQ1992_ROUTES)]


def _measured(fn):
    """(fn(), {route: counter delta}, executed MMA flops) of one call."""
    before = _counts()
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
    flops = _C.profile_read_exec_flops()
    return y, {r: a - b for r, (a, b) in enumerate(zip(_counts(), before)) if a != b}, flops


def _check(y, X, fmt, case):
    """y: the kernel's output; X: the float64 complex reference (B, F, T).  Returns the worst errors."""
    y = y.cpu().numpy().astype(np.float64)
    mag = np.abs(X)
    if fmt == "Phase":
        mask = mag > PHASE_FLOOR * mag.max()
        d = float(np.abs((y[..., 0] + 1j * y[..., 1]) - X / np.where(mag > 0, mag, 1))[mask].max())
        record_error("cqt1992_domain", case, phase_unit_max=d)
        assert d <= PHASE_BAR, (case, d)
        return dict(phase=d)
    got = y[..., 0] + 1j * y[..., 1] if fmt == "Complex" else y
    want = X if fmt == "Complex" else mag
    d = np.abs(got - want)
    emax = float(d.max() / mag.max())
    el2 = float(np.linalg.norm(d) / np.linalg.norm(mag))
    F = X.shape[1]
    per_group = [float(d[:, g:g + 8].max() / np.sqrt((mag[:, g:g + 8] ** 2).mean())) for g in range(0, F, 8)]
    worst = int(np.argmax(per_group))
    record_error("cqt1992_domain", case, max_rel=emax, l2_rel=el2, worst_group=worst,
                 worst_group_rel=per_group[worst])
    assert emax <= BAR and el2 <= BAR, (case, emax, el2)
    assert per_group[worst] <= GROUP_BAR, (case, worst, per_group)
    return dict(max_rel=emax, l2_rel=el2, group=per_group[worst])


@pytest.mark.parametrize("name", sorted(cd.ROWS))
def test_cqt1992_domain(name, monkeypatch):
    cls, ctor, B, L = cd.ROWS[name][:4]
    opts = cd.row_options(name)
    if opts["path"] != "auto":
        monkeypatch.setenv("NNAUDIO_B200_PATH", opts["path"])
    mod = build(cls, ctor).cuda()
    F, _, _ = cd.geometry(mod)
    T = cd.frames(mod, L)[1]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    xn = np.random.RandomState(len(name) * 1000 + B).standard_normal((B, L)).astype(np.float32)
    x = torch.from_numpy(xn).cuda()

    refs = {}
    for norm in opts["norms"]:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            c = run_oracle(cls, mod, xn, dict(output_format="Complex", normalization_type=norm), dtype=np.float64)
        refs[norm] = c[..., 0] + 1j * c[..., 1]

    for ctas in opts["tall_ctas"]:
        if ctas is None:
            monkeypatch.delenv("NNAB_TALL_CTAS", raising=False)
        else:
            monkeypatch.setenv("NNAB_TALL_CTAS", str(ctas))
        want_routes = cd.expected_route(mod, B, L, opts["path"], sms, ctas)
        want_flops = cd.expected_exec_flops(mod, B, L, opts["path"], sms, ctas)
        worst = {}
        for norm in opts["norms"]:
            X = refs[norm]
            for fmt in opts["formats"]:
                case = f"{name} ctas={ctas} B{B} L{L} {norm} {fmt}"
                shape = (B, F, T) + ((2,) if fmt != "Magnitude" else ())
                assert X.shape == shape[:3]
                buf = torch.full(shape, float("nan"), device="cuda")

                def into():
                    with _C.output_into(buf):
                        return mod(x, output_format=fmt, normalization_type=norm)

                y, routes, flops = _measured(into)
                assert y.data_ptr() == buf.data_ptr() and tuple(y.shape) == shape, case
                assert routes == want_routes, (case, routes, want_routes)
                assert flops == want_flops, (case, flops, want_flops)
                assert bool(torch.isfinite(y).all()), f"{case}: {int((~torch.isfinite(y)).sum())} cells never written"
                for k, v in _check(y, X, fmt, case).items():
                    worst[k] = max(worst.get(k, 0.0), v)
                again = _measured(lambda: mod(x, output_format=fmt, normalization_type=norm))[0]
                assert torch.equal(y, again), f"{case}: two calls differ"
        print(f"{name} ctas={ctas}: routes {{{', '.join(f'{cd.ROUTE_NAMES[r]}: {n}' for r, n in routes.items())}}}"
              f" flops {want_flops:.4e} worst " + " ".join(f"{k} {v:.2e}" for k, v in worst.items()))

        # 16-bit waveforms: the tensor-core routes read them as is, bit for bit with the fp32 upcast
        fmt, norm = opts["formats"][0], opts["norms"][0]
        args = mod._infer_args(fmt, norm)[1]
        for dt in (torch.bfloat16, torch.float16):
            xh = x.to(dt)
            if want_routes == {_C.CQ1992_SIMT: 1}:
                with pytest.raises(RuntimeError, match="status -6"):
                    _measured(lambda: _C.cqt1992v2_forward(xh, strict_dtype=True, **args))
                continue
            yh, routes, flops = _measured(lambda: _C.cqt1992v2_forward(xh, strict_dtype=True, **args))
            assert routes == want_routes and flops == want_flops, (name, dt, routes, flops)
            y32 = _measured(lambda: mod(xh.float(), output_format=fmt, normalization_type=norm))[0]
            assert torch.equal(yh, y32), (name, dt, float((yh - y32).nan_to_num().abs().max()))
