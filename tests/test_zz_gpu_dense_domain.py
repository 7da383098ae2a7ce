"""The STFT family off the block-partial kernel (-m gpu): the dense tensor-core kernel with and without split-K,
over 1, 2, 4 and 8 frame phases, at the tile-width edges of choose_bn and its N-tile bound, the fused filterbank
epilogue on a dense basis and the un-fused filterbank GEMM, MFCC, and the CUDA-core kernel.

Each row of tests/dense_domain.py's matrix runs on white noise and must
- write every output cell (the output buffer starts as NaN),
- take the routes the model predicts: the route counters must move by exactly ``plan``'s routes and the
  executed-MMA-flop counter by exactly its flops,
- match the float64 reference globally (1e-4), per bin or filter (1e-3 of that row's rms) and in phase,
- give bit-identical results on a second call (the fused rows included: the model allows them at most two atomic
  partial sums per filter), and
- on the tensor-core routes, give a bf16 / fp16 waveform's fp32-upcast result bit for bit under ``strict_dtype``;
  the CUDA-core kernel, which reads fp32 samples only, must refuse a 16-bit waveform."""
import gc
import math
import warnings

import numpy as np
import pytest
import torch

import dense_domain as dd
from conftest import record_error
from helpers import build
from nnaudio_b200 import _C

pytestmark = pytest.mark.gpu

BAR = 1e-4           # max|d| / max|ref| and ||d||_2 / ||ref||_2 (test_gpu_parity.py's bars)
BIN_BAR = 1e-3       # max|d| over one bin (or filter), over the rms of |ref| in it
PHASE_FLOOR = 0.01   # phases compared where |X| > PHASE_FLOOR max|X|
PHASE_BAR = 2e-3
FMT_IDS = {"Complex": _C.FMT_COMPLEX, "Magnitude": _C.FMT_MAGNITUDE, "Phase": _C.FMT_PHASE_ANGLE}


def _counts():
    return [_C.stft_route_count(r) for r in range(_C.STFT_ROUTES)]


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


def _bars(got, want, case, test):
    """Global and per-row (axis 1: bin / filter / coefficient) errors of a real output against float64."""
    d = np.abs(got - want)
    mag = np.abs(want)
    emax = float(d.max() / mag.max())
    el2 = float(np.linalg.norm(d) / np.linalg.norm(mag))
    per_row = d.max(axis=(0, 2)) / np.maximum(np.sqrt((mag ** 2).mean(axis=(0, 2))), 1e-30)
    worst = int(per_row.argmax())
    record_error(test, case, max_rel=emax, l2_rel=el2, worst_bin=worst, worst_bin_rel=float(per_row[worst]))
    assert emax <= BAR and el2 <= BAR, (case, emax, el2)
    assert per_row[worst] <= BIN_BAR, (case, worst, float(per_row[worst]))
    return dict(max_rel=emax, l2_rel=el2, bin=float(per_row[worst]))


def _check_stft(y, X, fmt, case, trainable=False):
    y = y.cpu().numpy().astype(np.float64)
    mag = np.abs(X)
    if fmt == "Phase":
        mask = mag > PHASE_FLOOR * mag.max()
        d = float(np.abs(np.exp(1j * y) - X / np.where(mag > 0, mag, 1))[mask].max())
        record_error("dense_domain", case, phase_unit_max=d)
        assert d <= PHASE_BAR, (case, d)
        return dict(phase=d)
    if fmt == "Complex":
        return _bars(y[..., 0] + 1j * y[..., 1], X, case, "dense_domain")
    return _bars(y, np.sqrt(mag ** 2 + (1e-8 if trainable else 0.0)), case, "dense_domain")


def _device_basis(n_fft, win):
    """(F, n_fft) fp32 planes of the windowed one-sided DFT, built on the device in row blocks."""
    F = n_fft // 2 + 1
    wcos = torch.empty((F, n_fft), dtype=torch.float32, device="cuda")
    wsin = torch.empty_like(wcos)
    n = torch.arange(n_fft, device="cuda")
    w = torch.from_numpy(win).cuda()
    rows = max(1, (1 << 24) // n_fft)
    for k0 in range(0, F, rows):
        k = torch.arange(k0, min(F, k0 + rows), device="cuda")
        ang = (2.0 * math.pi / n_fft) * ((k[:, None] * n[None, :]) % n_fft).double()
        wcos[k0:k0 + rows] = (torch.cos(ang) * w).float()
        wsin[k0:k0 + rows] = (torch.sin(ang) * w).float()
    return wcos, wsin


def _setup(name):
    """(call(x, fmt, strict), float64 reference, input, plan, trainable) of a row."""
    cls, ctor, (B, L) = dd.ROWS[name][:3]
    opts = dd.row_options(name)
    K, F, hop, center, pad_mode, _, trainable = dd.row_geometry(name)
    path = _C.PATH_SIMT if opts["path"] == "simt" else _C.PATH_AUTO
    xn = np.random.RandomState(len(name) * 1000 + B).standard_normal((B, L))
    if opts["levels"] is not None:
        xn = xn * np.resize(np.asarray(opts["levels"]), B)[:, None]
    xn = xn.astype(np.float32)
    pm = _C.PAD_REFLECT if pad_mode == "reflect" else _C.PAD_CONSTANT

    if cls.startswith("direct:"):
        cls = cls[len("direct:"):]
        win = dd.window(ctor.get("window", "hann"), K)
        wcos, wsin = _device_basis(K, win)
        packed = _C.pack_basis(wcos, wsin)
        X = dd.ref_stft_fft(xn, win, hop, center, pad_mode)
        fb_np = dd.bank(name)
        if cls == "STFT":
            def call(x, fmt, strict=False):
                return _C.stft_forward(x, wcos, wsin, packed, K, hop, center, pm, FMT_IDS[fmt], 0.0,
                                       strict_dtype=strict)
            fb = None
        else:
            fb = torch.from_numpy(fb_np.astype(np.float32)).cuda()
            table = _C.build_filterbank_table(fb)

            def call(x, fmt, strict=False):
                return _C.stft_filterbank_forward(x, wcos, wsin, packed, K, hop, center, pm, 0.0, 2.0, fb,
                                                  fb_table=table, strict_dtype=strict)
        plan = dd.row_plan(name)
        refs = {"Complex": X} if fb is None else {None: dd.ref_filterbank(X, fb_np, 2.0)}
        return call, refs, xn, plan, False

    mod = build(cls, ctor).cuda()
    if opts["nudge"]:
        with torch.no_grad():
            g = torch.Generator(device="cpu").manual_seed(7)
            mod.wcos.add_(opts["nudge"] * torch.randn(mod.wcos.shape, generator=g).cuda())
            mod.wsin.add_(opts["nudge"] * torch.randn(mod.wsin.shape, generator=g).cuda())
    stft = mod if cls == "STFT" else (mod.melspec_layer.stft if cls == "MFCC" else mod.stft)
    X = dd.ref_stft(xn, stft.wcos.detach().cpu().numpy(), stft.wsin.detach().cpu().numpy(), hop, center,
                    pad_mode)
    if cls == "STFT":
        def call(x, fmt, strict=False):
            return _C.stft_forward(x, path=path, strict_dtype=strict, **mod._infer_args(fmt)[1])
        fb_np = None
        refs = {"Complex": X}
    else:
        mel = mod.melspec_layer if cls == "MFCC" else mod
        fb_np = (mel.gammatone_basis if cls == "Gammatonegram" else mel.mel_basis).detach().cpu().numpy()
        S = dd.ref_filterbank(X, fb_np.astype(np.float64), float(mel.power), trainable)
        if cls == "MFCC":
            S = dd.ref_mfcc(S, mod.n_mfcc, mod._amin_host, mod._ref_host, mod.top_db)
        name_, kw = mod._infer_args()

        def call(x, fmt, strict=False):
            return getattr(_C, name_)(x, path=path, strict_dtype=strict, **kw)
        refs = {None: S}
    if opts["zero_edges"]:
        nz = np.flatnonzero(np.abs(fb_np).sum(axis=0))
        assert nz[0] >= 16 and nz[-1] < fb_np.shape[1] - 16, "the bank's first and last 16-bin blocks are zero"
    plan = dict(dd.row_plan(name, fb_np), bank=fb_np)
    return call, refs, xn, plan, trainable


@pytest.mark.parametrize("name", sorted(dd.ROWS))
def test_dense_domain(name):
    cls = dd.ROWS[name][0].split(":")[-1]
    opts = dd.row_options(name)
    claims = dd.ROWS[name][3]
    try:
        call, refs, xn, plan, trainable = _setup(name)
        assert all(plan[k] == v for k, v in claims.items() if k in plan), (name, plan, claims)
        want_routes, want_flops = plan["routes"], plan["flops"]
        x = torch.from_numpy(xn).cuda()
        formats = opts["formats"] if cls == "STFT" else (None,)
        worst = {}
        for fmt in formats:
            case = f"{name} {fmt or cls}"
            y0 = _measured(lambda: call(x, fmt))[0]  # shape; also warms the caches (basis, table)
            buf = torch.full(tuple(y0.shape), float("nan"), device="cuda")

            def into():
                with _C.output_into(buf):
                    return call(x, fmt)

            y, routes, flops = _measured(into)
            assert y.data_ptr() == buf.data_ptr(), case
            assert routes == want_routes, (case, {dd.ROUTE_NAMES[r]: n for r, n in routes.items()})
            assert flops == want_flops, (case, flops, want_flops)
            assert bool(torch.isfinite(y).all()), f"{case}: {int((~torch.isfinite(y)).sum())} cells never written"
            if cls == "STFT":
                errs = _check_stft(y, refs["Complex"], fmt, case, trainable)
            elif cls == "MFCC":
                # global bars only: a high coefficient's rms is far below the dB scale of the error
                d = np.abs(y.cpu().numpy() - refs[None])
                emax = float(d.max() / np.abs(refs[None]).max())
                el2 = float(np.linalg.norm(d) / np.linalg.norm(refs[None]))
                record_error("dense_domain", case, max_rel=emax, l2_rel=el2)
                assert emax <= BAR and el2 <= BAR, (case, emax, el2)
                errs = dict(max_rel=emax, l2_rel=el2)
            else:
                errs = _bars(y.cpu().numpy().astype(np.float64), refs[None], case, "dense_domain")
            for k, v in errs.items():
                worst[k] = max(worst.get(k, 0.0), v)
            assert torch.equal(y, _measured(lambda: call(x, fmt))[0]), f"{case}: two calls differ"
        print(f"{name}: routes {{{', '.join(f'{dd.ROUTE_NAMES[r]}: {n}' for r, n in want_routes.items())}}}"
              f" flops {want_flops:.4e} worst " + " ".join(f"{k} {v:.2e}" for k, v in worst.items()))

        # 16-bit waveforms: the tensor-core routes read them as is, bit for bit with the fp32 upcast
        fmt = formats[0]
        for dt in (torch.bfloat16, torch.float16):
            xh = x.to(dt)
            if _C.STFT_SIMT in want_routes:
                with pytest.raises(RuntimeError, match="status -6"):
                    _measured(lambda: call(xh, fmt, True))
                continue
            yh, routes, flops = _measured(lambda: call(xh, fmt, True))
            # the block-partial kernel runs two MMA passes on a bf16 waveform (its lo plane is zero)
            want16 = dd.row_plan(name, plan.get("bank"), 2 if dt == torch.bfloat16 else 3)["flops"]
            assert routes == want_routes and flops == want16, (name, dt, routes, flops, want16)
            y32 = _measured(lambda: call(xh.float(), fmt))[0]
            assert torch.equal(yh, y32), (name, dt, float((yh - y32).nan_to_num().abs().max()))
    finally:
        call = refs = None
        gc.collect()
        torch.cuda.empty_cache()
