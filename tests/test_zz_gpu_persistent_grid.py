"""Every persistent tensor-core kernel on grids of 1, 2, 3, 7 CTAs and the full grid (-m gpu).

A persistent CTA walks its work units in a loop that carries the stage-ring parities, the accumulator handoff, the
split-K chunk order and the balanced tall schedule's shared tiles from one unit to the next; on a small grid each CTA
walks many units, and the last round is ragged.  For each row of tests/grid_domain.py's matrix and each grid, an SM
reserve of (SMs - G) caps the grid, the caches are warmed once, and one call runs (into a NaN-filled output where
the route takes a caller buffer).  It must
- show in the persistent-grid ledger exactly the launches, summed CTAs and min / max grid the model predicts,
- move the route counters exactly as modelled at that grid (the tall kernel's schedule changes with G) and execute
  the modelled MMA flops,
- write every output cell and match the row's float64 reference at its domain's bars, and
- on ordered routes give the full grid's bits and the same bits twice; unordered routes (the atomic overlap-add,
  the rolled Mel epilogue) are held to the bars only, and the balanced tall schedule to its own bits at the same G.
The reserve is process wide (stream pools and Griffin-Lim read it too), so every leg restores it."""
import gc
import time
import warnings

import numpy as np
import pytest
import torch

import block_domain as bd
import dense_domain as dd
import grid_domain as gd
import ola_domain as od
import pyramid_domain as pd
from conftest import record_error
from helpers import oracle, run_oracle
from nnaudio_b200 import _C
from test_zz_gpu_dense_domain import _device_basis

pytestmark = pytest.mark.gpu

BAR = 1e-4        # global max|d| / max|ref| and ||d||_2 / ||ref||_2
ROW_BAR = 1e-3    # per bin / 8-bin group / octave / clip: max|d| over the rms of |ref| in it
FILTER_BAR = 1e-4  # per filter: max|d_j| / max|ref_j| (the filterbank domain's bar)
FMT_IDS = {"Complex": _C.FMT_COMPLEX, "Magnitude": _C.FMT_MAGNITUDE}


def _counters():
    c = {("stft", r): _C.stft_route_count(r) for r in range(_C.STFT_ROUTES)}
    c.update({("cq1992", r): _C.cqt1992v2_route_count(r) for r in range(_C.CQ1992_ROUTES)})
    c.update({("pyr", r): _C.pyramid_route_count(r) for r in range(_C.PYR_ROUTES)})
    c[("balanced", None)] = _C.balanced_launch_count()
    c[("ws", None)] = _C.block_ws_launch_count()
    return c


def _measured(fn):
    """(fn(), persistent-grid ledger, {counter: delta}, executed MMA flops) of one call."""
    before = _counters()
    _C.persistent_grid_read()
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
    ledger = _C.persistent_grid_read()
    flops = _C.profile_read_exec_flops()
    after = _counters()
    return y, ledger, {k: after[k] - before[k] for k in after if after[k] != before[k]}, flops


def _bars(got, want, row_axes, case):
    """Global bars, and the per-row bar over each index array of ``row_axes`` (rows of axis 1)."""
    d = np.abs(got - want)
    mag = np.abs(want)
    emax = float(d.max() / mag.max())
    el2 = float(np.linalg.norm(d) / np.linalg.norm(mag))
    per = [float(d[:, idx].max() / max(np.sqrt((mag[:, idx] ** 2).mean()), 1e-30)) for idx in row_axes]
    worst = int(np.argmax(per))
    record_error("persistent_grid", case, max_rel=emax, l2_rel=el2, worst_row=worst, worst_row_rel=per[worst])
    assert emax <= BAR and el2 <= BAR, (case, emax, el2)
    assert per[worst] <= ROW_BAR, (case, worst, per[worst])


def _per(n, width):
    return [np.arange(i, min(n, i + width)) for i in range(0, n, width)]


def _complex(y, fmt):
    y = y.cpu().numpy().astype(np.float64)
    return y[..., 0] + 1j * y[..., 1] if fmt == "Complex" else y


def _setup(name, mod):
    """(call(buf or None), check(y, case)) of a row: ``buf`` a NaN-filled output the call writes into (None where
    the route allocates its own)."""
    row = gd.ROWS[name]
    fam = row["family"]
    xn = gd.row_input(name)
    x = torch.from_numpy(xn).cuda()

    def into(fn):
        def call(buf):
            if buf is None:
                return fn()
            with _C.output_into(buf):
                return fn()
        return call

    if fam in ("dense", "block", "cqt1992", "pyramid"):
        fmt = row["fmt"]
        fn = into(lambda: mod(x, output_format=fmt))
        if fam == "dense":
            X = dd.ref_stft(xn, mod.wcos.detach().cpu().numpy(), mod.wsin.detach().cpu().numpy(),
                            row["ctor"]["hop_length"])
            rows = _per(X.shape[1], 1)
        elif fam == "block":
            X = bd.ref_stft(xn, row["ctor"]["n_fft"], row["ctor"]["hop_length"])
            rows = _per(X.shape[1], 1)
        else:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                c = run_oracle(row["cls"], mod, xn, dict(output_format="Complex"), dtype=np.float64)
            X = c[..., 0] + 1j * c[..., 1]
            # 8-bin groups (the tall and per-K-block-width N granularity), or octaves counted from the top
            n = X.shape[1]
            F = 8 if fam == "cqt1992" else pd.bank_shapes(mod)[0]
            rows = [np.arange(max(0, n - F * (i + 1)), n - F * i) for i in range(-(-n // F))]
        want = X if fmt == "Complex" else np.abs(X)
        return fn, lambda y, case: _bars(_complex(y, fmt), want, rows, case)

    if fam == "dense_direct":
        K, hop = row["ctor"]["n_fft"], row["ctor"]["hop_length"]
        win = dd.window(row["ctor"]["window"], K)
        wcos, wsin = _device_basis(K, win)
        packed = _C.pack_basis(wcos, wsin)
        X = dd.ref_stft_fft(xn, win, hop)
        fn = into(lambda: _C.stft_forward(x, wcos, wsin, packed, K, hop, True, _C.PAD_REFLECT,
                                          FMT_IDS[row["fmt"]], 0.0))
        return fn, lambda y, case: _bars(_complex(y, row["fmt"]), X, _per(X.shape[1], 1), case)

    if fam in ("fbank", "planes"):
        fbt = mod.gammatone_basis if fam == "planes" else mod.mel_basis
        fb = fbt.detach().cpu().numpy().astype(np.float64)
        X = dd.ref_stft(xn, mod.stft.wcos.detach().cpu().numpy(), mod.stft.wsin.detach().cpu().numpy(),
                        row["ctor"]["hop_length"])
        S = dd.ref_filterbank(X, fb, float(mod.power))
        empty = ~(fb != 0).any(axis=1)

        def check(y, case):
            got = y.cpu().numpy().astype(np.float64)
            d = np.abs(got - S)
            emax = float(d.max() / np.abs(S).max())
            el2 = float(np.linalg.norm(d) / np.linalg.norm(S))
            live = np.flatnonzero(~empty)
            per = d[:, live].max(axis=(0, 2)) / np.abs(S[:, live]).max(axis=(0, 2))
            record_error("persistent_grid", case, max_rel=emax, l2_rel=el2, worst_filter_rel=float(per.max()))
            assert emax <= BAR and el2 <= BAR, (case, emax, el2)
            assert per.max() <= FILTER_BAR, (case, int(live[per.argmax()]), float(per.max()))
            assert not np.any(got[:, empty]), (case, "empty filters not exactly zero")

        return into(lambda: mod(x)), check

    if fam == "istft":
        import nnaudio_b200 as nb
        n_fft, hop, T = row["n_fft"], row["hop"], row["T"]
        imod = nb.iSTFT(n_fft=n_fft, hop_length=hop, window="hann", center=True, verbose=False).cuda()
        win = imod.window_mask.reshape(-1).float().cpu().numpy()
        want = oracle.istft(xn, imod.kernel_cos.cpu().numpy(), imod.kernel_sin.cpu().numpy(),
                            imod.window_mask.cpu().numpy(), hop, center=True, onesided=True, length=None)
        good = od.istft_wss(win, hop, T, True, None) >= 1e-6
        return (lambda buf: imod(x, onesided=True),
                lambda y, case: _bars(y.cpu().numpy()[:, None, good], want[:, None, good], [np.arange(1)], case))

    if fam == "dx":
        K, hop, L = row["K"], row["hop"], row["L"]
        w_re, w_im = (w.astype(np.float32) for w in od.hann_dft_bases(K))
        packed = _C.pack_adjoint_basis(torch.from_numpy(w_re).cuda(), torch.from_numpy(w_im).cuda())
        want = od.ref_backward_input(xn, w_re, w_im, K, hop, True, "reflect", L)
        return (lambda buf: _C.framed_backward_input(x, packed, K, hop, True, _C.PAD_REFLECT, L),
                lambda y, case: _bars(y.cpu().numpy()[:, None, :], want[:, None, :], [np.arange(1)], case))
    raise ValueError(fam)


@pytest.mark.parametrize("name", sorted(gd.ROWS))
def test_persistent_grid(name):
    t0 = time.perf_counter()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    mod = gd.build_module(name)
    mod = mod.cuda() if mod is not None else None
    try:
        call, check = _setup(name, mod)
        bits = {}
        for G in gd.GRIDS:
            m = gd.model(name, mod, G, sms)
            case = f"{name} G={G or sms}"
            old = _C.set_sm_reserve(0 if G is None else sms - G)
            try:
                y0 = _measured(lambda: call(None))[0]  # warms the caches (bases, tables, workspaces)
                buf = torch.full(tuple(y0.shape), float("nan"), device="cuda")
                y, ledger, routes, flops = _measured(lambda: call(buf))
                again = _measured(lambda: call(None))[0]
            finally:
                _C.set_sm_reserve(old)
            if gd.ROWS[name]["family"] not in ("istft", "dx"):
                assert y.data_ptr() == buf.data_ptr(), case
            assert ledger == m["ledger"], (case, ledger, m["ledger"], m["launches"])
            assert routes == m["routes"], (case, routes, m["routes"])
            assert flops == m["flops"], (case, flops, m["flops"])
            assert bool(torch.isfinite(y).all()), f"{case}: {int((~torch.isfinite(y)).sum())} cells never written"
            check(y, case)
            key = m["bitwise_key"]
            if key is None:
                continue
            assert torch.equal(y, again), f"{case}: two calls differ"
            if key in bits:
                assert torch.equal(y, bits[key]), f"{case}: differs from the {key} leg"
            bits.setdefault(key, y)
        print(f"{name}: {time.perf_counter() - t0:.2f} s")
    finally:
        mod = call = check = None
        gc.collect()
        torch.cuda.empty_cache()
