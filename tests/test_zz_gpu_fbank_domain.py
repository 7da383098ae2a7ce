"""The filterbank stage of MelSpectrogram, Gammatonegram and MFCC across its bank domain (-m gpu): every row of
tests/fbank_domain.py's matrix -- fused epilogue on the warp-specialised, plain four-phase, one-phase and dense
kernels, operand planes on the warp-specialised and plain four-phase kernels, the power spectrogram plus
``filterbank_kernel`` after a dense and a block contraction, crafted banks, and the MFCC tail -- runs on white
noise and must
- take the routes the model predicts (``stft_route_count``), execute its MMA flops (which pins the tile width nb)
  and run the warp-specialised kernel exactly when the model says so (``block_ws_launch_count``);
- match the float64 reference globally (1e-4), per filter (each non-empty filter to 1e-4 of its own peak: a
  dropped or doubled partial sum at a range seam moves one filter by far more, but can hide under the global bar
  when the filter is quiet), and give exact zeros on empty filters;
- where the model calls the row deterministic, give bitwise equal results on a second call, on grids of 1, 2 and
  all SMs (warp-specialised rows), and for a bf16 waveform and its fp32 upcast (at the two-pass flops).
Crafted rows that edit the bank in place must switch routes without a module rebuild.  MFCC rows hold the tail
in isolation -- on the same module's GPU mel spectrogram -- to the fp32 bound of fbank_domain.tail_bound."""
import gc
import os
import warnings

import numpy as np
import pytest
import torch

import fbank_domain as fd
from conftest import record_error
from helpers import build
from nnaudio_b200 import _C

pytestmark = pytest.mark.gpu

BAR = 1e-4  # global max|d| / max|ref| and ||d||_2 / ||ref||_2; per filter max|d_j| / max|ref_j|


def _counts():
    return [_C.stft_route_count(r) for r in range(_C.STFT_ROUTES)] + [_C.block_ws_launch_count()]


def _measured(fn, reserve=0):
    """(fn(), {route: counter delta}, executed MMA flops, warp-specialised launches) of one call."""
    before = _counts()
    old = _C.set_sm_reserve(reserve)
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
        _C.set_sm_reserve(old)
    flops = _C.profile_read_exec_flops()
    d = [a - b for a, b in zip(_counts(), before)]
    return y, {r: n for r, n in enumerate(d[:-1]) if n}, flops, d[-1]


def _bank_tensor(cls, mod):
    mel = mod.melspec_layer if cls == "MFCC" else mod
    return mel.gammatone_basis if cls == "Gammatonegram" else mel.mel_basis


def _edit_in_place(fbt, edit):
    """Apply an edit to the module's own bank tensor (copy_: same storage, new version -> the table rebuilds)."""
    fb = fbt.detach().cpu().numpy().astype(np.float64)
    fd.EDITS[edit](fb)
    with torch.no_grad():
        fbt.copy_(torch.from_numpy(fb.astype(np.float32)))


def _check_filters(y, ref, empty, case):
    d = np.abs(y - ref)
    emax = float(d.max() / np.abs(ref).max())
    el2 = float(np.linalg.norm(d) / np.linalg.norm(ref))
    live = np.flatnonzero(~empty)
    per = d[:, live].max(axis=(0, 2)) / np.abs(ref[:, live]).max(axis=(0, 2))
    worst = int(live[per.argmax()])
    record_error("fbank_domain", case, max_rel=emax, l2_rel=el2, worst_filter=worst,
                 worst_filter_rel=float(per.max()))
    assert emax <= BAR and el2 <= BAR, (case, emax, el2)
    assert per.max() <= BAR, (case, worst, float(per.max()))
    assert not np.any(y[:, empty]), (case, "empty filters not exactly zero")


@pytest.mark.parametrize("name", sorted(fd.ROWS))
def test_fbank_domain(name):
    cls, ctor, edit, _, claims, _ = fd.ROWS[name]
    opts = fd.row_options(name)
    c = fd.module_ctor(name)
    n_fft, hop, power = c["n_fft"], c["hop_length"], fd.power_of(name)
    old_env = os.environ.get("NNAB_FB_PLANES")
    if not opts["planes"]:
        os.environ["NNAB_FB_PLANES"] = "0"
    try:
        mod = build(cls, ctor).cuda()
        fbt = _bank_tensor(cls, mod)
        xn = fd.row_input(name)
        x = torch.from_numpy(xn.astype(np.float32)).cuda()

        def call(xx, **kw):  # the module's inference call, its arguments (bank table included) taken anew
            name_, args = mod._infer_args()
            return getattr(_C, name_)(xx, **args, **kw)

        if edit is not None and opts["switch"]:
            # the unedited bank first: its own routes, then the in-place edit switches them
            p0 = fd.row_plan(name, fd.bank(name, edited=False))
            _, routes0, flops0, _ = _measured(lambda: call(x))
            assert routes0 == p0["routes"] and flops0 == p0["flops"], (name, routes0, flops0, p0["flops"])
        if edit is not None:
            _edit_in_place(fbt, edit)
        fb = fbt.detach().cpu().numpy().astype(np.float64)
        np.testing.assert_array_equal(fb, fd.bank(name))  # the model's bank is the module's
        p = fd.row_plan(name, fb)
        props = fd.properties(fb, p)
        assert all(p.get(k, props.get(k)) == v for k, v in claims.items()), (name, p, props, claims)

        y0 = _measured(lambda: call(x))[0]  # shape; warms the caches (basis, table)
        buf = torch.full(tuple(y0.shape), float("nan"), device="cuda")

        def into():
            with _C.output_into(buf):
                return call(x)

        y, routes, flops, ws = _measured(into)
        case = f"{name} {fd.cell(p)}"
        assert y.data_ptr() == buf.data_ptr(), case
        assert routes == p["routes"], (case, routes)
        assert flops == p["flops"], (case, flops, p["flops"])
        assert ws == p["ws"], (case, ws, p["ws"])
        assert bool(torch.isfinite(y).all()), f"{case}: {int((~torch.isfinite(y)).sum())} cells never written"
        got = y.cpu().numpy().astype(np.float64)

        S = fd.ref_output(xn, fb, n_fft, hop, power)
        if cls == "MFCC":
            amin, ref, top_db = mod._amin_host, mod._ref_host, mod.top_db
            want = fd.dd.ref_mfcc(S, mod.n_mfcc, amin, ref, top_db)
            assert got.shape == want.shape, (case, got.shape, want.shape)
            d = np.abs(got - want)
            emax = float(d.max() / np.abs(want).max())
            el2 = float(np.linalg.norm(d) / np.linalg.norm(want))
            fields = dict(max_rel=emax, l2_rel=el2)
            if p["deterministic"]:
                # the tail in isolation: the MFCC call's mel stage is bitwise this output
                mel = _measured(lambda: mod.melspec_layer(x))[0].cpu().numpy()
                dct = mod._dct_rows.cpu().numpy()
                c_ref, v = fd.mfcc_tail(mel, dct, amin, ref, top_db)
                excess = np.abs(got - c_ref) / fd.tail_bound(dct, v)
                fields["tail_bound_used"] = float(excess.max())
                assert excess.max() <= 1.0, (case, float(excess.max()))
                if opts["levels"] is not None and opts["levels"][-1] == 0.0:
                    c0 = fd.silent_c0(fbt.shape[0], amin, ref)
                    bound = fd.tail_bound(dct, v)[-1]
                    assert np.all(np.abs(got[-1, 0] - c0) <= bound[0]), (case, got[-1, 0, :4], c0)
                    assert np.all(np.abs(got[-1, 1:]) <= bound[1:]), case
            record_error("fbank_domain", case, **fields)
            assert emax <= BAR and el2 <= BAR, (case, emax, el2)
        else:
            _check_filters(got, S, ~(fb != 0).any(axis=1), case)

        if not p["deterministic"]:
            return
        assert torch.equal(y, _measured(lambda: call(x))[0]), f"{case}: two calls differ"
        if p["ws"]:
            sms = torch.cuda.get_device_properties(0).multi_processor_count
            for grid in (1, 2):
                _C.persistent_grid_read()
                yg, _, fg, wg = _measured(lambda: call(x), reserve=sms - grid)
                assert wg == 1 and fg == p["flops"], (case, grid, wg, fg)
                # the ledger proves the leg's grid: no persistent launch ran more CTAs, and the block kernel's did
                n, ctas, lo, hi = _C.persistent_grid_read()
                assert n >= 1 and hi == grid and 1 <= lo and ctas <= n * grid, (case, grid, n, ctas, lo, hi)
                assert torch.equal(y, yg), (case, grid)
        # a bf16 waveform: two MMA passes on the block-partial kernel, bit for bit with its fp32 upcast
        xh = x.to(torch.bfloat16)
        yh, routes_h, flops_h, _ = _measured(lambda: call(xh, strict_dtype=True))
        assert routes_h == p["routes"] and flops_h == fd.row_plan(name, fb, passes=2)["flops"], (case, flops_h)
        assert torch.equal(yh, _measured(lambda: call(xh.float()))[0]), case
    finally:
        if old_env is None:
            os.environ.pop("NNAB_FB_PLANES", None)
        else:
            os.environ["NNAB_FB_PLANES"] = old_env
        mod = fbt = None
        gc.collect()
        torch.cuda.empty_cache()
