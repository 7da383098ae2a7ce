"""Training through the modules on the GPU (-m gpu): every row of tests/train_domain.py runs the module's training
composition — forward under autograd, then ``backward()`` through the dX, dW, FIR-adjoint and inverse-adjoint
kernels — and is held to the float64 reference graph of the same operation.

Per row: the training forward equals the inference forward (bit for bit where no scale or tail is applied in torch,
except the inverse STFT, whose overlap-add atomics make two runs differ in the last bits);
y, ``x.grad`` and every parameter gradient are within ``BAR`` of float64 globally and within ``ROW_BAR`` per clip /
per bin; samples no frame reads get exactly zero gradient; a 16-bit waveform gets its gradient in its own dtype,
within one of its ulps of the fp32 run's; a B = 65 536 row matches the 65 535 + 1 split made by hand.  The offline
route counters and the executed-MMA-flop counter, read over the forward and separately over ``backward()``, equal
the launch model of tests/train_domain.py (so a row that fell onto another route, or ran a GEMM of another shape,
fails); no PYR_* counter may move, since the training pyramid runs octave by octave.  The
reference graphs are pinned on the CPU by tests/test_train_domain_host.py (goldens, oracle, module wiring to 1e-9)."""
import gc
import warnings

import pytest
import torch

import train_domain as td
from conftest import record_error
from helpers import build
from nnaudio_b200 import _C

pytestmark = pytest.mark.gpu

BAR = 1e-4       # max|d| / max|ref| and ||d||_2 / ||ref||_2
FWD_BAR = 2e-6   # training vs inference forward where both read the same contraction: 16 fp32 ulps of the largest
ROW_BAR = 1e-3   # per clip (x.grad) or per bin (dW): max|d| over the rms of the reference row
MANT = {torch.bfloat16: 7, torch.float16: 10}
DTYPES = {"float32": torch.float32, "bfloat16": torch.bfloat16, "float16": torch.float16}


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _run(name, mod, x):
    r = td.ROWS[name]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if r["family"] != "istft":
            return mod(x, **r["fwd"])
        if r["cls"] == "STFT":
            return mod.inverse(x, onesided=r["onesided"], length=r["length"])
        return mod(x, onesided=r["onesided"], length=r["length"])


_COUNTERS = [("stft", r, _C.stft_route_count) for r in range(_C.STFT_ROUTES)] + \
    [("cq", r, _C.cqt1992v2_route_count) for r in range(_C.CQ1992_ROUTES)] + \
    [("pyr", r, _C.pyramid_route_count) for r in range(_C.PYR_ROUTES)]


def _counted(fn):
    """(fn(), {(family, route): count} the offline route counters moved, executed MMA flops added)."""
    before = {(f, r): c(r) for f, r, c in _COUNTERS}
    _C.profile_read_exec_flops()
    _C.profile_enable(True)
    try:
        out = fn()
        torch.cuda.synchronize()
    finally:
        _C.profile_enable(False)
        _C.profile_read()
    flops = _C.profile_read_exec_flops()
    moved = {k: c(k[1]) - before[k] for f, r, c in _COUNTERS for k in [(f, r)]}
    return out, {k: v for k, v in moved.items() if v}, flops


def _train(name, mod, x, W, launches=None):
    """(y, x.grad, {param: grad}) of the module's training path for L = sum(W * y); ``launches``, a dict, receives
    the routes and flops of the forward and of backward() separately."""
    for p in mod.parameters():
        p.grad = None
    x = x.detach().clone().requires_grad_(True)
    y, fwd, fwd_flops = _counted(lambda: _run(name, mod, x))
    _, bwd, bwd_flops = _counted(lambda: (y * W.to(y.dtype)).sum().backward())
    if launches is not None:
        launches.update(fwd=fwd, fwd_flops=fwd_flops, bwd=bwd, bwd_flops=bwd_flops)
    named = dict(mod.named_parameters())
    return y.detach(), x.grad, {n: named[n].grad.detach().clone() for n in td.ROWS[name]["params"]}


def _check_launches(name, mod, got, B=None):
    """4. The routes and executed flops of the forward and of backward() are the launch model's."""
    want = td.launch_model(name, mod, B)
    for k in ("fwd", "bwd"):
        assert got[k] == want[k], (name, k, got[k], want[k])
        assert got[k + "_flops"] == want[k + "_flops"], (name, k, got[k + "_flops"], want[k + "_flops"])


def _check(got, want, name, what, rows, keep=None):
    """Global max-rel and l2-rel against the float64 reference, and per row (clip or bin) max|d| / rms(ref)."""
    got, want = got.double(), want.double()
    assert got.shape == want.shape, (name, what, got.shape, want.shape)
    if keep is not None:
        got, want = got * keep, want * keep
    d = (got - want).abs()
    emax = float(d.max() / want.abs().max())
    el2 = float(d.norm() / want.norm())
    R = want.shape[0]
    rms = want.reshape(R, -1).pow(2).mean(1).sqrt()
    per = (d.reshape(R, -1).max(1)[0] / rms.clamp_min(1e-300))
    per = float(per[rms > 0].max()) if bool((rms > 0).any()) else 0.0
    record_error("train_domain", f"{name}|{what}", max_rel=emax, l2_rel=el2, **{f"worst_{rows}_rel": per})
    assert emax <= BAR and el2 <= BAR, (name, what, emax, el2)
    assert per <= ROW_BAR, (name, what, rows, per)
    return emax, el2, per


def _phase_keep(name, y_ref, W):
    """The cells the loss reads (the |c| mask), where an angle is well defined."""
    if td.ROWS[name]["fwd"].get("output_format") != "Phase":
        return None
    return (W != 0).double()


def _exact_tail(name):
    """Rows whose training forward is bit for bit the inference call: no scale or tail applied in torch."""
    r = td.ROWS[name]
    fmt, norm = r["fwd"].get("output_format"), r["fwd"].get("normalization_type", "librosa")
    return fmt == "Complex" and (r["family"] == "stft" or (r["family"] == "cqt" and norm == "convolutional"))


def _fwd_bar(name):
    """How far the training forward may be from inference.  Where both read the same contraction and torch only
    applies the scale, magnitude, power, banded filterbank, dB or DCT tail that the kernel fuses: FWD_BAR of the largest
    value (an angle moves by that over |c|, and the loss reads cells down to MASK_REL of the largest |c|).  The
    pyramids (whose inference is one fused call with its own FIR and octave routes), the inverse STFT (whose
    overlap-add atomics differ between runs) and the trainable v1 banks (folded in fp32 under autograd, in float64
    for inference) compute a different sum: BAR."""
    r = td.ROWS[name]
    if r["family"] in ("pyramid", "istft") or (r["family"] == "v1" and r["params"]):
        return BAR
    if r["cls"] == "Gammatonegram":
        # inference applies the dense gammatone bank as a second split-bf16 tensor-core GEMM over the 513 bins
        # (STFT_FB_PLANES), training as a torch fp32 matmul: 3.9e-6 measured on the fp16 row
        return 10 * FWD_BAR
    fmt = r["fwd"].get("output_format")
    return FWD_BAR / td.MASK_REL["Phase"] if fmt == "Phase" else FWD_BAR


ROWS = [n for n, r in td.ROWS.items() if r["B"] <= td.MAX_BATCH]
BIG = [n for n, r in td.ROWS.items() if r["B"] > td.MAX_BATCH]


@pytest.mark.parametrize("name", ROWS)
def test_train_domain(name, monkeypatch):
    r = td.ROWS[name]
    if r["env"]:
        monkeypatch.setenv("NNAUDIO_B200_PATH", r["env"])
    dtype = DTYPES[r["dtype"]]
    try:
        mod = build(r["cls"], r["ctor"]).cuda()
        x = td.make_input(name).cuda().to(dtype)
        y_ref, g_ref, W, _ = td.gradients(name, mod, x.float())
        launches = {}
        y, gx, gp = _train(name, mod, x, W, launches)
        _check_launches(name, mod, launches)

        # 1. the training forward is the inference forward
        with torch.no_grad():
            y_inf = _run(name, mod, x)
        keep = _phase_keep(name, y_ref, W)
        if _exact_tail(name):
            assert torch.equal(y, y_inf), name
        else:
            a, b = (y, y_inf) if keep is None else (y * keep, y_inf * keep)
            d = float((a.double() - b.double()).abs().max() / b.double().abs().max())
            assert d <= _fwd_bar(name), (name, "training vs inference forward", d, _fwd_bar(name))

        # 2. forward and gradients against float64
        if r["fwd"].get("output_format") == "Phase" and r["family"] == "stft":
            # angles compared as unit vectors on the cells the loss reads (no wrap at +-pi)
            yu = torch.stack((torch.cos(y.double()), torch.sin(y.double())), -1)
            ru = torch.stack((torch.cos(y_ref), torch.sin(y_ref)), -1)
            _check(yu, ru, name, "y", "clip", keep[..., None])
        else:
            _check(y, y_ref, name, "y", "clip", keep)
        assert gx.dtype == dtype, (name, gx.dtype)
        g32 = gx if dtype == torch.float32 else _train(name, mod, x.float(), W)[1]
        _check(g32, g_ref["x"], name, "x.grad", "clip")
        for n in r["params"]:
            _check(gp[n], g_ref[n], name, n, "bin")

        # 3. samples no frame reads: exactly zero
        dead = g_ref["x"] == 0
        if bool(dead.any()):
            assert bool((gx[dead] == 0).all()), (name, int(dead.sum()), float(gx[dead].abs().max()))

        # 5. 16-bit waveforms: x.grad in the input's dtype, within one of its ulps of the fp32 run's gradient
        # (the float64 comparison above is of the fp32 run: a 16-bit gradient is 2^-9 off by its rounding alone)
        if dtype != torch.float32:
            e = torch.floor(torch.log2(g32.abs().clamp_min(1e-30)))
            ulp = torch.exp2(e - MANT[dtype]).clamp_min(torch.finfo(dtype).tiny * 2.0 ** -MANT[dtype])
            off = (gx.float() - g32).abs()
            assert bool((off <= ulp).all()), (name, float((off / ulp).max()))
            el2 = float(off.norm() / g32.norm())
            assert el2 <= 2.0 ** -MANT[dtype], (name, el2)
    finally:
        _free()


@pytest.mark.parametrize("name", BIG)
def test_train_domain_large_batch(name):
    """65 536 clips, one more than one C call takes: forward and backward equal the 65 535 + 1 split made by hand
    (dW as the sum of the two), and the float64 reference."""
    r = td.ROWS[name]
    n = td.MAX_BATCH
    try:
        mod = build(r["cls"], r["ctor"]).cuda()
        x = td.make_input(name).cuda()
        y_ref, g_ref, W = td.gradients_by_parts(name, mod, x)
        launches = {}
        y, gx, gp = _train(name, mod, x, W, launches)
        _check_launches(name, mod, launches)
        ya, gxa, gpa = _train(name, mod, x[:n], W[:n])
        yb, gxb, gpb = _train(name, mod, x[n:], W[n:])
        split = [(gx, torch.cat((gxa, gxb), 0), "x.grad")]
        if r["family"] == "istft":
            split.append((y, torch.cat((ya, yb), 0), "y"))
        else:
            assert torch.equal(y, torch.cat((ya, yb), 0)), name
        # the overlap-add atomics make two runs of one gradient (and of an inverse STFT) differ in the last bits
        for got, want, what in split + \
                [(gp[p], gpa[p] + gpb[p], p) for p in r["params"]]:
            d = float((got - want).abs().max() / want.abs().max())
            assert d <= 1e-5, (name, what, "vs hand split", d)
        _check(y, y_ref, name, "y", "clip")
        _check(gx, g_ref["x"], name, "x.grad", "clip")
        for p in r["params"]:
            _check(gp[p], g_ref[p], name, p, "bin")
    finally:
        _free()
