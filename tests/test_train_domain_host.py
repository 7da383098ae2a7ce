"""CPU checks of the training-domain references and of the host compositions they hold the GPU to.

* The float64 reference graphs of tests/train_domain.py reproduce every input-, parameter- and inverse-gradient golden
  of the reference's own autograd (fp32, so <= 2e-5) and the oracle's forwards (<= 1e-9).
* Every row runs through the real modules, converted to float64, with float64-preserving stand-ins for the C calls:
  y, x.grad and every parameter gradient equal the reference graph to 1e-9.  This pins the host wiring — stage order,
  padding, octave loop, crop, normalisation, magnitude / phase / dB tails, the iSTFT adjoint — independently of the
  kernels.
* The five training and inverse wrappers of ``_C`` split a batch of more than ``MAX_BATCH`` clips: with a library
  that refuses larger batches, 65 536 clips give exactly the unchunked result and dW is the sum of its chunks.
"""
import contextlib
import warnings

import numpy as np
import pytest
import torch

from helpers import build, ref_outputs, rel_errors, run_oracle  # noqa: E402 (sets sys.path)
import cpu_kernels  # noqa: E402
import train_domain as td  # noqa: E402
from cases import CASES, GRAD_CASES, ISTFT_GRAD_CASES, WGRAD_CASES, loss_weights, make_input
from nnaudio_b200 import _C

REFERENCED = ("STFT", "MelSpectrogram", "MFCC", "Gammatonegram", "CQT1992v2", "CQT2010v2", "VQT", "CQT1992",
              "CQT2010")
FAMILY = {"STFT": "stft", "MelSpectrogram": "mel", "Gammatonegram": "mel", "MFCC": "mfcc", "CQT1992v2": "cqt",
          "CQT2010v2": "pyramid", "VQT": "pyramid", "CQT1992": "v1", "CQT2010": "pyramid"}


def _quiet():
    ctx = contextlib.ExitStack()
    ctx.enter_context(warnings.catch_warnings())
    warnings.simplefilter("ignore")
    return ctx


@contextlib.contextmanager
def _adhoc_row(name, family, cls, ctor, fwd, params=(), **extra):
    """A golden case as a temporary row of the matrix, so the same reference graph serves both."""
    name = "golden:" + name
    td.ROWS[name] = dict(family=family, cls=cls, ctor=ctor, fwd=fwd, B=0, L=0, sig="noise", seed=0,
                         dtype="float32", params=tuple(params), env=None, edge="golden", host=False, **extra)
    try:
        yield name
    finally:
        del td.ROWS[name]


# ---------------------------------------------------------------------------------- references vs goldens ----
_GRAD = [c for c in GRAD_CASES if c[1] in REFERENCED]
_WGRAD = [c for c in WGRAD_CASES if c[1] in REFERENCED]


def _golden_grads(cid, cls, ctor, inp, kw, names):
    mod = build(cls, ctor)
    x = torch.from_numpy(make_input(inp))
    with _adhoc_row(cid, FAMILY[cls], cls, ctor, kw, names) as row:
        y, leaves, _ = td.reference(row, mod, x)
        (y * torch.from_numpy(loss_weights(cid, tuple(y.shape))).double()).sum().backward()
    return {n: t.grad for n, t in leaves.items()}


@pytest.mark.parametrize("case", _GRAD, ids=[c[0] for c in _GRAD])
def test_reference_graph_reproduces_input_gradient_golden(case):
    cid, cls, ctor, inp, kw = case
    got = _golden_grads(cid, cls, ctor, inp, kw, ())["x"].numpy()
    want = ref_outputs()["grad|" + cid]
    emax, el2 = rel_errors(got, want)
    assert emax < 2e-5 and el2 < 2e-5, (cid, emax, el2)


@pytest.mark.parametrize("case", _WGRAD, ids=[c[0] for c in _WGRAD])
def test_reference_graph_reproduces_parameter_gradient_golden(case):
    """<= 2e-5 in l2.  The largest single element may be 4e-5 off: these goldens are Magnitude losses, whose
    c/|c| term amplifies the fp32 rounding of the reference's own autograd (wgrad_stft's worst wsin element:
    2.6e-5, with 4.5e-6 in l2)."""
    cid, cls, ctor, inp, kw, names = case
    grads = _golden_grads(cid, cls, ctor, inp, kw, names)
    for n in names:
        want = ref_outputs()[f"wgrad|{cid}|{n}"]
        emax, el2 = rel_errors(grads[n].numpy(), want)
        assert grads[n].shape == want.shape and emax < 4e-5 and el2 < 2e-5, (cid, n, emax, el2)


@pytest.mark.parametrize("case", ISTFT_GRAD_CASES, ids=[c[0] for c in ISTFT_GRAD_CASES])
def test_reference_graph_reproduces_inverse_gradient_golden(case):
    cid, n_fft, hop, win, kind, spec = case
    ref = ref_outputs()
    X = torch.from_numpy(ref[cid + "|X"])
    if kind == "roundtrip":
        cls, ctor, onesided, length = "STFT", dict(n_fft=n_fft, hop_length=hop, window=win, iSTFT=True), True, \
            spec["length"]
    else:
        cls, ctor, onesided, length = "iSTFT", dict(n_fft=n_fft, hop_length=hop, window=win), False, None
    mod = build(cls, ctor)
    with _adhoc_row(cid, "istft", cls, ctor, {}, onesided=onesided, length=length) as row:
        y, leaves, _ = td.reference(row, mod, X)
        (y * torch.from_numpy(loss_weights(cid, tuple(y.shape))).double()).sum().backward()
    want = ref[cid + "|dX"]
    emax, el2 = rel_errors(leaves["x"].grad.numpy(), want)
    assert emax < 2e-5 and el2 < 2e-5, (cid, emax, el2)


_FWD = [(c[0], c[1], c[2], c[3], kw) for c in CASES if c[1] in REFERENCED and c[0] != "stft_default_hop_1d_input"
        for kw in c[4]]


@pytest.mark.parametrize("case", _FWD, ids=[f"{c[0]}-{c[4].get('output_format', '')}" for c in _FWD])
def test_reference_graph_reproduces_the_oracle_forward(case):
    cid, cls, ctor, inp, kw = case
    mod = build(cls, ctor)
    x = make_input(inp)
    with _adhoc_row(cid, FAMILY[cls], cls, ctor, kw) as row, torch.no_grad():
        y, _, extra = td.reference(row, mod, torch.from_numpy(x))
    want = np.asarray(run_oracle(cls, mod, x, kw), dtype=np.float64)
    y = y.numpy()
    if kw.get("output_format") == "Phase":
        # an angle is only defined where |c| is not lost in the rounding of the two computations
        c = extra["c"].numpy()
        keep = np.hypot(c[..., 0], c[..., 1]) > 1e-6 * np.abs(c).max()
        if cls == "STFT":
            y, want = np.exp(1j * y), np.exp(1j * want)
        else:
            keep = keep[..., None].repeat(2, -1)
        assert np.abs(y - want)[keep].max() < 1e-9, cid
        return
    emax, el2 = rel_errors(y, want)
    # the oracle's DCT is float64 where the module's rows are fp32; its v1 forward folds the two stages in float64,
    # which rounds differently from the two fp32-bank stages here (5e-8 measured)
    bar = 1e-7 if cls in ("MFCC", "CQT1992", "CQT2010") else 1e-9
    assert emax < bar and el2 < bar, (cid, kw, emax, el2)


# ------------------------------------------------------------------ the modules' wiring, row by row (float64) ----
def _framed64(x, w_re, w_im, hop, center, pad_mode):
    return cpu_kernels._framed(x.double(), w_re.double(), w_im.double(), hop, center, pad_mode)


def _format64(c, out_format, sqrt_eps):
    re, im = c[..., 0], c[..., 1]
    if out_format == _C.FMT_COMPLEX:
        return c
    if out_format == _C.FMT_MAGNITUDE:
        return torch.sqrt(re * re + im * im + sqrt_eps)
    if out_format == _C.FMT_PHASE_ANGLE:
        return torch.atan2(im, re)
    ang = torch.atan2(im, re)
    return torch.stack((torch.cos(ang), torch.sin(ang)), -1)


def _stft64(x, wcos, wsin, packed, n_fft, hop, center, pad_mode, out_format, sqrt_eps, path=None):
    return _format64(_framed64(x, cpu_kernels._mat(wcos), cpu_kernels._mat(wsin), hop, center, pad_mode),
                     out_format, sqrt_eps)


def _cqt64(x, k_real, k_imag, packed, k_begin, k_end, hop, center, pad_mode, scale, scale_all, out_format,
           sqrt_eps, path=None):
    c = _framed64(x, k_real, k_imag, hop, center, pad_mode)
    if scale is not None:
        c = c * scale.double().view(1, -1, 1, 1)
    return _format64(c * scale_all, out_format, sqrt_eps)


def _dx64(g, packed_adj, K, hop, center, pad_mode, L_in):
    w_re, w_im = packed_adj
    x = torch.zeros((g.shape[0], L_in), dtype=torch.float64, requires_grad=True)
    with torch.enable_grad():
        (dx,) = torch.autograd.grad(_framed64(x, w_re, w_im, hop, center, pad_mode), x, g.double())
    return dx


def _dw64(g, x, K, hop, center, pad_mode):
    F_ = g.shape[1]
    w = [torch.zeros((F_, K), dtype=torch.float64, requires_grad=True) for _ in range(2)]
    with torch.enable_grad():
        return torch.autograd.grad(_framed64(x, w[0], w[1], hop, center, pad_mode), w, g.double())


def _fir64(x, fir, factor):
    return td._fir(x.double(), fir.double(), factor)


def _fir_adj64(g, fir, factor, L_in):
    x = torch.zeros((g.shape[0], L_in), dtype=torch.float64, requires_grad=True)
    with torch.enable_grad():
        (dx,) = torch.autograd.grad(td._fir(x, fir.double(), factor), x, g.double())
    return dx


def _istft64(X, packed, window, n_fft, hop, center, length):
    kc, ks, onesided = packed
    mod = type("M", (), dict(n_fft=n_fft, stride=hop, center=center))()
    P = dict(kernel_cos=kc.double(), kernel_sin=ks.double(), window_mask=window)
    return td._istft(P, mod, X.double(), onesided, length)


def install_f64(monkeypatch):
    """cpu_kernels.install, with every stand-in the training and inverse paths call kept in float64."""
    cpu_kernels.install(monkeypatch)
    monkeypatch.setattr(_C, "block_layout_ok", lambda K, hop: False)   # the packing is never read here
    for name, fn in (("stft_forward", _stft64), ("cqt1992v2_forward", _cqt64), ("framed_backward_input", _dx64),
                     ("framed_backward_weight", _dw64), ("fir_decimate", _fir64),
                     ("fir_decimate_adjoint", _fir_adj64), ("istft_forward", _istft64)):
        monkeypatch.setattr(_C, name, fn)


def _module(name):
    r = td.ROWS[name]
    return build(r["cls"], r["ctor"])


def _run_module(name, mod, x):
    r = td.ROWS[name]
    with _quiet():
        if r["family"] != "istft":
            return mod(x, **r["fwd"])
        if r["cls"] == "STFT":
            return mod.inverse(x, onesided=r["onesided"], length=r["length"])
        return mod(x, onesided=r["onesided"], length=r["length"])


HOST_ROWS = [n for n, r in td.ROWS.items() if r["host"]]


@pytest.mark.parametrize("name", HOST_ROWS)
def test_module_training_graph_equals_the_reference_graph(name, monkeypatch):
    """The modules' training compositions with exact float64 contractions equal the float64 reference graph:
    1e-9 for y, x.grad and every parameter gradient.  The inverse STFT's adjoint runs in fp32 on the host by design
    (``_InverseSTFTFn`` casts the waveform gradient, the window is fp32), so its dX is held to 1e-6."""
    install_f64(monkeypatch)
    r = td.ROWS[name]
    mod = _module(name).double()
    x = td.make_input(name)
    with _quiet():
        y_ref, g_ref, W, _ = td.gradients(name, mod, x)
    for p in mod.parameters():
        p.grad = None
    xm = x.double().requires_grad_(True)
    y = _run_module(name, mod, xm)
    assert y.dtype == torch.float64 and y.shape == y_ref.shape, (name, y.dtype, y.shape, y_ref.shape)
    (y * W).sum().backward()
    # v1 CQT1992 / CQT2010 fold their two stages into one fp32 time-domain bank by design (cqt_v1.py), so they are
    # held to that rounding: 2e-6, on the cells the loss reads for Phase
    folded = r["cls"] in ("CQT1992", "CQT2010")
    bar_y = 2e-6 if folded else 1e-9
    keep, bar_phase = 1.0, bar_y
    if folded and r["fwd"].get("output_format") == "Phase":
        # an angle moves by (bank rounding) / |c|, and the loss reads cells down to MASK_REL of the largest |c|
        keep, bar_phase = (W != 0).double(), bar_y / td.MASK_REL["Phase"]
    emax, el2 = rel_errors((y.detach() * keep).numpy(), (y_ref * keep).numpy())
    assert emax < bar_phase and el2 < bar_phase, (name, "y", emax, el2)
    named = dict(mod.named_parameters())
    bar_y = bar_phase   # the Phase gradients carry the same 1 / |c|
    bar_x = 1e-6 if r["family"] == "istft" else bar_y
    for n, want in g_ref.items():
        got = xm.grad if n == "x" else named[n].grad
        assert got is not None and got.shape == want.shape, (name, n)
        emax, el2 = rel_errors(got.numpy(), want.numpy())
        bar = bar_x if n == "x" else bar_y
        assert emax < bar and el2 < bar, (name, n, emax, el2)
    print(f"{name}: {r['edge']}")


@pytest.mark.parametrize("name", [n for n, r in td.ROWS.items() if r["family"] == "mfcc"])
def test_mfcc_rows_keep_clear_of_the_floor_and_have_a_unique_peak(name):
    """A cell within a rounding error of the top_db floor, or a tie for the peak, would make the row's gradient a
    coin flip between two values; the rows' inputs keep every cell DB_MARGIN dB away from both."""
    mod = _module(name)
    margin, gap = td.mfcc_margins(name, mod, td.make_input(name))
    print(f"{name}: floor margin {margin:.3g} dB, peak gap {gap:.3g} dB")
    assert margin > td.DB_MARGIN and gap > td.DB_MARGIN, (name, margin, gap)
    if mod.top_db == 10.0:
        with torch.no_grad():
            db = td.reference(name, mod, td.make_input(name))[2]["db"].flatten(1)
        floored = (db < db.max(1, keepdim=True)[0] - mod.top_db).double().mean()
        assert floored > 0.5, (name, float(floored))


def test_masked_rows_still_train_on_most_cells():
    """The |c| masks drop only the few cells where the magnitude or phase is ill-conditioned."""
    for name, r in td.ROWS.items():
        if not r["host"] or r["fwd"].get("output_format") not in td.MASK_REL:
            continue
        with _quiet():
            mod = _module(name)
            y, _, extra = td.reference(name, mod, td.make_input(name))
        kept = float(td.loss_mask(name, y.detach(), extra).mean())
        print(f"{name}: loss weight on {kept:.1%} of cells")
        assert kept > 0.6, (name, kept)


# ---------------------------------------------------------------------------------------- batch chunking ----
class _FakeLib:
    """The five entry points, computed in float64 on the CPU from the arguments ``_ptr`` hands over (patched to the
    tensors themselves); like the library they refuse more than 65 535 clips with NNAB_EUNSUPPORTED."""

    def __init__(self):
        self.calls = []

    def _ok(self, name, B):
        self.calls.append((name, int(B)))
        return B <= 65535

    def nnab_istft_workspace_bytes(self, *a):
        return 0

    nnab_framed_backward_input_workspace_bytes = nnab_framed_backward_weight_workspace_bytes = \
        nnab_istft_workspace_bytes

    def nnab_istft_forward(self, X, B, f_in, T, packed, window, n_fft, hop, center, length, out, want, ws, wsb,
                           stream):
        if not self._ok("istft", B):
            return _C.EUNSUPPORTED
        out.copy_(_istft64(X, packed, window, n_fft, hop, bool(center), None if length < 0 else length))
        return 0

    def nnab_fir_decimate(self, x, B, Ln, pitch, fir, taps, factor, y, Ly, stream):
        if not self._ok("fir", B):
            return _C.EUNSUPPORTED
        y.copy_(_fir64(x, fir, factor))
        return 0

    def nnab_fir_decimate_adjoint(self, g, B, Ly, pitch, fir, taps, factor, dx, L_in, stream):
        if not self._ok("fir_adj", B):
            return _C.EUNSUPPORTED
        dx.copy_(_fir_adj64(g, fir, factor, L_in))
        return 0

    def nnab_framed_backward_input(self, g, B, F_, T, packed, K, hop, center, pad_mode, dx, L_in, ws, wsb, stream):
        if not self._ok("dx", B):
            return _C.EUNSUPPORTED
        dx.copy_(_dx64(g, packed, K, hop, bool(center), pad_mode, L_in))
        return 0

    def nnab_framed_backward_weight(self, g, x, B, Ln, pitch, F_, T, K, hop, center, pad_mode, dw, ws, wsb,
                                    stream):
        if not self._ok("dw", B):
            return _C.EUNSUPPORTED
        d_re, d_im = _dw64(g, x, K, hop, bool(center), pad_mode)
        dw.copy_(torch.cat((d_re, -d_im), 0))
        return 0

    def nnab_strerror(self, rc):
        return b"unsupported"


@pytest.fixture
def fake_lib(monkeypatch):
    lib = _FakeLib()
    monkeypatch.setattr(_C, "lib", lambda: lib)
    monkeypatch.setattr(_C, "_ptr", lambda t: t)
    monkeypatch.setattr(_C, "_stream", lambda device: None)
    monkeypatch.setattr(_C, "_dev_f32", lambda t, name: t)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    return lib


B_BIG = _C.MAX_BATCH + 1


def _ints(shape, seed, lo=-3, hi=4):
    """Small integers: every sum below is exact in fp32, so chunked and unchunked results are bit-equal."""
    return torch.randint(lo, hi, shape, generator=torch.Generator().manual_seed(seed)).float()


def test_batches_past_the_limit_are_refused_by_one_call(fake_lib):
    """The fake refuses what the library refuses, so the tests below see the chunking and nothing else."""
    with pytest.raises(RuntimeError):
        _C._check(fake_lib.nnab_fir_decimate(torch.zeros(B_BIG, 8), B_BIG, 8, 8, torch.ones(3), 3, 2,
                                             torch.zeros(B_BIG, 4), 4, None), "nnab_fir_decimate")


def test_istft_forward_chunks_past_the_limit(fake_lib):
    n_fft, hop, T = 8, 2, 3
    X = _ints((B_BIG, n_fft // 2 + 1, T, 2), 1)
    kc, ks = _ints((n_fft, n_fft), 2), _ints((n_fft, n_fft), 3)
    win = torch.ones(n_fft)
    y = _C.istft_forward(X, (kc, ks, True), win, n_fft, hop, True, None)
    want = _istft64(X, (kc, ks, True), win, n_fft, hop, True, None).float()
    assert torch.equal(y, want)
    assert [c for c in fake_lib.calls] == [("istft", 65535), ("istft", 1)]


def test_fir_pair_chunks_past_the_limit(fake_lib):
    x, fir = _ints((B_BIG, 40), 4), _ints((9,), 5)
    y = _C.fir_decimate(x, fir, 2)
    assert torch.equal(y, _fir64(x, fir, 2).float())
    g = _ints(tuple(y.shape), 6)
    dx = _C.fir_decimate_adjoint(g, fir, 2, 40)
    assert torch.equal(dx, _fir_adj64(g, fir, 2, 40).float())
    assert fake_lib.calls == [("fir", 65535), ("fir", 1), ("fir_adj", 65535), ("fir_adj", 1)]


def test_framed_backward_input_chunks_past_the_limit(fake_lib):
    K, hop, F_, L = 8, 4, 3, 32
    T = L // hop + 1
    g = _ints((B_BIG, F_, T, 2), 7)
    w = (_ints((F_, K), 8), _ints((F_, K), 9))
    dx = _C.framed_backward_input(g, w, K, hop, True, _C.PAD_REFLECT, L)
    assert torch.equal(dx, _dx64(g, w, K, hop, True, _C.PAD_REFLECT, L).float())
    assert fake_lib.calls == [("dx", 65535), ("dx", 1)]


def test_framed_backward_weight_sums_its_chunks(fake_lib):
    """dW contracts over every frame of every clip: a chunked batch is the SUM of the chunks' gradients (exactly
    the unchunked result on integer data), added in chunk order."""
    K, hop, F_, L = 8, 4, 3, 32
    T = L // hop + 1
    g, x = _ints((B_BIG, F_, T, 2), 10), _ints((B_BIG, L), 11)
    d_re, d_im = _C.framed_backward_weight(g, x, K, hop, True, _C.PAD_CONSTANT)
    w_re, w_im = _dw64(g, x, K, hop, True, _C.PAD_CONSTANT)
    assert d_re.shape == (F_, K) and d_im.shape == (F_, K)
    assert torch.equal(d_re, w_re.float()) and torch.equal(d_im, w_im.float())
    assert fake_lib.calls == [("dw", 65535), ("dw", 1)]
    # the last chunk alone is not the answer: both chunks count
    l_re, _ = _dw64(g[-1:], x[-1:], K, hop, True, _C.PAD_CONSTANT)
    assert not torch.equal(d_re, l_re.float())


@pytest.mark.parametrize("n_mfcc,n_mels", [(13, 40), (40, 40), (20, 128)])
def test_mfcc_dct_rows_are_the_orthonormal_dct(n_mfcc, n_mels):
    """The reference graph reads MFCC's fp32 DCT rows like any other basis; they are the orthonormal DCT-II."""
    mod = build("MFCC", dict(sr=16000, n_fft=512, n_mels=n_mels, n_mfcc=n_mfcc))
    D = td.dct_ortho(min(n_mfcc, n_mels), n_mels)
    assert mod._dct_rows.shape == D.shape
    assert float((mod._dct_rows.double() - D).abs().max()) < 1e-7


def test_launch_model_reaches_every_claimed_route():
    """Every route a row's edge names is the route the launch model gives that row's training forward, and the
    matrix reaches the block, dense, split-K and SIMT STFT routes and the tall, VarN, dense, split-K and SIMT
    CQT1992v2 routes.  No row's model moves a pyramid (PYR_*) counter: the training pyramid runs octave by octave."""
    claims = td.route_claims()
    reached = set()
    for name, r in td.ROWS.items():
        with _quiet():
            m = td.launch_model(name, _module(name))
        reached |= set(m["fwd"]) | set(m["bwd"])
        assert not any(k[0] == "pyr" for k in list(m["fwd"]) + list(m["bwd"])), name
        assert m["bwd_flops"] > 0, name
        if name in claims:
            assert claims[name] in m["fwd"], (name, claims[name], m["fwd"])
        print(f"{name}: fwd {m['fwd']} {m['fwd_flops']:.3g} flops, bwd {m['bwd']} {m['bwd_flops']:.3g} flops")
    want = {("stft", _C.STFT_BLOCK), ("stft", _C.STFT_DENSE), ("stft", _C.STFT_DENSE_SPLITK), ("stft", _C.STFT_SIMT),
            ("cq", _C.CQ1992_TALL), ("cq", _C.CQ1992_VARN_SPLITK), ("cq", _C.CQ1992_DENSE),
            ("cq", _C.CQ1992_DENSE_SPLITK), ("cq", _C.CQ1992_SIMT)}
    assert want <= reached, want - reached
    assert set(claims.values()) <= reached
