"""Griffin_Lim across its shape domain, stage by stage (-m gpu).

The loop as a whole cannot be held tightly to anything (the phase renormalisation amplifies rounding where |angles|
~ 0, tests/test_griffin_lim.py), so every row of tests/griffin_domain.py's matrix is checked on what the module
itself computed: a recorder keeps the float32 input and output of every inverse and forward call, and
- every inverse output must match the float64 inverse STFT of its recorded input, and every forward output the
  float64 STFT of its recorded input on the module's own bases (the bars of the overlap-add and dense domain tests);
- the input of every inverse after the first must equal S times the float64 update of the two forward outputs
  before it, within ``glue_bound``, and the first inverse's input S (cos 2 pi phase, sin 2 pi phase) within
  ``initial_bound``: a wrong decay, a stale tprev or a conjugated spectrum leaves those bounds;
- the route counters must rise by exactly n_iter forward calls per chunk on the planned route and by nothing on any
  other, and the executed-MMA-flop counter by exactly n_iter forwards and n_iter + 1 inverses: a dense or CUDA-core
  fallback, or a missing or extra inverse, fails;
- a call past 65 535 clips must equal its two chunks run alone, and two calls must be bitwise equal where the launch
  model says both kernels are deterministic;
- the refusal edges raise before any answer, with the error pinned."""
import gc
import warnings

import numpy as np
import pytest
import torch

import dense_domain as dd
import griffin_domain as gd
import ola_domain as od
from conftest import record_error
from nnaudio_b200 import _C

import nnaudio_b200 as nb

pytestmark = pytest.mark.gpu

BAR = 1e-4       # max|d| / max|ref| and ||d||_2 / ||ref||_2
ROW_BAR = 1e-3   # per clip (inverse) or per bin (forward): max|d| over the rms of the reference row


def _counts():
    return [_C.stft_route_count(r) for r in range(_C.STFT_ROUTES)]


def _measured(fn):
    """(fn(), {route: counter delta}, executed MMA flops) of one call."""
    before = _counts()
    _C.profile_read_exec_flops()
    _C.profile_enable(True)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            y = fn()
        torch.cuda.synchronize()
    finally:
        _C.profile_enable(False)
        _C.profile_read()
    flops = _C.profile_read_exec_flops()
    return y, {r: a - b for r, (a, b) in enumerate(zip(_counts(), before)) if a != b}, flops


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _errors(got, want, axes):
    """(max-rel, l2-rel, worst per-row rel) of real or complex arrays; a row is what ``axes`` reduce over."""
    d = np.abs(got - want)
    mag = np.abs(want)
    per_row = d.max(axis=axes) / np.maximum(np.sqrt((mag ** 2).mean(axis=axes)), 1e-30)
    return float(d.max() / mag.max()), float(np.linalg.norm(d) / np.linalg.norm(mag)), float(per_row.max())


def _module(row):
    return nb.Griffin_Lim(**gd.ctor(row)).cuda()


@pytest.mark.parametrize("name", sorted(gd.ROWS))
def test_griffin_lim_stages(name):
    row = gd.ROWS[name]
    n_fft, hop, n_iter, m = row["n_fft"], row["hop"], row["n_iter"], row["momentum"]
    try:
        mod = _module(row)
        model = gd.call_model(row, gd.module_block(mod))
        assert model["route"] == row["route"], (name, dd.ROUTE_NAMES[model["route"]])
        S, ph = gd.problem(row)
        Sd, phd = torch.from_numpy(S).cuda(), torch.from_numpy(ph).cuda()
        with gd.Recorder(mod) as rec:
            y, routes, flops = _measured(lambda: mod(Sd, rand_phase=phd))
        assert routes == model["routes"], (name, {dd.ROUTE_NAMES[r]: n for r, n in routes.items()})
        assert flops == model["flops"], (name, flops, model["flops"])
        assert rec.kinds() == gd.call_order(n_iter)
        assert torch.equal(rec.calls[-1][2], y.cpu())
        assert y.shape == (row["B"], gd.clips_len(row))

        st = mod._stft
        win = st.window_mask.reshape(-1).cpu().numpy()
        wcos, wsin = st.wcos.cpu().numpy(), st.wsin.cpu().numpy()
        wss = od.istft_wss(win, hop, row["T"], True, None)
        good = wss >= 1e-6 * wss.max()
        worst = dict(inv_max=0.0, inv_l2=0.0, inv_clip=0.0, fwd_max=0.0, fwd_l2=0.0, fwd_bin=0.0, glue=0.0)
        for i, (X, out) in enumerate(rec.inverses()):
            out = out.numpy()
            assert np.isfinite(out).all(), (name, "inverse", i)
            want = gd.ref_inverse(gd.cplx(X), win, hop)
            e = _errors(out[:, good].astype(np.float64), want[:, good], (1,))
            for k, v in zip(("inv_max", "inv_l2", "inv_clip"), e):
                worst[k] = max(worst[k], v)
            assert e[0] <= BAR and e[1] <= BAR and e[2] <= ROW_BAR, (name, "inverse", i, e)
        for i, (x, out) in enumerate(rec.forwards()):
            out = gd.cplx(out.numpy())
            assert np.isfinite(out).all(), (name, "forward", i)
            want = gd.ref_forward(x.numpy(), wcos, wsin, hop, row["pad_mode"])
            e = _errors(out, want, (0, 2))
            for k, v in zip(("fwd_max", "fwd_l2", "fwd_bin"), e):
                worst[k] = max(worst[k], v)
            assert e[0] <= BAR and e[1] <= BAR and e[2] <= ROW_BAR, (name, "forward", i, e)

        # the glue: the first inverse reads S e^{2 pi i phase}, every later one S times the float64 update of the
        # two forward outputs before it
        first = gd.cplx(rec.calls[0][1].numpy())
        want = S.astype(np.float64) * gd.ref_initial(ph)
        bound = gd.initial_bound(ph, S)
        q0 = max(gd.ratio(first.real - want.real, bound), gd.ratio(first.imag - want.imag, bound))
        assert q0 <= 1.0, (name, "initial phase", q0)
        fwd = [gd.cplx(o.numpy()) for _, o in rec.forwards()]
        inv_in = [gd.cplx(X.numpy()) for X, _ in rec.inverses()]
        for i, r in enumerate(fwd):
            p = fwd[i - 1] if i else np.zeros_like(r)
            want = S.astype(np.float64) * gd.ref_update(r, p, m)
            bound = gd.glue_bound(r, p, m, S)
            q = max(gd.ratio(inv_in[i + 1].real - want.real, bound), gd.ratio(inv_in[i + 1].imag - want.imag, bound))
            worst["glue"] = max(worst["glue"], q)
            assert q <= 1.0, (name, "update", i, q)
        record_error("griffin_domain", f"{name} n_fft{n_fft} hop{hop} B{row['B']} T{row['T']} n_iter{n_iter}",
                     route=dd.ROUTE_NAMES[model["route"]], flops=model["flops"], initial_phase_ratio=q0, **worst)
        print(f"{name}: route {dd.ROUTE_NAMES[model['route']]} x{n_iter} flops {model['flops']:.4e} "
              + " ".join(f"{k} {v:.2e}" for k, v in worst.items()) + f" initial {q0:.2e}")
    finally:
        mod = rec = None
        _free()


@pytest.mark.parametrize("name", sorted(n for n, r in gd.ROWS.items() if gd.call_model(r)["deterministic"]))
def test_griffin_lim_is_deterministic(name):
    """Two calls are bitwise equal where every overlap-add sample takes at most two atomic additions and the
    forward's plan is deterministic (``gd.call_model``)."""
    row = gd.ROWS[name]
    try:
        mod = _module(row)
        S, ph = gd.problem(row)
        Sd, phd = torch.from_numpy(S).cuda(), torch.from_numpy(ph).cuda()
        with torch.no_grad():
            a = mod(Sd, rand_phase=phd)
            b = mod(Sd, rand_phase=phd)
        assert torch.equal(a, b), (name, float((a - b).abs().max()))
    finally:
        mod = None
        _free()


@pytest.mark.parametrize("name", sorted(n for n, r in gd.ROWS.items()
                                        if r["B"] > gd.MAX_BATCH and gd.call_model(r)["deterministic"]))
def test_griffin_lim_batch_chunks(name):
    """A batch past 65 535 clips runs every transform as a 65 535-clip call and a 1-clip call, with the update on
    the whole batch in between: it equals, bit for bit, the module run on clips 0..65 534 and on clip 65 535 alone,
    with the same phase."""
    row = gd.ROWS[name]
    try:
        mod = _module(row)
        S, ph = gd.problem(row)
        Sd, phd = torch.from_numpy(S).cuda(), torch.from_numpy(ph).cuda()
        n = gd.MAX_BATCH
        whole = mod(Sd, rand_phase=phd)
        head = mod(Sd[:n], rand_phase=phd[:n])
        tail = mod(Sd[n:], rand_phase=phd[n:])
        assert torch.equal(whole, torch.cat((head, tail), 0))
    finally:
        mod = None
        _free()


# --------------------------------------------------------------------------------------------- edges ----
def test_reflect_padding_too_short_raises():
    """Reflect padding needs the rebuilt clips longer than n_fft // 2 = 128 samples.  At hop (T - 1) = 128 the
    first forward raises torch's ReflectionPad1d error, which the reference's padding layer raises; at 64 samples the
    reference's own assertion.  Both come before any output."""
    mod = nb.Griffin_Lim(n_fft=256, hop_length=64, n_iter=2).cuda()
    for T, err, msg in ((3, RuntimeError, "Padding size should be less than the corresponding input dimension"),
                        (2, AssertionError, r"Signal length shorter than reflect padding length \(n_fft // 2\)")):
        S = torch.rand(1, 129, T, device="cuda")
        with pytest.raises(err, match=msg):
            mod(S, rand_phase=torch.rand_like(S))
        torch.cuda.synchronize()


def test_constant_padding_single_frame_raises():
    """T = 1 with constant padding: the centred inverse of one frame has no samples left after the n_fft // 2
    trims, and the library's inverse refuses the empty output with its invalid-argument status before any forward
    runs.  The shortest clip that runs is T = 2 (the ``constant_T2`` row)."""
    mod = nb.Griffin_Lim(n_fft=256, hop_length=64, n_iter=2, pad_mode="constant").cuda()
    S = torch.rand(1, 129, 1, device="cuda")
    with pytest.raises(RuntimeError, match=r"nnab_istft_forward failed: invalid argument.*\(status -1\)"):
        mod(S, rand_phase=torch.rand_like(S))
    torch.cuda.synchronize()


def test_odd_n_fft_raises():
    """An odd n_fft gives n_fft - 1 inverse kernel rows (the reference's own construction of kernel_cos_inv), and
    the first inverse refuses them."""
    mod = nb.Griffin_Lim(n_fft=255, hop_length=64, n_iter=2).cuda()
    S = torch.rand(1, 128, 20, device="cuda")
    with pytest.raises(RuntimeError, match=r"inverse kernels must be \(n_fft, n_fft\)"):
        mod(S, rand_phase=torch.rand_like(S))
    torch.cuda.synchronize()


def test_center_false_fails_to_broadcast():
    """center=False: the inverse keeps its n_fft / 2 margins, the centred forward returns n_fft / hop = 4 frames
    more than S has, and the update cannot subtract tprev (the oracle's loop fails the same way,
    tests/test_griffin_domain_host.py)."""
    mod = nb.Griffin_Lim(n_fft=256, hop_length=64, n_iter=2, center=False).cuda()
    S = torch.rand(2, 129, 40, device="cuda")
    with pytest.raises(RuntimeError, match=r"The size of tensor a \(44\) must match the size of tensor b \(40\)"):
        mod(S, rand_phase=torch.rand_like(S))
    torch.cuda.synchronize()
