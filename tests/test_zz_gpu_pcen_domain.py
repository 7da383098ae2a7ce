"""GPU: PCEN held to its float64 spec under the derived elementwise bounds of tests/pcen_domain.py (-m gpu).

For every row of the matrix, scalar and per-channel parameters:
* forward: every element within ``forward_bound``, written into a NaN-filled buffer (an unwritten cell fails);
* backward for E only, parameters only and both: dE elementwise and each parameter gradient within
  ``backward_bound``, gradients not asked for are None, and two runs give the same bits;
* route proof by torch.profiler: each call launches exactly ``launch_model``'s kernels, so no torch kernel runs;
* streams: 1-frame steps, steps across tile edges, device row maps (fewer and more rows than slots, rows mapped
  outside the slots), device counts past T, a count-0 step of an unprimed slot and masked resets mid-stream, each
  completed stream bitwise equal to the offline call and within ``forward_bound`` of float64;
* the empty cases: a graph-connected empty P with an empty dE and zero parameter gradients, and the C entry point
  clearing the parameter gradients of an empty batch.
The worst fraction of each bound goes to ``record_error``.
"""
import ctypes

import numpy as np
import pytest
import torch

import pcen_domain as pd
from conftest import record_error
from nnaudio_b200 import _C
from nnaudio_b200.pcen import PCEN, PCENStream

pytestmark = pytest.mark.gpu

CASES = [(n, k) for n in sorted(pd.ROWS) for k in pd.ROWS[n]["kinds"]]
WANTS = {"E": (True, False), "params": (False, True), "both": (True, True)}


def _module(row, kind, trainable=False):
    s, g, b, r, eps = pd.params_of(row, kind)
    nc = row["C"] if kind == "channel" else None
    return PCEN(n_channels=nc, s=s, gain=g, bias=b, power=r, eps=eps, trainable=trainable).cuda(), (s, g, b, r, eps)


def _kernels(fn, model):
    """fn(), with the library's launch counter checked to rise by exactly len(model), the kernel count of
    ``pd.launch_model``; which kernels they are, and that no torch kernel runs, ``test_route_proof`` shows with
    torch.profiler."""
    torch.cuda.synchronize()
    before = _C.launch_count()
    out = fn()
    torch.cuda.synchronize()
    assert _C.launch_count() - before == len(model), (_C.launch_count() - before, model)
    return out


def _profiled(fn):
    """The CUDA kernels fn() launches, by torch.profiler (memcpy / memset aside), named as in ``pd.KERNELS``."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type.name == "CUDA" and "memcpy" not in e.name.lower()
             and "memset" not in e.name.lower()]
    return [next((k for k in pd.KERNELS if k in n), n) for n in names]


@pytest.fixture(scope="module", autouse=True)
def _warm():
    m = PCEN(trainable=True).cuda()
    E = torch.rand(1, 1, 3, device="cuda", requires_grad=True)
    m(E).backward(torch.ones(1, 1, 3, device="cuda"))
    PCENStream(m, 1).reset()
    torch.cuda.synchronize()


def _fresh_backward(m, E, W):
    """m(E).backward(W) with no gradient left from an earlier call (accumulating into one would launch an add)."""
    m.zero_grad(set_to_none=True)
    E.grad = None
    m(E).backward(W)


def _route_names(kind):
    """{call: (kernels torch.profiler saw, launch_model's list)} for each call kind, each call warmed up once and
    then profiled: inference, training for E / parameters / both, a stream step, a reset and the empty calls."""
    row = pd.ROWS["prm_power_two"]
    dims = {k: row[k] for k in "BCT"}
    E, W = pd.problem(row, seed=9)
    Ed, Wd = torch.from_numpy(E).cuda(), torch.from_numpy(W).cuda()
    calls = []
    m, _ = _module(row, kind)
    calls.append(("inference", lambda: m(Ed), dict(kind="inference", **dims)))
    for want, (want_E, want_params) in WANTS.items():
        mt, _ = _module(row, kind, trainable=want_params)
        Eg = Ed.clone().requires_grad_(want_E)
        calls.append((f"train {want}", lambda mt=mt, Eg=Eg: _fresh_backward(mt, Eg, Wd),
                      dict(kind="train", want_E=want_E, want_params=want_params, **dims)))
    st = PCENStream(m, row["B"], n_channels=row["C"])
    calls.append(("step", lambda: st.step(Ed), dict(kind="step", **dims)))
    calls.append(("reset", lambda: st.reset(), dict(kind="reset")))
    Z = torch.zeros(0, row["C"], 5, device="cuda", requires_grad=True)
    mz, _ = _module(row, kind, trainable=True)
    calls.append(("empty train", lambda: _fresh_backward(mz, Z, torch.empty(0, row["C"], 5, device="cuda")),
                  dict(kind="train", want_E=True, want_params=True, B=0, C=row["C"], T=5)))
    calls.append(("empty inference", lambda: m(Z.detach()), dict(kind="inference", B=0, C=row["C"], T=5)))
    out = {}
    for what, fn, call in calls:
        with torch.set_grad_enabled(what.startswith(("train", "empty train"))):
            fn()  # warm-up
            out[what] = (_profiled(fn), pd.launch_model(call))
    return out


@pytest.mark.parametrize("kind", ["scalar", "channel"])
def test_route_proof(kind):
    """Each call kind launches exactly ``launch_model``'s kernels and nothing else: inference one forward;
    training the forward, the backward and, when parameters want gradients, the reduction; a stream step one
    forward; a reset one reset kernel; an empty spectrogram nothing.  It runs in a fresh interpreter:
    torch.profiler loses kernel records once its first session in a process is some seconds old, so a session
    here would also blind the profiler of every later test in this one."""
    import json
    import os
    import subprocess
    import sys

    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import json, sys; sys.path[:0] = [{here!r}, {os.path.dirname(here)!r}]; "
            f"import test_zz_gpu_pcen_domain as t; print(json.dumps(t._route_names({kind!r})))")
    flags = ["-s"] if sys.flags.no_user_site else []
    res = subprocess.run([sys.executable, *flags, "-c", code], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr[-4000:]
    routes = json.loads(res.stdout.strip().splitlines()[-1])
    assert len(routes) == 8
    for what, (names, model) in routes.items():
        assert names == model, (what, names, model)
    record_error("pcen_domain_routes", kind, **{what: names for what, (names, _) in routes.items()})


@pytest.mark.parametrize("name,kind", CASES)
def test_forward_within_bound(name, kind):
    row = pd.ROWS[name]
    m, (s, g, b, r, eps) = _module(row, kind)
    E, _ = pd.problem(row, seed=7)
    Ed = torch.from_numpy(E).cuda()
    buf = torch.full(E.shape, float("nan"), device="cuda")

    def run():
        with torch.no_grad(), _C.output_into(buf):
            return m(Ed)

    P = _kernels(run, pd.launch_model(dict(kind="inference", **{k: row[k] for k in "BCT"})))
    assert P.data_ptr() == buf.data_ptr()
    got = P.cpu().numpy()
    assert np.isfinite(got).all(), "an unwritten or non-finite cell"
    ref, _, _ = pd.reference(E, s, g, b, r, pd.eps32(eps))
    q = pd.ratio(got - ref, pd.forward_bound(E, s, g, b, r, eps))
    record_error("pcen_domain_forward", f"{name} {kind} B{row['B']} C{row['C']} T{row['T']}", bound_fraction=q)
    assert q <= 1.0, (name, kind, q)


def _train(m, Eg, Wd):
    P = m(Eg)
    P.backward(Wd)
    return P.detach(), Eg.grad, {n: getattr(m, n).grad for n in pd.PARAMS}


@pytest.mark.parametrize("name,kind", CASES)
def test_backward_within_bound(name, kind):
    row = pd.ROWS[name]
    E, W = pd.problem(row, seed=8)
    Ed, Wd = torch.from_numpy(E).cuda(), torch.from_numpy(W).cuda()
    pc = kind == "channel"
    worst = {}
    ref = bound = None
    for want, (want_E, want_params) in WANTS.items():
        m, (s, g, b, r, eps) = _module(row, kind, trainable=want_params)
        model = pd.launch_model(dict(kind="train", want_E=want_E, want_params=want_params,
                                     **{k: row[k] for k in "BCT"}))
        runs = []
        for i in range(2):
            m.zero_grad(set_to_none=True)
            Eg = Ed.clone().requires_grad_(want_E)
            out = _kernels(lambda: _train(m, Eg, Wd), model)
            runs.append(out)
        (P, dE, grads), (P2, dE2, grads2) = runs
        assert torch.equal(P, P2)
        if ref is None:
            ref = pd.reference_grad(E, s, g, b, r, pd.eps32(eps), W, pc)
            bound = pd.backward_bound(E, s, g, b, r, eps, W, pc)
        if want_E:
            assert torch.equal(dE, dE2)
            q = pd.ratio(dE.cpu().double().numpy() - ref["E"], bound["E"])
            worst[f"{want}_dE"] = q
            assert q <= 1.0, (want, "dE", q)
        else:
            assert dE is None and dE2 is None
        for n in pd.PARAMS:
            if not want_params:
                assert grads[n] is None and grads2[n] is None, n
                continue
            assert torch.equal(grads[n], grads2[n]), n
            got = grads[n].cpu().double().numpy()
            assert got.shape == ref[n].shape, n
            q = pd.ratio(got - ref[n], bound[n])
            worst[f"{want}_{n}"] = q
            assert q <= 1.0, (want, n, q)
        m = None
    record_error("pcen_domain_backward", f"{name} {kind} B{row['B']} C{row['C']} T{row['T']}", **worst)


# ------------------------------------------------------------------------------------------- streams ----
def _stream_case(kind="channel", B=4, C=40, T=300, seed=3):
    row = dict(B=B, C=C, T=T, prm="mix" if kind == "mix" else "librosa")
    m, prm = _module(row, "channel" if kind == "mix" else kind)
    E, _ = pd.problem(row, seed)
    return m, prm, torch.from_numpy(E).cuda(), E


def _check_stream(name, got, m, prm, Ed, E):
    with torch.no_grad():
        whole = m(Ed)
    assert torch.equal(got, whole), name
    s, g, b, r, eps = prm
    ref, _, _ = pd.reference(E, s, g, b, r, pd.eps32(eps))
    q = pd.ratio(got.cpu().numpy() - ref, pd.forward_bound(E, s, g, b, r, eps))
    record_error("pcen_domain_stream", name, bound_fraction=q)
    assert q <= 1.0, (name, q)


@pytest.mark.parametrize("kind", ["scalar", "mix"])
def test_stream_one_frame_steps(kind):
    m, prm, Ed, E = _stream_case(kind, T=150)
    st = PCENStream(m, Ed.shape[0], n_channels=Ed.shape[1])
    model = pd.launch_model(dict(kind="step", B=4, C=40, T=1))
    with torch.no_grad():
        frames = [Ed[:, :, t:t + 1].contiguous() for t in range(Ed.shape[2])]
        parts = [_kernels(lambda: st.step(f), model) for f in frames]
    _check_stream(f"one_frame {kind}", torch.cat(parts, 2), m, prm, Ed, E)


@pytest.mark.parametrize("kind", ["scalar", "mix"])
def test_stream_steps_across_tile_edges(kind):
    m, prm, Ed, E = _stream_case(kind, T=431)
    st = PCENStream(m, Ed.shape[0])
    cuts = [0, 63, 64, 65, 129, 192, 193, 300, 431]
    with torch.no_grad():
        parts = [st.step(Ed[:, :, a:b]) for a, b in zip(cuts[:-1], cuts[1:])]
    _check_stream(f"tile_edges {kind}", torch.cat(parts, 2), m, prm, Ed, E)


def test_stream_device_row_maps_and_counts():
    """Ragged device counts (some past T, clamped), device row maps that permute the slots with fewer rows than
    slots and map extra rows to -1 and to ``slots`` (which compute nothing and leave every slot alone), a count-0
    step of an unprimed slot and a masked reset mid-stream: every stream equals the offline call bit for bit and
    float64 within ``forward_bound``."""
    S, C, T_total, chunk = 5, 40, 400, 48
    m, prm, Ed, E = _stream_case("mix", B=S, C=C, T=T_total, seed=11)
    st = PCENStream(m, S)
    rng = np.random.default_rng(5)
    pos = np.zeros(S, int)
    rows_out = [[] for _ in range(S)]
    restarted = False
    with torch.no_grad():
        # an unprimed slot stepped with count 0 stays unprimed, so its first real frame starts settled
        zero = torch.zeros(1, C, chunk, device="cuda")
        out = st.step(zero, torch.zeros(1, dtype=torch.int32, device="cuda"),
                      torch.tensor([4], dtype=torch.int32, device="cuda"))
        assert torch.count_nonzero(out).item() == 0
        assert torch.count_nonzero(st.primed[4]).item() == 0
        tick = 0
        while (pos < T_total).any():
            tick += 1
            R = int(rng.integers(2, S + 3))  # fewer rows than slots, or more
            perm = rng.permutation(S)[:min(R, S)].tolist()
            slot_of = perm + [(-1 if i % 2 else S) for i in range(R - len(perm))]  # extra rows: outside the slots
            order = rng.permutation(R)
            slot_of = [slot_of[i] for i in order]
            counts = np.zeros(R, int)
            frames = torch.full((R, C, chunk), 7.0, device="cuda")  # junk past the counts and in unmapped rows
            for i, sl in enumerate(slot_of):
                if 0 <= sl < S:
                    n = int(min(rng.integers(0, chunk + 1), T_total - pos[sl]))
                    frames[i, :, :n] = Ed[sl, :, pos[sl]:pos[sl] + n]
                    counts[i] = n if n < chunk or rng.random() < 0.5 else chunk + 100  # past T: clamped
                else:
                    counts[i] = chunk
            state_before = st.state.clone()
            primed_before = st.primed.clone()
            dev_slots = torch.tensor(slot_of, dtype=torch.int32, device="cuda")
            dev_counts = torch.tensor(counts, dtype=torch.int32, device="cuda")
            out = _kernels(lambda: st.step(frames, dev_counts, dev_slots), ["pcen_forward_kernel"])
            touched = set()
            for i, sl in enumerate(slot_of):
                n = min(counts[i], chunk)
                assert torch.count_nonzero(out[i, :, n if 0 <= sl < S else 0:]).item() == 0, (tick, i, sl)
                if 0 <= sl < S:
                    rows_out[sl].append(out[i:i + 1, :, :n].clone())
                    pos[sl] += n
                    if n:
                        touched.add(sl)
            for sl in set(range(S)) - touched:  # no frames, or only rows mapped outside: state unchanged
                assert torch.equal(st.state[sl], state_before[sl]) and torch.equal(st.primed[sl], primed_before[sl])
            if not restarted and pos[0] >= 150:
                # a masked reset mid-stream: slot 0 starts again from frame 0 of its clip, the others continue
                mask = torch.zeros(S, dtype=torch.bool, device="cuda")
                mask[0] = True
                before = st.primed.clone()
                _kernels(lambda: st.reset(mask), pd.launch_model(dict(kind="reset")))
                assert torch.count_nonzero(st.primed[0]).item() == 0 and torch.equal(st.primed[1:], before[1:])
                pos[0], rows_out[0], restarted = 0, [], True
    assert restarted
    got = torch.cat([torch.cat(r, 2) for r in rows_out], 0)
    _check_stream("device_maps", got, m, prm, Ed, E)


# --------------------------------------------------------------------------------------- empty cases ----
@pytest.mark.parametrize("shape", [(0, 4, 9), (2, 4, 0)])
@pytest.mark.parametrize("kind", ["scalar", "channel"])
def test_empty_input_under_autograd(shape, kind):
    row = dict(B=shape[0], C=4, T=shape[2], prm="librosa")
    m, _ = _module(row, kind, trainable=True)
    E = torch.zeros(shape, device="cuda", requires_grad=True)

    def run():
        P = m(E)
        assert P.shape == shape and P.requires_grad and P.grad_fn is not None
        P.backward(torch.empty_like(P))
        return P

    assert pd.launch_model(dict(kind="train", B=shape[0], C=4, T=shape[2], want_E=True, want_params=True)) == []
    _kernels(run, [])
    assert E.grad is not None and E.grad.shape == shape
    for n in pd.PARAMS:
        gr = getattr(m, n).grad
        assert gr is not None and gr.shape == getattr(m, n).shape and torch.count_nonzero(gr).item() == 0, n
    with torch.no_grad():
        _kernels(lambda: m(E), [])


@pytest.mark.parametrize("B,T", [(0, 9), (3, 0)])
@pytest.mark.parametrize("n_out", [1, 4])
def test_backward_entry_point_clears_parameter_gradients_of_empty_input(B, T, n_out):
    C = 4
    E = torch.zeros(B, C, T, device="cuda")
    prm = [torch.full((n_out,), v, device="cuda") for v in (0.1, 0.9, 2.0, 0.5)]
    dp = torch.full((4, n_out), float("nan"), device="cuda")
    dE = torch.empty(B, C, T, device="cuda")
    ws = torch.empty(max(_C.lib().nnab_pcen_workspace_bytes(B, C), 1), dtype=torch.uint8, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    rc = _C.lib().nnab_pcen_backward(p(E), p(E), p(E), B, C, T, *(p(t) for t in prm), int(n_out > 1),
                                     ctypes.c_float(1e-6), p(dE), p(dp), p(ws), ws.numel(),
                                     ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, _C.lib().nnab_strerror(rc)
    torch.cuda.synchronize()
    assert torch.count_nonzero(dp).item() == 0, dp
    dE2, dp2 = _C.pcen_backward(E, E, E, prm, 1e-6)
    assert dE2.shape == (B, C, T) and dp2.shape == (4, n_out) and torch.count_nonzero(dp2).item() == 0
