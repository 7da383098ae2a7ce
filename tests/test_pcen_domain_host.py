"""No-GPU checks of PCEN's float64 spec and its error bounds (tests/pcen_domain.py).

* the analytic float64 adjoint ``reference_grad`` equals float64 autograd through ``reference_torch``;
* a float32 emulation of the forward and backward kernels' op order stays inside ``forward_bound`` /
  ``backward_bound`` on every row of the matrix small enough to emulate, with the fraction of each bound it used
  printed and recorded;
* each planted slip (``pd.MUTATIONS``) leaves the bound by at least 100x somewhere in the matrix, so the bounds
  bite;
* ``launch_model`` and ``layout`` agree with the matrix: every stated tile and block edge is reached.
"""
import numpy as np
import pytest
import torch

import pcen_domain as pd
from conftest import record_error

SMALL = sorted(n for n in pd.ROWS if n not in pd.BIG)


def _case(name, kind, seed=1):
    row = pd.ROWS[name]
    s, g, b, r, eps = pd.params_of(row, kind)
    E, W = pd.problem(row, seed)
    return row, (s, g, b, r), eps, E, W


@pytest.mark.parametrize("kind", ["scalar", "channel"])
@pytest.mark.parametrize("B,C,T", [(1, 1, 1), (2, 3, 70), (1, 6, 130)])
def test_reference_grad_matches_autograd(B, C, T, kind):
    row = dict(B=B, C=C, T=T, prm="librosa")
    s, g, b, r, eps = pd.params_of(row, kind)
    E, W = pd.problem(row, seed=B + C + T)
    got = pd.reference_grad(E, s, g, b, r, eps, W, per_channel=kind == "channel")
    Ed = torch.from_numpy(E).double().requires_grad_(True)
    prm = [torch.tensor(np.asarray(v, np.float64), requires_grad=True) for v in (s, g, b, r)]
    (pd.reference_torch(Ed, *prm, eps) * torch.from_numpy(W).double()).sum().backward()
    want = {"E": Ed.grad.numpy(), **{n: p.grad.numpy() for n, p in zip(pd.PARAMS, prm)}}
    for n, w in want.items():
        assert got[n].shape == w.shape, n
        scale = max(np.abs(w).max(), 1e-300)
        assert np.abs(got[n] - w).max() <= 1e-12 * scale, (n, np.abs(got[n] - w).max() / scale)


@pytest.mark.parametrize("name", SMALL)
def test_emulation_within_bounds(name):
    row = pd.ROWS[name]
    used = {}
    for kind in row["kinds"]:
        _, (s, g, b, r), eps, E, W = _case(name, kind)
        pc = kind == "channel"
        e32 = pd.eps32(eps)
        P, _, _ = pd.reference(E, s, g, b, r, e32)
        Pe, Me = pd.emulate_forward(E, s, g, b, r, eps)
        used[f"{kind}_forward"] = pd.ratio(Pe - P, pd.forward_bound(E, s, g, b, r, eps))
        ref = pd.reference_grad(E, s, g, b, r, e32, W, pc)
        bound = pd.backward_bound(E, s, g, b, r, eps, W, pc)
        dE, grads = pd.emulate_backward(E, Me, W, s, g, b, r, eps, pc)
        used[f"{kind}_dE"] = pd.ratio(dE - ref["E"], bound["E"])
        for n in pd.PARAMS:
            assert grads[n].shape == ref[n].shape, n
            used[f"{kind}_{n}"] = pd.ratio(grads[n] - ref[n], bound[n])
    record_error("pcen_emulation", name, **used)
    print(name, " ".join(f"{k} {v:.3f}" for k, v in used.items()))
    assert max(used.values()) <= 1.0, used


# rows the mutations run on: every parameter family, tile ends and both kinds
MUTATION_ROWS = [("T129", "channel"), ("mix", "channel"), ("prm_s_one", "scalar"), ("T431", "scalar"),
                 ("rows514", "channel")]


@pytest.mark.parametrize("mutation", pd.MUTATIONS)
def test_mutations_leave_the_bound(mutation):
    worst = 0.0
    for name, kind in MUTATION_ROWS:
        _, (s, g, b, r), eps, E, W = _case(name, kind)
        pc = kind == "channel"
        e32 = pd.eps32(eps)
        if mutation in ("shift_M", "s_perturbed"):
            P, _, _ = pd.reference(E, s, g, b, r, e32)
            Pe, _ = pd.emulate_forward(E, s, g, b, r, eps, mutate=mutation)
            worst = max(worst, pd.ratio(Pe - P, pd.forward_bound(E, s, g, b, r, eps)))
            continue
        _, Me = pd.emulate_forward(E, s, g, b, r, eps)
        ref = pd.reference_grad(E, s, g, b, r, e32, W, pc)
        bound = pd.backward_bound(E, s, g, b, r, eps, W, pc)
        dE, grads = pd.emulate_backward(E, Me, W, s, g, b, r, eps, pc, mutate=mutation)
        worst = max([worst, pd.ratio(dE - ref["E"], bound["E"])]
                    + [pd.ratio(grads[n] - ref[n], bound[n]) for n in pd.PARAMS])
    record_error("pcen_mutations", mutation, worst_ratio=worst)
    print(mutation, f"{worst:.3g}x the bound")
    assert worst >= 100.0, (mutation, worst)


def test_matrix_reaches_its_edges():
    lay = {n: pd.layout(r["B"], r["C"], r["T"]) for n, r in pd.ROWS.items()}
    assert {pd.ROWS[n]["T"] for n in pd.ROWS} >= {1, 2, 63, 64, 65, 127, 128, 129, 431}
    assert {lay[n]["last_tile"] for n in pd.ROWS} >= {1, 2, 63, 64}, "partial, near-full and full last tiles"
    assert max(lay[n]["tiles"] for n in pd.ROWS) == 1875
    assert {pd.ROWS[n]["B"] * pd.ROWS[n]["C"] for n in pd.ROWS} >= {1, 31, 32, 33, 256 * 128}
    assert {pd.ROWS[n]["C"] for n in pd.ROWS} >= {1, 40, 257}
    assert lay["rows31"]["blocks"] == 1 and lay["rows31"]["last_block"] == 31
    assert lay["rows32"]["blocks"] == 1 and lay["rows32"]["last_block"] == 32
    assert lay["rows33"]["blocks"] == 2 and lay["rows33"]["last_block"] == 1
    assert lay["rows514"]["spans_batch"] and lay["rows514"]["last_block"] == 2
    assert lay["T431"]["spans_batch"] and lay["T431"]["last_block"] == 16
    for n in ("T65", "T129"):
        assert lay[n]["last_tile"] == 1, "the reverse walk starts on a 1-frame tile"
    assert lay["T64"]["tiles"] == 1 and lay["T128"]["tiles"] == 2
    # every boundary of the constructor's domain appears, scalar and in the per-channel mix
    sets = {pd.ROWS[n]["prm"] for n in pd.ROWS}
    assert sets >= set(pd.PARAM_SETS) | {"mix"}
    s, g, b, r, _ = pd.params_of(pd.ROWS["mix"], "channel")
    assert len({(float(a), float(c), float(d), float(e)) for a, c, d, e in zip(s, g, b, r)}) == len(pd.EXTREMES)
    eps = {pd.PARAM_SETS[pd.ROWS[n]["prm"]][4] for n in pd.ROWS if pd.ROWS[n]["prm"] != "mix"}
    assert eps >= {1e-12, 1.0}


def test_problem_holds_every_input_pattern():
    E, _ = pd.problem(pd.ROWS["T431"], 1)
    rows = E.reshape(-1, E.shape[-1])
    assert (rows == 0).all(axis=1).any(), "an all-zero row"
    assert ((rows[:, 0] == 0) & (rows[:, 1:].min(axis=1) >= 1e4)).any(), "a zero first frame, then loud frames"
    assert ((rows == rows[:, :1]).all(axis=1) & (rows[:, 0] > 0)).any(), "a constant row"
    nz = rows[rows > 0]
    assert nz.min() < 1e-9 and nz.max() > 1e5


def test_launch_model():
    call = lambda kind, **kw: pd.launch_model(dict(kind=kind, **kw))  # noqa: E731
    assert call("inference", B=2, C=40, T=5) == ["pcen_forward_kernel"]
    assert call("step", B=2, C=40, T=1) == ["pcen_forward_kernel"]
    both = call("train", B=2, C=40, T=5, want_E=True, want_params=True)
    assert both == ["pcen_forward_kernel", "pcen_backward_kernel", "pcen_param_reduce_kernel"]
    assert call("train", B=2, C=40, T=5, want_E=True, want_params=False) == ["pcen_forward_kernel",
                                                                             "pcen_backward_kernel"]
    assert call("train", B=2, C=40, T=5, want_E=False, want_params=True) == both
    assert call("reset", B=0, C=0, T=0) == ["pcen_reset_kernel"]
    for B, C, T in ((0, 40, 5), (2, 40, 0)):
        for kind in ("inference", "step", "train"):
            assert call(kind, B=B, C=C, T=T, want_E=True, want_params=True) == []
