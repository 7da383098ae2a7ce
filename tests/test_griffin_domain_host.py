"""Griffin_Lim's float64 stage references, glue bound and launch model on the host (tests/griffin_domain.py):
- the composed stage references equal the reference source restated (``oracle.griffin_lim``) in float64;
- the float32 torch update stays within ``glue_bound``, and three plausible glue bugs leave it;
- ``call_model`` agrees with ``dense_domain.plan`` and ``ola_domain``, and every row's claimed route with the plan;
- the stage recorder the GPU test uses sees the calls of the module in their order, on the CPU stand-ins."""
import numpy as np
import pytest
import torch

import cpu_kernels
import dense_domain as dd
import griffin_domain as gd
import ola_domain as od
from helpers import oracle

import nnaudio_b200 as nb

SMALL = sorted(n for n, r in gd.ROWS.items() if r["n_fft"] <= 2048 and r["B"] * r["T"] <= 4096)


def _exact_bases(row):
    """The oracle's window (scipy's, rounded to float32, centred in n_fft) and its DFT rows in float64."""
    n_fft = row["n_fft"]
    w = oracle._padded_window(row["window"], gd.win_length_of(row), n_fft, np.float64)
    k = np.arange(n_fft // 2 + 1)[:, None]
    ang = 2.0 * np.pi * ((k * np.arange(n_fft)[None, :]) % n_fft) / n_fft
    return w, np.cos(ang) * w, np.sin(ang) * w


@pytest.mark.parametrize("name", SMALL)
def test_ref_loop_matches_oracle(name):
    row = gd.ROWS[name]
    S, ph = gd.problem(row)
    w, wcos, wsin = _exact_bases(row)
    wss = od.istft_wss(w, row["hop"], row["T"], True, None)
    assert wss.min() > 1e-10, "every row's window sum-square is positive inside the output"
    got = gd.ref_loop(S, ph, row["hop"], w, wcos, wsin, row["n_iter"], row["momentum"], row["pad_mode"])
    want = oracle.griffin_lim(S, ph, row["n_fft"], n_iter=row["n_iter"], hop=row["hop"],
                              win_length=gd.win_length_of(row), window=row["window"], pad_mode=row["pad_mode"],
                              momentum=row["momentum"])
    assert got.shape == want.shape == (row["B"], gd.clips_len(row))
    err = float(np.abs(got - want).max() / np.abs(want).max())
    assert err < 1e-12, (name, err)


def test_ref_inverse_keeps_the_undivided_sum_where_the_oracle_is_not_finite():
    """hop == n_fft with a Hann window: the window sum-square is zero at every frame start inside the output.  The
    oracle (torch.istft's rule) divides anyway; the stage reference (the library's rule) keeps the sum there."""
    n_fft = hop = 64
    rng = np.random.RandomState(5)
    X = rng.standard_normal((1, n_fft // 2 + 1, 6)) + 1j * rng.standard_normal((1, n_fft // 2 + 1, 6))
    w = oracle._padded_window("hann", n_fft, n_fft, np.float64)
    wss = od.istft_wss(w, hop, 6, True, None)
    with np.errstate(divide="ignore", invalid="ignore"):
        want = oracle.torch_istft_restated(X, n_fft, hop, w, True)
    got = gd.ref_inverse(X, w, hop)
    zero = wss <= 1e-10
    assert zero.any() and not np.isfinite(want[:, zero]).all()
    assert np.isfinite(got).all()
    assert np.abs(got[:, ~zero] - want[:, ~zero]).max() < 1e-12 * np.abs(want[:, ~zero]).max()


# ------------------------------------------------------------------------------------------ the glue ----
def _recorded(cfg, monkeypatch, S, ph):
    """(module output, Recorder) of one call of the module on the CPU stand-ins."""
    cpu_kernels.install(monkeypatch)
    mod = nb.Griffin_Lim(**cfg)
    with gd.Recorder(mod) as rec:
        y = mod(torch.from_numpy(S), rand_phase=torch.from_numpy(ph))
    assert "_inverse" not in vars(mod) and "forward" not in vars(mod._stft), "the recorder restores the module"
    return y, rec, mod


def _torch_update(r, p, decay):
    """Griffin_Lim.forward's update in float32 torch, from (..., 2) float32 r and p."""
    a = r - decay * p
    return a / (torch.sqrt(a.pow(2).sum(-1)).unsqueeze(-1) + 1e-16)


def _glue_ratio(spec, S, r, p, m):
    """Worst ratio of |spec - S ref_update(r, p, m)| to glue_bound; spec, r, p: (..., 2) float32."""
    want = S.astype(np.float64) * gd.ref_update(gd.cplx(r), gd.cplx(p), m)
    got = gd.cplx(spec)
    bound = gd.glue_bound(gd.cplx(r), gd.cplx(p), m, S)
    return max(gd.ratio(got.real - want.real, bound), gd.ratio(got.imag - want.imag, bound))


def _times_S(angles, S):
    """S4 * angles in float32 torch, as the module forms the next inverse's input."""
    return torch.from_numpy(S).unsqueeze(-1) * angles


MUTATIONS = {
    "decay_is_momentum": lambda r, p, pp, m: _torch_update(r, p, m),
    "tprev_one_iteration_late": lambda r, p, pp, m: _torch_update(r, pp, m / (1 + m)),
    "conjugate_rebuilt": lambda r, p, pp, m: _torch_update(r * torch.tensor([1.0, -1.0]), p, m / (1 + m)),
}


def _glue_problem(monkeypatch):
    row = gd.ROWS["block1_256_64"]
    S, ph = gd.problem(row)
    _, rec, _ = _recorded(gd.ctor(row), monkeypatch, S, ph)
    fwd = [o for _, o in rec.forwards()]
    inv = [i for i, _ in rec.inverses()]
    return row, S, fwd, inv


def test_float32_glue_stays_within_glue_bound(monkeypatch):
    """The update the module ran (recorded as the next inverse's input) and the same torch expression re-run here
    both stay within glue_bound of float64 on every cell; the worst cell uses a fair share of it, so the bound is
    not loose by orders of magnitude."""
    row, S, fwd, inv = _glue_problem(monkeypatch)
    m = row["momentum"]
    worst = 0.0
    for i, r in enumerate(fwd):
        p = fwd[i - 1] if i else torch.zeros_like(r)
        q_rec = _glue_ratio(inv[i + 1], S, r, p, m)
        q_re = _glue_ratio(_times_S(_torch_update(r, p, m / (1 + m)), S), S, r, p, m)
        assert q_rec <= 1.0 and q_re <= 1.0, (i, q_rec, q_re)
        worst = max(worst, q_rec, q_re)
    assert worst > 0.02, worst


@pytest.mark.parametrize("mutation", sorted(MUTATIONS))
def test_glue_mutations_leave_glue_bound(mutation, monkeypatch):
    """Each plausible glue bug exceeds the bound by orders of magnitude at the same cells where the real update
    stays within it: the bound could be loosened 1000-fold and still catch them."""
    row, S, fwd, _ = _glue_problem(monkeypatch)
    m = row["momentum"]
    for i in range(2, len(fwd)):
        r, p, pp = fwd[i], fwd[i - 1], fwd[i - 2]
        q = _glue_ratio(_times_S(MUTATIONS[mutation](r, p, pp, m), S), S, r, p, m)
        assert q > 1e3, (mutation, i, q)


def test_initial_phase_bound_bites():
    """S (cos 2 pi phase, sin 2 pi phase) in float32 torch stays within initial_bound, and swapped cos / sin is far
    outside it."""
    row = gd.ROWS["block1_256_64"]
    S, ph = gd.problem(row)
    t = torch.from_numpy(ph)
    got = torch.stack((torch.cos(2 * np.pi * t), torch.sin(2 * np.pi * t)), -1) * torch.from_numpy(S)[..., None]
    want = S.astype(np.float64) * gd.ref_initial(ph)
    bound = gd.initial_bound(ph, S)
    g = gd.cplx(got.numpy())
    assert max(gd.ratio(g.real - want.real, bound), gd.ratio(g.imag - want.imag, bound)) <= 1.0
    assert gd.ratio(g.real - want.imag, bound) > 1e3


# ------------------------------------------------------------------------------------------ launch model ----
@pytest.mark.parametrize("name", sorted(gd.ROWS))
def test_call_model_agrees_with_the_kernel_models(name):
    row = gd.ROWS[name]
    model = gd.call_model(row)
    n_fft, hop, T, n_iter = row["n_fft"], row["hop"], row["T"], row["n_iter"]
    F = n_fft // 2 + 1
    assert model["route"] == row["route"], (name, dd.ROUTE_NAMES[model["route"]])
    parts = gd.chunks(row["B"])
    assert sum(parts) == row["B"] and max(parts) <= 65535
    plans = [dd.plan(n_fft, F, hop, b, hop * (T - 1), True, gd.row_block(row)) for b in parts]
    assert all(p["routes"] == {row["route"]: 1} for p in plans)
    assert model["routes"] == ({row["route"]: n_iter * len(parts)} if n_iter else {})
    inv = sum(od.ola_exec_flops(*od.istft_operands(b, T, n_fft, F)) for b in parts)
    assert model["flops"] == n_iter * sum(p["flops"] for p in plans) + (n_iter + 1) * inv
    if row["route"] == gd.BLK:
        assert gd.row_block(row) and plans[0]["nb"] is not None
    else:
        assert plans[0]["nb"] is None


def test_matrix_covers_the_issue_edges():
    """The routes and edges the matrix exists for are present, including both determinism outcomes."""
    rows = gd.ROWS.values()
    assert {r["route"] for r in rows} == {gd.BLK, gd.DENSE}
    assert any(r["route"] == gd.BLK and r["hop"] % 128 == 0 for r in rows)           # four-phase
    assert any(r["route"] == gd.BLK and r["hop"] % 128 != 0 for r in rows)           # one-phase
    assert any(dd.num_phases(r["hop"]) == 4 and r["route"] == gd.DENSE for r in rows)
    assert any(r["B"] > 65535 for r in rows)
    assert any(r["momentum"] == 0 for r in rows) and any(r["n_iter"] == 0 for r in rows)
    det = {gd.call_model(r)["deterministic"] for r in rows}
    assert det == {True, False}
    # the largest n_fft runs the four-phase kernel over 11 N tiles and cuts its overlap-add GEMM into 3 K chunks
    big = gd.ROWS["block4_8192_2048"]
    K_gemm = od.istft_operands(1, big["T"], 8192, 4097)[2]
    assert od.ola_k_splits(K_gemm) == 3 and gd.ola_addends(big) == 12


def test_module_block_agrees_with_row_block():
    for name in ("block1_256_64", "block1_384_192", "block4_512_128", "dense_hamming_512_128", "dense_400_160",
                 "dense_512_160_wl400"):
        row = gd.ROWS[name]
        mod = nb.Griffin_Lim(**gd.ctor(row))
        assert gd.module_block(mod) == gd.row_block(row) == (row["route"] == gd.BLK), name


# ------------------------------------------------------------------------------------------ the recorder ----
CFG = [
    dict(n_fft=256, n_iter=6, hop_length=64),
    dict(n_fft=512, n_iter=4, hop_length=128, win_length=400, window="hamming", momentum=0.5),
    dict(n_fft=256, n_iter=3, hop_length=64, pad_mode="constant"),
]


@pytest.mark.parametrize("cfg", CFG, ids=[f"cfg{i}" for i in range(len(CFG))])
def test_recorder_sees_every_stage_in_order(cfg, monkeypatch):
    """On the CPU stand-ins: the calls alternate inverse / forward and end with an inverse, each forward reads the
    inverse just before it, the module returns the last inverse, and every recorded stage equals its float64
    reference (the stand-ins compute in float64)."""
    row = dict(n_fft=cfg["n_fft"], hop=cfg["hop_length"], T=40, B=2, window=cfg.get("window", "hann"),
               win_length=cfg.get("win_length"), pad_mode=cfg.get("pad_mode", "reflect"))
    S, ph = gd.problem(row)
    y, rec, mod = _recorded(cfg, monkeypatch, S, ph)
    assert rec.kinds() == gd.call_order(cfg["n_iter"])
    for (_, _, a_out), (kind, f_in, _) in zip(rec.calls[0::2], rec.calls[1::2]):
        assert kind == "forward" and torch.equal(a_out, f_in)
    assert torch.equal(rec.calls[-1][2], y)
    win = mod._stft.window_mask.reshape(-1).numpy()
    wcos, wsin = mod._stft.wcos.numpy(), mod._stft.wsin.numpy()
    for X, out in rec.inverses():
        want = gd.ref_inverse(gd.cplx(X), win, cfg["hop_length"])
        assert np.abs(out.numpy() - want).max() <= 1e-6 * np.abs(want).max()
    for x, out in rec.forwards():
        want = gd.ref_forward(x.numpy(), wcos, wsin, cfg["hop_length"], row["pad_mode"])
        assert np.abs(gd.cplx(out.numpy()) - want).max() <= 1e-6 * np.abs(want).max()
    first = gd.cplx(rec.calls[0][1].numpy())
    want = S.astype(np.float64) * gd.ref_initial(ph)
    bound = gd.initial_bound(ph, S)
    assert max(gd.ratio(first.real - want.real, bound), gd.ratio(first.imag - want.imag, bound)) <= 1.0


# --------------------------------------------------------------------------------------------- edges ----
def test_center_false_fails_to_broadcast_like_the_oracle(monkeypatch):
    """center=False: the inverse keeps its n_fft / 2 margins, so the centred forward returns n_fft / hop more frames
    than S has and the update cannot subtract tprev.  The module and the oracle's loop both fail there."""
    cpu_kernels.install(monkeypatch)
    row = gd.ROWS["block1_256_64"]
    S, ph = gd.problem(row)
    mod = nb.Griffin_Lim(**gd.ctor(row), center=False)
    with pytest.raises(RuntimeError, match=r"The size of tensor a \(44\) must match the size of tensor b \(40\)"):
        mod(torch.from_numpy(S), rand_phase=torch.from_numpy(ph))
    with np.errstate(divide="ignore", invalid="ignore"), \
            pytest.raises(ValueError, match="operands could not be broadcast together"):
        oracle.griffin_lim(S, ph, 256, n_iter=1, hop=64, center=False)
