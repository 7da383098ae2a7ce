"""No-GPU checks of CFP's shape matrix, route model and host layer (tests/cfp_domain.py):

- ``_stft_geometry`` frames exactly as ``torch.stft(center=True, pad_mode="constant")`` does, for every parity of
  n_fft and window, frame count included;
- the host layer (half vectors, mirror counts, cut-off weights, mean removal and restore, crops) with every
  contraction swapped for an exact float64 one equals the float64 oracle on every row;
- every row builds the plan it claims, and the matrix reaches every route of every stage kind;
- each row's end-to-end bar is at least 3x what the split-bf16 emulation of its routes gives, and each stage's
  emulated error sits at most a quarter of its route's ``TAU``;
- in-place edits of ``h`` and the two log-frequency maps reach the next call (the bank caches key on ``_version``)."""
import warnings

import numpy as np
import pytest
import torch

import cfp_domain as fd
import cpu_kernels
from helpers import build, rel_errors
from nnaudio_b200 import _C
from nnaudio_b200.features.cfp import _stft_geometry

HOST_MAX_N = 22050  # larger N build multi-gigabyte cosine banks: those rows run on the GPU only
HOST_ROWS = sorted(n for n in fd.ROWS if fd.build_row(n).N <= HOST_MAX_N)
EXACT_BAR = 1e-9     # float64 host layer vs float64 oracle: rounding of different summation orders only
STAGE_ONLY_ABOVE = 1e-3


def _shape(name):
    return fd.row_options(name)["host"] or fd.ROWS[name][2]


def _maps(mod, x, drop):
    with torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return [t.double().numpy() for t in mod._maps(x, drop)]


def _errors(got, want):
    return rel_errors(got, want) if want.size else (0.0, 0.0)


@pytest.mark.parametrize("N", [62, 63, 64, 65, 127])
def test_stft_geometry_frames_like_torch_stft(N):
    """Brute force: the K-tap bank of ``_stft_geometry`` (window shifted j taps, frames centred by K // 2, cropped
    to torch's frame count) against torch.stft with a random window, for windows of both parities up to N."""
    rs = np.random.RandomState(N)
    for W in sorted({1, 2, 3, N // 2, N // 2 + 1, N - 2, N - 1, N}):
        for L, hop in ((50, 7), (63, 9), (64, 8), (130, 13)):
            left, K, j = _stft_geometry(N, W)
            assert K % 64 == 0 and j >= 0 and j + W <= K, (N, W)
            h = torch.from_numpy(rs.standard_normal(W))
            x = torch.from_numpy(rs.standard_normal((1, L)))
            ref = torch.stft(x, N, hop_length=hop, win_length=W, window=h, center=True, pad_mode="constant",
                             onesided=False, return_complex=True)
            H = N // 2 + 1
            k, m = torch.arange(H)[:, None], torch.arange(W)[None, :]
            ang = 2 * np.pi * ((k * (m + left)) % N).double() / N
            w_re = torch.zeros((H, K), dtype=torch.float64)
            w_im = torch.zeros((H, K), dtype=torch.float64)
            w_re[:, j:j + W], w_im[:, j:j + W] = torch.cos(ang) * h, torch.sin(ang) * h
            A = fd.frames64(x, K, hop, True)
            assert A.shape[1] == L // hop + 1
            got = (A @ w_re.T - 1j * (A @ w_im.T)).transpose(1, 2)
            T = (L + 2 * (N // 2) - N) // hop + 1
            assert ref.shape[-1] == T
            np.testing.assert_allclose(got[..., :T].numpy(), ref[:, :H].numpy(), rtol=0, atol=1e-10 * L)


@pytest.mark.parametrize("name", HOST_ROWS)
def test_host_layer_is_exact(name, monkeypatch):
    """With exact float64 contractions (and the module's fp32 STFT / cosine banks checked against exact ones) the
    host layer equals the float64 oracle; a wrong mirror count, cut weight, mean restore or crop is O(1) off."""
    cpu_kernels.install(monkeypatch)
    mod = fd.build_row(name)
    monkeypatch.setattr(_C, "cqt1992v2_forward", fd.exact_forward(mod))
    B, L = _shape(name)
    x = fd.make_input(name, B, L)
    drop = fd.drops(name)
    got, want = _maps(mod, torch.from_numpy(x).double(), drop), fd.run_oracle(mod, x, drop)
    null = fd.row_options(name)["null"]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape, (name, i, g.shape, w.shape)
        if i in null:  # exactly zero: both within round-off of the frame-mean cancellation
            scale = np.abs(got[1]).max()
            assert np.abs(g).max() <= 1e-8 * scale and np.abs(w).max() <= 1e-8 * scale, (name, i)
            continue
        emax, el2 = _errors(g, w)
        assert emax <= EXACT_BAR and el2 <= EXACT_BAR, (name, i, emax, el2)


@pytest.mark.parametrize("name", sorted(fd.ROWS))
def test_row_builds_the_plan_it_claims(name):
    mod = fd.build_row(name)
    B, L = fd.ROWS[name][2]
    steps = fd.plan(mod, B, L, fd.drops(name))
    claims = fd.ROWS[name][4]
    stft, rs = steps[0]
    by_kind = {}
    for c, r in steps:
        by_kind.setdefault(c["stage"], set()).add(r["route"])
    left, K, j = _stft_geometry(mod.N, int(mod.window_size))
    have = dict(N=mod.N, K=K, j=j, kept=fd.kept_frames(mod, L, fd.drops(name)), layers=mod.NumofLayer,
                n_f=fd.crops(mod)[0], stft_ks=rs["ks"], stft_n_ph=rs["n_ph"], stft_rows_mode=rs["rows_mode"],
                stft_T=rs["T"])
    cos = [(c, r) for c, r in steps if c["stage"] == "cos"]
    if cos:
        have.update(cos_K=cos[0][0]["K"], cos_ks=cos[0][1]["ks"],
                    cos_m_tiles=-(-cos[0][0]["B"] * cos[0][1]["T"] // fd.TC_BM))
    for k, v in claims.items():
        if k in ("stft", "cos", "freq", "quef"):
            assert by_kind[k] == {v}, (name, k, [fd.ROUTE_NAMES[r] for r in by_kind[k]])
        else:
            assert have[k] == v, (name, k, have[k], v)
    # stage count: the STFT stage, then (with frames left) NumofLayer - 1 cosine stages and the two maps
    kept = fd.kept_frames(mod, L, fd.drops(name))
    assert len(steps) == (1 if kept == 0 else mod.NumofLayer + 2)
    assert all(r["route"] == fd.S and r["flops"] == 0.0 for _, r in fd.plan(mod, B, L, fd.drops(name), "simt"))


def test_matrix_reaches_every_route_of_every_stage():
    seen = {}
    for name in fd.ROWS:
        mod = fd.build_row(name)
        B, L = fd.ROWS[name][2]
        for c, r in fd.plan(mod, B, L, fd.drops(name)):
            key = c["stage"]
            if key == "cos" and r["route"] == fd.D and 4096 <= c["K"] < 8192:
                seen.setdefault(key, set()).add("dense_single_accumulator_k4096_8192")
            seen.setdefault(key, set()).add(fd.ROUTE_NAMES[r["route"]])
    assert {"dense", "dense_splitk", "simt"} <= seen["stft"], seen["stft"]
    assert {"dense", "dense_splitk", "simt", "dense_single_accumulator_k4096_8192"} <= seen["cos"], seen["cos"]


def test_flops_of_the_default_row_by_hand():
    """default, B = 2, L = 8000, hop 320: the STFT stage packs 4001 bins as 36 N tiles of 224 columns (8002 columns,
    the least padding within 128 tiles) over 2112 / 64 = 33 k-blocks; ceil((8000 + 2112) / 320) = 32 frame slots
    per clip, 64 frames = one M tile; three bf16 split terms of 2 flops per MAC."""
    mod = fd.build_row("default")
    (c, r) = fd.plan(mod, 2, 8000, False)[0]
    assert (r["bn"], r["n_tiles"], r["nkb"]) == (224, 36, 33)
    assert r["flops"] == 6.0 * 1 * 128 * 36 * 33 * 64 * 224
    cos_c, cos_r = fd.plan(mod, 2, 8000, False)[1]
    # 26 frames per clip, each a clip of one 4032-sample hop: 52 rows, one M tile, 2001 bins in the two banks
    assert (cos_c["K"], cos_c["F"], cos_r["T"]) == (4032, 2001, 26)
    assert cos_r["flops"] == 6.0 * 128 * cos_r["n_tiles"] * cos_r["bn"] * 4032


@pytest.mark.parametrize("name", HOST_ROWS)
def test_bars_cover_the_emulated_error(name, monkeypatch):
    """The row's end-to-end bar is >= 3x the error of the split-bf16 emulation of its routes (rows above 1e-3 are
    stage-only), and every stage's emulated ratio is <= TAU / 4 of its route."""
    cpu_kernels.install(monkeypatch)
    mod = fd.build_row(name)
    rec = []
    monkeypatch.setattr(_C, "cqt1992v2_forward", fd.emulated_forward(mod, record=rec))
    B, L = _shape(name)
    x = fd.make_input(name, B, L)
    drop = fd.drops(name)
    got, want = _maps(mod, torch.from_numpy(x), drop), fd.run_oracle(mod, x, drop)
    for stage, r, ratio in rec:
        assert ratio <= fd.TAU[r] / 4, (name, stage, fd.ROUTE_NAMES[r], ratio)
    emax, el2 = _errors(got[1], want[1])
    assert max(emax, el2) * 3 <= 1e-4, (name, "tfrL0", emax, el2)
    null = fd.row_options(name)["null"]
    worst = max([max(_errors(got[i], want[i])) for i in (0, 2, 3) if i not in null] + [0.0])
    bar = fd.row_options(name)["bar"]
    if bar is None:  # stage-only: the emulation is too far off, or the outputs are exactly zero (null)
        assert worst > STAGE_ONLY_ABOVE or null, (name, worst)
    else:
        assert worst * 3 <= bar, (name, worst, bar)


@pytest.mark.parametrize("name", ["default", "n16000_cos_k8064", "n22050_cos_splitk", "odd_n_fr3"])
def test_simt_tau_covers_the_fp32_emulation(name, monkeypatch):
    cpu_kernels.install(monkeypatch)
    mod = fd.build_row(name)
    rec = []
    monkeypatch.setattr(_C, "cqt1992v2_forward", fd.emulated_forward(mod, "simt", rec))
    B, L = _shape(name)
    _maps(mod, torch.from_numpy(fd.make_input(name, B, L)), fd.drops(name))
    assert rec and all(r == fd.S for _, r, _ in rec)
    for stage, r, ratio in rec:
        assert ratio <= fd.TAU[r] / 4, (name, stage, ratio)


def test_in_place_edits_reach_the_next_call(monkeypatch):
    """The STFT bank keys on h's _version, the maps on their buffers' _version: after a first call, editing each in
    place must change the next call's result to the oracle's for the edited buffers."""
    cpu_kernels.install(monkeypatch)
    mod = fd.build_row("comb_default")
    x = fd.make_input("comb_default")
    xt = torch.from_numpy(x).double()

    def check():
        monkeypatch.setattr(_C, "cqt1992v2_forward", fd.exact_forward(mod))
        for g, w in zip(_maps(mod, xt, True), fd.run_oracle(mod, x, True)):
            emax, el2 = _errors(g, w)
            assert emax <= EXACT_BAR and el2 <= EXACT_BAR, (emax, el2)

    check()
    with torch.no_grad():
        mod.h[: mod.h.shape[0] // 3] *= 0.5          # an asymmetric window: a different bank
    check()
    with torch.no_grad():
        mod.freq2logfreq_matrix[5:40] *= 2.0
    check()
    with torch.no_grad():
        mod.quef2logfreq_matrix[:, 3:50] += 0.25
    check()


def test_quefrency_crop_past_n_low_raises_like_the_oracle(monkeypatch):
    """fc < 2 fr puts HighQuefIdx past n_low: the quefrency map then has more columns than the transform keeps,
    which the reference's matmul refuses; so do the module and the oracle."""
    cpu_kernels.install(monkeypatch)
    mod = build("Combined_Frequency_Periodicity", dict(fr=8, fc=10, window_size=1025))
    assert mod.HighQuefIdx > fd.crops(mod)[1]
    monkeypatch.setattr(_C, "cqt1992v2_forward", fd.exact_forward(mod))
    x = np.random.RandomState(0).standard_normal((1, 4000)).astype(np.float32)
    with pytest.raises(RuntimeError, match="size mismatch"):
        _maps(mod, torch.from_numpy(x).double(), True)
    with pytest.raises(ValueError):
        fd.run_oracle(mod, x, True)


@pytest.mark.parametrize("name", ["default", "odd_n_fr3"])
def test_real_fft_half_is_the_full_vector_fft(name, monkeypatch):
    """``_real_fft_half`` on a half vector with a large DC term equals Re FFT_N of the full symmetric vector / sqrt(N)
    at every q, q = 0 included (the mean restore, which no cropped output shows: the cut-offs always remove q = 0),
    with the mirror weights and with the mirrored cut-off weights."""
    cpu_kernels.install(monkeypatch)
    mod = fd.build_row(name)
    monkeypatch.setattr(_C, "cqt1992v2_forward", fd.exact_forward(mod))
    N, H = mod.N, mod.N // 2 + 1
    n = torch.arange(N)
    mirror = torch.minimum(n, N - n)
    v = torch.from_numpy(np.random.RandomState(N).rand(2, H, 3)) + 50.0
    for c in (None, 1, 7, 0):
        if c is None:
            w_in, full = mod._mirror_count("cpu"), v[:, mirror]
        else:
            keep, w_in = mod._cut_weights(c, "cpu")
            full = (v * keep[None, :, None].double())[:, mirror]
            full[:, N - c if c else 0:] = 0
        want = torch.fft.fft(full, dim=1).real[:, :H] / np.sqrt(N)
        got = mod._real_fft_half(v if c is None else v * mod._cut_weights(c, "cpu")[0][None, :, None].double(),
                                 w_in.double())
        assert float((got - want).abs().max()) <= 1e-9 * float(want.abs().max() + 1), (name, c)
