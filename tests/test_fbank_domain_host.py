"""CPU checks of tests/fbank_domain.py: every row builds the bank and plan it claims, the plan's fused width and
warp-specialised flag agree with a bin-by-bin replay of fb_steps_kernel's range cuts, the matrix reaches every
(route, kernel) cell, the float64 references equal the oracle, the MFCC tail bound holds for an emulated fp32
tail, and the crafted edits change the support as claimed (tests/test_zz_gpu_fbank_domain.py then holds the GPU
to all of it)."""
import warnings

import numpy as np
import pytest

import block_domain as bd
import dense_domain as dd
import fbank_domain as fd
from helpers import build, run_oracle


@pytest.fixture(scope="module")
def banks():
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # empty mel filters are part of the matrix
        return {name: fd.bank(name) for name in fd.ROWS}


@pytest.mark.parametrize("name", sorted(fd.ROWS))
def test_row_builds_the_bank_and_plan_it_claims(name, banks):
    fb = banks[name]
    p = fd.row_plan(name, fb)
    props = fd.properties(fb, p)
    claims = fd.ROWS[name][4]
    assert all(p.get(k, props.get(k)) == v for k, v in claims.items()), (name, p, props, claims)
    if fd.BLK in p["routes"]:
        # the fused width, and whether it is deterministic, replayed bin by bin over fb_steps_kernel's cuts
        nb, det, worst = fd.replay_widths(fb, p["K"], p["hop"])
        if fd.FUSED in p["routes"]:
            assert (nb, det) == bd.fbank_nb(fb, p["K"], p["hop"]), name
            assert p["nb"] == nb and (worst[nb] <= 2) == det, name
            assert p["deterministic"] == (det and fd.power_of(name) == 2.0), name
            if bd.poly4(p["hop"]):
                assert max(bd.bp.fb_ranges(fb, nb)) == worst[nb], name
        else:
            assert p["nb"] == bd.bp.choose_nb(bd.basis_bins(p["K"], p["hop"])) and p["deterministic"], name
        assert p["ws"] == int(bd.poly4(p["hop"]) and p["nb"] <= bd.WS_NB_MAX and fd.GEMM not in p["routes"])
    else:
        assert p["nb"] is None and p["ws"] == 0, name


def test_the_matrix_reaches_every_cell(banks):
    cells = {}
    for name in fd.ROWS:
        cells.setdefault(fd.cell(fd.row_plan(name, banks[name])), []).append(name)
    assert set(cells) == fd.CELLS, sorted(cells)
    # power 1, 1.5 and 2 on the fused WS, fused plain four-phase and planes routes
    for c in (("fused", "ws"), ("fused", "ph4"), ("planes", "ws")):
        powers = {fd.power_of(n) for n in cells[c]} | ({fd.power_of(n) for n in cells[("planes", "ph4")]}
                                                      if c[0] == "planes" else set())
        assert powers >= {1.0, 1.5, 2.0}, (c, powers)
    # both determinism outcomes on the fused four-phase kernels, and the planes GEMM at 1 and 2 N tiles
    for c in (("fused", "ws"), ("fused", "ph4")):
        assert {fd.row_plan(n, banks[n])["deterministic"] for n in cells[c]} == {True, False}, c
    fh = {(banks[n].shape[0] + 1) // 2 for n in cells[("planes", "ws")]}
    assert min(fh) <= 128 < max(fh)


def test_mfcc_rows_reach_the_tail_edges(banks):
    rows = [n for n in fd.ROWS if fd.ROWS[n][0] == "MFCC"]
    n_mfcc = {fd.ROWS[n][1].get("n_mfcc", 20) for n in rows}
    assert {1, 32, 33, 64} <= n_mfcc
    n_mels = {banks[n].shape[0] for n in rows}
    assert min(n_mels) < 20 and {400, 1600, 2048} <= n_mels
    assert max(n_mels) > fd.MFCC_MEL_SLICE
    assert any(fd.cell(fd.row_plan(n, banks[n]))[0] == "planes" for n in rows)
    long_rows = [n for n in rows if banks[n].shape[0] * fd.row_plan(n, banks[n])["T"] > fd.CLIP_MAX_CELLS]
    assert long_rows


def test_long_clip_output_depends_on_the_strided_peak():
    """mfcc_long_clip: each clip's peak cell lies past the first CLIP_MAX_CELLS cells of its (n_mels, T) block, so
    only a later stride of clip_max_kernel's capped grid reads it, and the top_db floor binds: a per-clip maximum
    that missed those cells would move the coefficients by far more than the 1e-4 bar."""
    from nnaudio_b200 import design
    name = "mfcc_long_clip"
    c = fd.module_ctor(name)
    fb = fd.bank(name)
    S = fd.ref_output(fd.row_input(name), fb, c["n_fft"], c["hop_length"], 2.0)
    n_mels, T = S.shape[1:]
    assert n_mels * T > fd.CLIP_MAX_CELLS
    flat = S.reshape(S.shape[0], -1)
    assert (flat.argmax(axis=1) >= fd.CLIP_MAX_CELLS).all()
    dct = design.dct2_ortho_matrix(20, n_mels)
    amin, ref, top_db = 1e-10, 1.0, c["top_db"]
    want, v = fd.mfcc_tail(S, dct, amin, ref, top_db)
    floor = v.min(axis=(1, 2))
    assert ((v == floor[:, None, None]).mean(axis=(1, 2)) > 0.5).all(), "the floor clamps most cells"
    # the same tail with the peak of the cells the grid's first strides reach only
    early = flat[:, :fd.CLIP_MAX_CELLS].max(axis=1)
    v_early = 10.0 * np.log10(np.maximum(S, amin))
    v_early = np.maximum(v_early, (10.0 * np.log10(early) - top_db)[:, None, None])
    moved = np.abs(np.matmul(dct, v_early) - want).max() / np.abs(want).max()
    assert moved > 100 * 1e-4, moved


@pytest.mark.parametrize("edit,claim", [("negate_odd", 2), ("extra_nonzero", 3), ("zero_rows", 2)])
def test_crafted_edits_change_the_support_as_claimed(edit, claim):
    fb = fd.bank("cfg2_bank")
    nz = fb != 0
    ed = fb.copy()
    fd.EDITS[edit](ed)
    assert dd.fb_entries(ed)[1] == claim
    if edit == "negate_odd":
        np.testing.assert_array_equal(ed != 0, nz)
        assert (ed[1::2] <= 0).all() and (ed[::2] >= 0).all()
        assert fd.replay_widths(ed, 2048, 512)[:2] == fd.replay_widths(fb, 2048, 512)[:2]
    elif edit == "extra_nonzero":
        assert (ed != fb).sum() == 1
    else:
        assert (~(ed != 0).any(axis=1)).sum() == 3 and (~nz.any(axis=1)).sum() == 0


@pytest.mark.parametrize("case", ["mel_small", "mel_cfg2_shape", "gammatone_small", "mfcc_cfg5_shape",
                                  "mfcc_small_no_topdb", "mfcc_more_coefficients_than_mels"])
def test_references_equal_the_oracle(case):
    from helpers import CASES, case_input
    if case == "mfcc_more_coefficients_than_mels":
        cls, ctor = "MFCC", dict(sr=16000, n_mfcc=20, n_mels=16, n_fft=512, hop_length=128)
        x = np.random.RandomState(4).standard_normal((2, 6000)).astype(np.float32)
    else:
        _, cls, ctor, inp, _ = next(c for c in CASES if c[0] == case)
        x = case_input(case, inp)
    mod = build(cls, ctor)
    mel = mod.melspec_layer if cls == "MFCC" else mod
    fbt = mel.gammatone_basis if cls == "Gammatonegram" else mel.mel_basis
    fb = fbt.numpy().astype(np.float64)
    K, hop = mel.n_fft, mel.stride
    S = fd.ref_output(x, fb, K, hop, float(mel.power))
    if cls == "MFCC":
        got = dd.ref_mfcc(S, mod.n_mfcc, mod._amin_host, mod._ref_host, mod.top_db)
        # the same tail written out: dB, floor, the module's fp32 DCT rows (n_mfcc > n_mels: n_mels rows)
        tail = fd.mfcc_tail(S, mod._dct_rows.numpy(), mod._amin_host, mod._ref_host, mod.top_db)[0]
        assert tail.shape == got.shape
        assert np.abs(tail - got).max() <= 1e-7 * np.abs(got).max()
    else:
        got = S
    want = run_oracle(cls, mod, x, {})
    assert got.shape == want.shape
    # the Hann basis in float64 against the module's fp32 buffers
    assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max(), case


@pytest.mark.parametrize("n_mels,n_mfcc,top_db,ref,amin,levels", [
    (128, 20, 80.0, 1.0, 1e-10, (1.0, 1e-3, 1e-6, 0.0)),
    (40, 33, None, 0.5, 1e-10, (1.0, 1e-2)),
    (400, 40, 0.0, 1e-12, 1e-10, (1.0, 1.0)),
    (2048, 40, 80.0, 2.0, 1e-5, (1.0, 1e-4)),
])
def test_tail_bound_holds_for_an_emulated_fp32_tail(n_mels, n_mfcc, top_db, ref, amin, levels):
    """fp32 dB (log2 rounded, times 10 log10 2 rounded, minus ref_dB rounded) and a sequential fp32 DCT sum (two
    roundings per term, coarser than the kernel's fmaf) stay inside fd.tail_bound."""
    from nnaudio_b200 import design
    rng = np.random.RandomState(n_mels)
    T = 7
    S = (rng.standard_normal((len(levels), n_mels, T)) ** 2 * np.asarray(levels)[:, None, None] ** 2)
    S = S.astype(np.float32)
    dct32 = design.dct2_ortho_matrix(min(n_mfcc, n_mels), n_mels).astype(np.float32)
    want, v = fd.mfcc_tail(S, dct32, amin, ref, top_db)
    f32 = np.float32
    ref_db = f32(10.0 * np.log10(max(amin, abs(ref))))
    v32 = (f32(3.0102999566) * np.log2(np.maximum(S, f32(amin))).astype(f32)).astype(f32) - ref_db
    if top_db is not None:
        peak = (f32(3.0102999566) * np.log2(np.maximum(S, f32(amin)).max(axis=(1, 2)))).astype(f32) - ref_db
        v32 = np.maximum(v32, (peak - f32(top_db))[:, None, None])
    acc = np.zeros((len(levels), dct32.shape[0], T), dtype=f32)
    for m in range(n_mels):
        acc = (acc + (dct32[None, :, m, None] * v32[:, None, m, :]).astype(f32)).astype(f32)
    excess = np.abs(acc - want) / fd.tail_bound(dct32, v)
    assert excess.max() <= 1.0, float(excess.max())
    if levels[-1] == 0.0:  # the fp32 DCT rows round at ~6e-8
        np.testing.assert_allclose(want[-1, 0], fd.silent_c0(n_mels, amin, ref), rtol=1e-7)
        assert np.abs(want[-1, 1:]).max() <= 1e-7 * abs(fd.silent_c0(n_mels, amin, ref))
