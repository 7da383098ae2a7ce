"""No-GPU checks of CQT1992v2's shape matrix and route model (tests/cqt1992_domain.py): every row builds the
geometry and takes the route it claims, the matrix reaches every route counter of the library, the VarN chunk
model agrees with the library's own plan, and the flop model agrees with counts made by hand."""
import ctypes

import numpy as np
import pytest

import cqt1992_domain as cd
from helpers import build
from nnaudio_b200 import _C


def _module(name):
    cls, ctor = cd.ROWS[name][:2]
    return build(cls, ctor)


def _plans(name):
    cls, ctor, B, L = cd.ROWS[name][:4]
    mod = _module(name)
    opts = cd.row_options(name)
    return mod, [cd.plan(mod, B, L, opts["path"], tall_ctas=c) for c in opts["tall_ctas"]]


@pytest.mark.parametrize("name", sorted(cd.ROWS))
def test_row_builds_the_geometry_and_route_it_claims(name):
    geometry, route, claims = cd.ROWS[name][4:7]
    mod, plans = _plans(name)
    assert cd.geometry(mod) == geometry
    for p in plans:
        assert p["route"] == route, (name, cd.ROUTE_NAMES[p["route"]], cd.ROUTE_NAMES[route])
        assert p["T"] >= 1
        for k, v in claims.items():
            assert p[k] == v, (name, k, p[k], v)


def test_matrix_reaches_every_route():
    seen = set()
    for name in cd.ROWS:
        seen |= {p["route"] for p in _plans(name)[1]}
    assert seen == set(range(_C.CQ1992_ROUTES)), sorted(set(range(_C.CQ1992_ROUTES)) - seen)


def test_balanced_rows_are_static_on_the_full_grid():
    """Without NNAB_TALL_CTAS the 29 tiles of tall_balanced_forced fit one round of a 132-SM grid."""
    mod = _module("tall_balanced_forced")
    B, L = cd.ROWS["tall_balanced_forced"][2:4]
    p = cd.plan(mod, B, L)
    assert p["route"] == _C.CQ1992_TALL and p["tiles"] == 29 and p["grid"] == 29
    assert cd.plan(mod, B, L, tall_ctas=29)["route"] == _C.CQ1992_TALL  # a cap >= the grid changes nothing
    assert cd.plan(mod, B, L, tall_ctas=5, balance=False)["route"] == _C.CQ1992_TALL
    # too few clips: the split-K scratch cannot hold one 96 KB slot per CTA
    assert cd.plan(mod, 2, L, tall_ctas=5)["route"] == _C.CQ1992_TALL


def _library_varn_plan(sup, F, K, want):
    n = -(-K // 64)
    order, groups = (ctypes.c_int32 * n)(), (ctypes.c_int32 * n)()
    begin = (ctypes.c_int32 * 17)()
    n_blocks, n_chunks = ctypes.c_int32(0), ctypes.c_int32(0)
    b, e = (None, None) if sup is None else (np.ascontiguousarray(sup[0]), np.ascontiguousarray(sup[1]))
    rc = _C.lib().nnab_debug_varn_plan(_C._kb(b), _C._kb(e), F, K, want, order, groups, begin,
                                       ctypes.byref(n_blocks), ctypes.byref(n_chunks))
    assert rc == 0, rc
    nb, nc = n_blocks.value, n_chunks.value
    return list(groups[:nb]), list(order[:nb]), list(begin[:nc + 1])


@pytest.mark.parametrize("name", sorted(n for n in cd.ROWS if cd.ROWS[n][5] in (cd.V, cd.VS)))
def test_varn_model_agrees_with_the_library_plan(name):
    mod, (p,) = _plans(name)
    F, K, _ = cd.geometry(mod)
    sup = cd.support(mod)
    assert (p["groups"], p["order"], p["chunk_begin"]) == _library_varn_plan(sup, F, K, p["chunks"])
    # and the chunk count the launcher asks for: <= 64 active blocks per chunk
    probe = _library_varn_plan(sup, F, K, 1)
    assert p["chunks"] == min(-(-len(probe[0]) // 64), 16)
    for want in (1, 2, 5, 16, 40):  # the cut itself, at other chunk counts
        model = cd.varn_plan(cd.block_groups(sup, F, K), F, want)
        assert model == _library_varn_plan(sup, F, K, want), (name, want)


def test_varn_model_without_support():
    g = cd.block_groups(None, 60, 8192)
    assert g == [8] * 128
    assert cd.varn_plan(g, 60, 2) == _library_varn_plan(None, 60, 8192, 2)


def _active_cols(mod):
    kr = mod.cqt_kernels_real.detach().numpy()[:, 0]
    ki = mod.cqt_kernels_imag.detach().numpy()[:, 0]
    return (kr != 0) | (ki != 0)


def test_flops_of_the_tall_row_by_hand():
    """tall_hop64_k4096, B = 2, L = 8000: planes of ceil((8000 + 4096) / 64) = 189 frame slots per clip, 378
    frames = 3 M tiles; every K block inside the bank's active interval runs 16 rows per 8-bin group it reaches
    (at least one) over 64 taps, in three bf16 split terms of 2 flops per MAC."""
    mod = _module("tall_hop64_k4096")
    nz = _active_cols(mod)
    F, K = nz.shape
    cols = [kb for kb in range(K // 64) if nz[:, kb * 64:(kb + 1) * 64].any()]
    total = 0
    for kb in range(cols[0], cols[-1] + 1):
        rows = np.nonzero(nz[:, kb * 64:(kb + 1) * 64].any(axis=1))[0]
        total += 16 * max(int(rows.max()) // 8 + 1 if rows.size else 1, 1) * 64
    assert cols[-1] - cols[0] + 1 == 54
    want = 3 * 2 * 3 * 128 * total
    assert cd.expected_exec_flops(mod, 2, 8000) == want
    assert cd.expected_route(mod, 2, 8000) == {_C.CQ1992_TALL: 1}


def test_flops_of_the_dense_rows_by_hand():
    """dense_k2048, B = 3, L = 8000: one N tile of 96 columns (48 bins), ceil((8000 + 2048) / 256) = 40 slots per
    clip, 120 frames = 1 M tile, one frame phase, K blocks spanning the bank's non-zero taps.  dense_hop441 has 8
    frame phases; with 5 frames (center=False) only 5 of them launch."""
    mod = _module("dense_k2048")
    nz = _active_cols(mod)
    taps = np.nonzero(nz.any(axis=0))[0]
    blocks = -(-(int(taps[-1]) + 1) // 64) - int(taps[0]) // 64
    assert cd.expected_exec_flops(mod, 3, 8000) == 3 * 2 * 1 * 128 * blocks * 64 * 96
    few = _module("dense_hop441_fewframes")
    full = build("CQT1992v2", dict(cd.ROWS["dense_hop441_fewframes"][1], center=False))
    L = 16384 + 441 * 4
    assert cd.frames(few, L)[1] == 5
    p5, p9 = cd.plan(few, 2, L), cd.plan(full, 2, L + 441 * 4)
    assert p5["launched"] == 5 and p9["launched"] == 8
    slots = lambda n: -(-n // (441 * 8))  # noqa: E731
    assert p5["flops"] * 8 * (-(-2 * slots(L + 441 * 4) // 128)) == p9["flops"] * 5 * (-(-2 * slots(L) // 128))


def test_simt_adds_no_flops():
    mod = _module("simt_base")
    assert cd.expected_exec_flops(mod, 2, 22050, "simt") == 0.0


def test_route_counter_bounds():
    """Host-only query: any value outside the NNAB_CQ1992_* range reads 0."""
    for r in (-1, _C.CQ1992_ROUTES, 1 << 20):
        assert _C.cqt1992v2_route_count(r) == 0
    assert all(_C.cqt1992v2_route_count(r) >= 0 for r in range(_C.CQ1992_ROUTES))
