"""No-GPU checks of tests/grid_domain.py's persistent-grid model and of the host side of the SM reserve and the
persistent-grid ledger: the matrix has the shapes it claims (many units per CTA at G = 1, ragged last rounds, a
row that work rather than the reserve limits, ring phases that cross units, the tall kernel's schedule switching
with G), every persistent kernel family is reached, and the model agrees with the domain models it is built on."""
import pytest

import cqt1992_domain as cd
import grid_domain as gd
from nnaudio_b200 import _C

SMS = 132  # an H100 SXM; the model takes the device's count on the GPU


@pytest.fixture(scope="module")
def models():
    out = {}
    for name in gd.ROWS:
        mod = gd.build_module(name)
        out[name] = (mod, {G: gd.model(name, mod, G, SMS) for G in gd.GRIDS})
    return out


@pytest.mark.parametrize("name", sorted(gd.ROWS))
def test_row_model(name, models):
    row = gd.ROWS[name]
    mod, ms = models[name]
    full = ms[None]
    for G, m in ms.items():
        g = SMS if G is None else G
        units = [u for _, u, _ in m["launches"]]
        assert m["grids"] == [min(u, g) for u in units]
        assert m["ledger"] == (len(units), sum(m["grids"]), min(m["grids"]), max(m["grids"]))
        # the launches, their units and the flops do not depend on the grid
        assert [(k.replace("tall_balanced", "tall"), u, kb) for k, u, kb in m["launches"]] == \
               [(k.replace("tall_balanced", "tall"), u, kb) for k, u, kb in full["launches"]]
        assert m["flops"] == full["flops"] > 0
        if G == 1:
            assert m["ledger"] == (len(units), len(units), 1, 1)
            if not row.get("small"):
                assert min(units) >= 8, (name, units)  # every CTA of a G = 1 launch walks >= 8 units
    if row.get("small"):
        assert max(u for _, u, _ in full["launches"]) < 7, name
        assert ms[7]["grids"] == full["grids"], "work, not the reserve, sets this row's grids"
    if row["family"] == "cqt1992":
        # the route the CQT1992v2 domain model gives at each grid
        for G, m in ms.items():
            r = cd.plan(mod, row["B"], row["L"], sms=SMS if G is None else G)["route"]
            assert ("cq1992", r) in m["routes"], (name, G)


def test_matrix_claims(models):
    # a launch whose last round is ragged (units % G != 0): in most rows at G = 3 and 7; at G = 2 in 40 % of them
    # (the N-tile counts of the block-partial and split-K rows are even)
    for G, share in ((2, 0.4), (3, 0.5), (7, 0.5)):
        ragged = [n for n, (_, ms) in models.items() if any(u % G for _, u, _ in ms[G]["launches"])]
        assert len(ragged) > share * len(gd.ROWS), (G, sorted(set(gd.ROWS) - set(ragged)))
    assert any(row.get("small") for row in gd.ROWS.values())
    # a K-block count per unit that is not a multiple of the ring depth: the ring's parity crosses a unit
    # (the tall and per-K-block-width kernels read CQT banks whose supports are symmetric about the kernel centre:
    # their active block counts are even, so no such row exists for them)
    for kernel in ("dense",):
        assert any(kb % gd.STAGES[kernel] for _, ms in models.values()
                   for k, _, kb in ms[1]["launches"] if k.startswith(kernel)), kernel
    # (the block-partial ring is 2 to 4 stages deep: 5 K blocks are a multiple of none of those)
    assert 5 in {kb for _, ms in models.values() for k, _, kb in ms[1]["launches"] if k == "block"}


def test_tall_schedule_switches_with_the_grid(models):
    _, ms = models["cqt1992_tall"]
    assert ms[1]["launches"][0][0] == "tall" and ms[None]["launches"][0][0] == "tall"
    balanced = [G for G in (2, 3, 7) if ms[G]["launches"][0][0] == "tall_balanced"]
    assert balanced == [2, 3, 7]
    for G in balanced:
        assert ms[G]["routes"][("balanced", None)] == 1 and ms[G]["bitwise_key"] == ("G", G)
    assert ms[1]["bitwise_key"] == ms[None]["bitwise_key"] == "all"
    _, ms = models["cqt1992_tall_hop64"]
    assert all(m["launches"][0][0] == "tall" for m in ms.values()), "no split-K scratch: static only"


def test_every_persistent_kernel_has_a_row(models):
    reached = set()
    for _, ms in models.values():
        for m in ms.values():
            reached |= gd.kernels_of(m)
    assert reached == set(gd.KERNELS), set(gd.KERNELS) - reached
    fams = {row["family"] for row in gd.ROWS.values()}
    assert {"dense", "dense_direct", "block", "fbank", "planes", "cqt1992", "istft", "dx", "pyramid"} <= fams
    routes = set()
    for _, ms in models.values():
        for m in ms.values():
            routes |= set(m["routes"])
    for r in (("stft", _C.STFT_DENSE), ("stft", _C.STFT_DENSE_SPLITK), ("stft", _C.STFT_BLOCK),
              ("stft", _C.STFT_FB_FUSED), ("stft", _C.STFT_FB_PLANES), ("cq1992", _C.CQ1992_TALL),
              ("cq1992", _C.CQ1992_TALL_BALANCED), ("cq1992", _C.CQ1992_VARN), ("cq1992", _C.CQ1992_VARN_SPLITK),
              ("cq1992", _C.CQ1992_DENSE), ("cq1992", _C.CQ1992_DENSE_SPLITK), ("pyr", _C.PYR_PLAN_GEN2),
              ("pyr", _C.PYR_PLAN_GEN1), ("pyr", _C.PYR_OCT_KERNEL), ("pyr", _C.PYR_OCT_DENSE_PLANES),
              ("pyr", _C.PYR_FIR_BANDED), ("pyr", _C.PYR_FIR_DENSE), ("ws", None)):
        assert r in routes, r


def test_ordered_and_unordered_rows(models):
    unordered = {n for n, (_, ms) in models.items() if not ms[None]["ordered"]}
    assert unordered == {"istft_256", "dx_256", "block_mel_rolled"}
    for n in unordered:
        assert all(m["bitwise_key"] is None for m in models[n][1].values()), n


def test_sm_reserve_round_trip_is_host_only():
    old = _C.set_sm_reserve(1000)
    try:
        assert _C.set_sm_reserve(old) == 1000, "a reserve above 64 SMs is kept (a one-CTA grid on any device)"
    finally:
        _C.set_sm_reserve(old)
    assert _C.set_sm_reserve(-5) == old and _C.set_sm_reserve(old) == 0, "negative reserves become 0"


def test_persistent_grid_ledger_reads_zero_without_launches():
    _C.persistent_grid_read()  # drops whatever an earlier test launched
    assert _C.persistent_grid_read() == (0, 0, 0, 0)
