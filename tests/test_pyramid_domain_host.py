"""No-GPU checks of the CQT pyramid's shape matrix and route model (tests/pyramid_domain.py): every row builds the
geometry it claims, the level model agrees with the module's own length plan, the route model follows the C rules it
restates, and the matrix reaches every route counter of the library."""
import warnings

import pytest

import pyramid_domain as pd
from helpers import build
from nnaudio_b200 import _C
from nnaudio_b200.features.cqt import _octave_plan


def _module(name):
    cls, ctor = pd.ROWS[name][:2]
    return build(cls, ctor)


@pytest.mark.parametrize("name", sorted(pd.ROWS))
def test_row_builds_the_geometry_it_claims(name):
    n_octaves, widths, F, hop, factor = pd.ROWS[name][4]
    mod = _module(name)
    assert mod.n_octaves == n_octaves
    assert pd.bank_shapes(mod) == (F, widths)
    assert mod.hop_length == hop
    assert pd.early_factor(mod) == factor


@pytest.mark.parametrize("name", sorted(pd.ROWS))
def test_levels_agree_with_the_module_plan(name):
    mod = _module(name)
    B, near = pd.ROWS[name][2:4]
    L = pd.valid_length(mod, near)
    assert pd.valid_length(mod, L) == L
    lv = pd.levels(mod, L)
    f = pd.early_factor(mod)
    L0 = (L - 2) // f + 1 if f > 1 else L
    T, fallbacks = _octave_plan(L0, mod.hop_length, [l.width for l in lv], mod.pad_mode)
    assert lv[0].len == L0 and lv[0].hop == mod.hop_length
    for i, l in enumerate(lv):
        if i:
            assert l.len == (lv[i - 1].len - 2) // 2 + 1 and l.hop == lv[i - 1].hop // 2
        assert l.pad == l.width // 2
        assert l.mode == ("constant" if fallbacks[i] else mod.pad_mode)
        assert (l.len + 2 * l.pad - l.width) // l.hop + 1 == T, (i, l)


def test_valid_length_skips_lengths_the_module_rejects():
    """A hop that does not halve exactly (300 -> 150 -> 75 -> 37) gives octaves different frame counts at
    most lengths; valid_length finds the nearest one they agree at.  (Every hop of the matrix halves exactly down
    to its last octave or the early factor divides it, so every length is valid there.)"""
    mod = build("CQT2010v2", dict(sr=22050, n_bins=48, hop_length=300, earlydownsample=False))
    valid = [n for n in range(19000, 21000) if _valid(mod, n)]
    assert 0 < len(valid) < 1000
    L = pd.valid_length(mod, 20000)
    assert L in valid and all(abs(n - 20000) >= abs(L - 20000) for n in valid)
    with pytest.raises(RuntimeError, match="Sizes of tensors must match"):
        pd.levels(mod, next(n for n in range(19000, 21000) if n not in valid))


def _valid(mod, n):
    try:
        pd.levels(mod, n)
        return True
    except RuntimeError:
        return False


@pytest.mark.parametrize("F,K,hop,ok", [
    (12, 256, 512, True), (12, 256, 2048, True), (12, 256, 64, True), (12, 256, 8, True),
    (12, 256, 4, False),        # not a presplit level
    (12, 256, 448, False),      # hop % 64 != 0
    (12, 256, 192, False),      # hb = 3 is not a power of two
    (12, 256, 24, False),       # does not divide 64
    (24, 256, 512, False),      # F > 16
    (12, 4096, 512, False),     # 64 K blocks
    (12, 512, 512, True), (12, 576, 512, False),  # 8 / 9 K blocks
    (12, 200, 512, False),      # not whole K blocks
    (12, 512, 8, True),         # (8 - 1) / 1 = 7 row shifts
])
def test_octave_kernel_rule(F, K, hop, ok):
    assert pd.octave_tc_ok(F, K, hop, 2) is ok


def test_route_model_plan_order():
    """A 16-bit waveform has no per-octave plan; the plans above it take it as is."""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        base = _module("gen2_base")
        early = _module("gen1_early2")
    assert pd.expected_routes(base, 3, 20000, "bfloat16") == pd.expected_routes(base, 3, 20000)
    assert pd.expected_routes(early, 2, 40000, "float16")[_C.PYR_PLAN_GEN1] == 1
    assert pd.expected_routes(base, 3, 20000, "bfloat16", path="simt") is None
    assert pd.expected_routes(base, 3, 20000, "float16", lowpass_packed=False) is None
    # B beyond the pre-pass grid: neither fused plan
    assert pd.expected_routes(base, 70000, 20000)[_C.PYR_PLAN_PER_OCTAVE] == 1


def test_matrix_reaches_every_route():
    seen = set()
    for name in pd.ROWS:
        opts = pd.row_options(name)
        mod = _module(name)
        B, near = pd.ROWS[name][2:4]
        seen |= set(pd.expected_routes(mod, B, pd.valid_length(mod, near), "float32", opts["path"],
                                       opts["lowpass_packed"]))
    assert seen == set(range(_C.PYR_ROUTES)), sorted(set(range(_C.PYR_ROUTES)) - seen)


def test_route_counter_bounds():
    """Host-only query: any value outside the NNAB_PYR_* range reads 0."""
    for r in (-1, _C.PYR_ROUTES, 1 << 20):
        assert _C.pyramid_route_count(r) == 0
    assert all(_C.pyramid_route_count(r) >= 0 for r in range(_C.PYR_ROUTES))
