"""Level model, route model and shape matrix of the CQT pyramid (``nnab_cqt_pyramid_forward``, csrc/nnab_api.cu), shared
by tests/test_pyramid_domain_host.py (CPU) and tests/test_zz_gpu_pyramid_domain.py (-m gpu).

``expected_routes`` restates, in Python, how one call picks its plan (gen-2, gen-1 or per-octave) and, inside the
plan, the route of every octave and FIR stage.  A GPU test compares it with the library's route counters
(``_C.pyramid_route_count``), so a shape that silently falls through to a slower route fails on the counters even
when its numbers still match the float64 reference."""
from collections import Counter, namedtuple

import helpers  # noqa: F401  (puts the repository on sys.path)
from block_domain import choose_bn
from nnaudio_b200 import _C
from nnaudio_b200.features.cqt import _decimated_len, _octave_levels, _octave_plan

Level = namedtuple("Level", "len hop width pad mode")

MAX_B = 65535       # select_fused2 / select_fused: the pre-pass kernels put the clip index in gridDim.y
MAX_OCTAVES = 32    # the plans' level arrays
OCT_MAX_KB = 8      # tct_kernels.cu: K blocks of the octave kernel's resident bank
TC_MAX_N_TILES = 128


def early_factor(mod):
    return int(mod.downsample_factor) if mod.earlydownsample else 1


def bank_shapes(mod):
    """(n_filters, per-octave bank widths) of a CQT2010v2 / VQT / CQT2010 module, read from its buffers on the
    host (the folded CQT2010 bank is n_fft wide, like the DFT rows it is folded with)."""
    if hasattr(mod, "cqt_kernels_real_0"):  # VQT: one bank per octave
        banks = [getattr(mod, f"cqt_kernels_real_{i}") for i in range(mod.n_octaves)]
        return int(banks[0].shape[0]), [int(b.shape[-1]) for b in banks]
    F = int(mod.cqt_kernels_real.shape[0])
    width = int(mod.wcos.shape[-1]) if hasattr(mod, "wcos") else int(mod.cqt_kernels_real.shape[-1])
    return F, [width] * mod.n_octaves


def levels(mod, L):
    """Per-octave Level(len, hop, width, pad, mode) of ``mod`` on clips of ``L`` samples: the early stage's
    length rule, then the ÷2 pyramid (features.cqt).  ``mode`` is the pad mode the octave runs with: reflect
    falls back to constant when pad >= len.  Raises like the module does when the octaves' frame counts differ."""
    f = early_factor(mod)
    L0 = _decimated_len(L, f) if f > 1 else L
    _, widths = bank_shapes(mod)
    _, fallbacks = _octave_plan(L0, mod.hop_length, widths, mod.pad_mode)
    lens, hops = _octave_levels(L0, mod.hop_length, len(widths))
    return [Level(n, h, w, w // 2, "constant" if fb else mod.pad_mode)
            for n, h, w, fb in zip(lens, hops, widths, fallbacks)]


def valid_length(mod, near):
    """The clip length nearest ``near`` (the shorter one on a tie) at which every octave has the same frame count."""
    for d in range(0, near):
        for L in (near - d, near + d):
            try:
                levels(mod, L)
                return L
            except RuntimeError:
                pass
    raise ValueError(f"no valid length near {near}")


# ------------------------------------------------------------------------------------------- route model ----
def presplit(hop):
    """plan_pyramid / plan_pyramid2 (nnab_api.cu: `l.presplit = ... (cur_hop % 8) == 0`): the octave reads the
    level's planes at one frame phase; other hops run from the fp32 level, split per frame phase."""
    return hop > 0 and hop % 8 == 0


def dense_ok(F, K):
    """tc_supported (tc_kernels.cu) for a dense bank: K >= 16 and at most TC_MAX_N_TILES N tiles of choose_bn.
    (Its row / plane-size limits hold for every shape of the matrix.)"""
    return K >= 16 and -(-2 * F // choose_bn(F)) <= TC_MAX_N_TILES


def octave_tc_ok(F, K, hop, B):
    """octave_tc_ok (tct_kernels.cu) of a gen-2 octave on its level planes: tc_tile_n(F) == 32 (F <= 16), whole
    K blocks, at most OCT_MAX_KB of them, a hop that is a multiple of 64 with a power-of-two number of 64-column
    blocks hb or a divisor of 64 of at least 8, and row shifts (K / 64 - 1) / hb <= 8.  Its last test, planes
    whose row pitch is a multiple of the effective hop, holds by construction in plan_pyramid2 (pitch is a
    multiple of lcm(hop, 256)).  The pyramid's formats are all ones the kernel has an epilogue for."""
    if not presplit(hop) or F > 16 or K % 64 != 0 or K // 64 > OCT_MAX_KB or B > MAX_B:
        return False
    if (hop % 64 != 0) if hop >= 64 else (hop < 8 or 64 % hop != 0):
        return False
    hb = max(hop, 64) // 64
    return hb & (hb - 1) == 0 and (K // 64 - 1) // hb <= 8


def gen2_ok(lv, F, B, f):
    """select_fused2 / plan_pyramid2 (nnab_api.cu): no early stage (`all_packed && early_factor <= 1`), every
    level non-empty, every FIR source level (all but the last) padded by exactly 128 (256- or 257-wide bank:
    the FIR frame origin is the CQT padding origin), and every octave on the octave kernel or the dense one."""
    if f > 1 or B > MAX_B or len(lv) > MAX_OCTAVES:
        return False
    if any(l.len <= 0 or l.hop <= 0 for l in lv) or any(l.pad != 128 for l in lv[:-1]):
        return False
    return all(octave_tc_ok(F, l.width, l.hop, B) or dense_ok(F, l.width) for l in lv)


def gen1_ok(lv, F, B):
    """select_fused (nnab_api.cu): tc_supported for every octave (the FIR stages, 64 outputs per row of a
    256-tap band, always are)."""
    return B <= MAX_B and len(lv) <= MAX_OCTAVES and all(dense_ok(F, l.width) for l in lv)


def packed_ok(F, K):
    """pack_basis gives a packed bank (nnab_packed_basis_bytes > 0)."""
    return _C.lib().nnab_packed_basis_bytes(int(F), int(K)) > 0


def expected_routes(mod, B, L, dtype="float32", path="auto", lowpass_packed=True):
    """Counter deltas (route -> count, PYR_* constants) of one ``nnab_cqt_pyramid_forward`` call of ``mod`` on
    (B, L) clips of ``dtype`` under kernel family ``path`` ("auto" / "simt"), or None when the call returns
    NNAB_EUNSUPPORTED before enqueuing anything (a 16-bit waveform on the per-octave plan; the module then
    reruns the fp32 upcast, and ``strict_dtype=True`` raises instead).  ``lowpass_packed=False`` is a caller that
    passes no packed FIR.  The plan order is nnab_cqt_pyramid_forward_ex's: gen-2, else gen-1, else per-octave."""
    lv = levels(mod, L)
    F, _ = bank_shapes(mod)
    f = early_factor(mod)
    n = len(lv)
    all_packed = path != "simt" and lowpass_packed and all(packed_ok(F, l.width) for l in lv)
    r = Counter()
    if all_packed and gen2_ok(lv, F, B, f):
        r[_C.PYR_PLAN_GEN2] = 1
        for l in lv:  # pyramid_fused2: octave kernel, else dense on the planes, else dense from fp32
            r[_C.PYR_OCT_KERNEL if octave_tc_ok(F, l.width, l.hop, B)
              else _C.PYR_OCT_DENSE_PLANES if presplit(l.hop) else _C.PYR_OCT_DENSE_FP32] += 1
        r[_C.PYR_FIR_BANDED] = n - 1
    elif all_packed and gen1_ok(lv, F, B):
        r[_C.PYR_PLAN_GEN1] = 1
        for l in lv:  # pyramid_fused: dense on the level planes, else dense from fp32
            r[_C.PYR_OCT_DENSE_PLANES if presplit(l.hop) else _C.PYR_OCT_DENSE_FP32] += 1
        r[_C.PYR_FIR_DENSE] = n - 1 + (f > 1)
    else:
        if dtype != "float32":  # the per-octave FIR stages read the waveform as fp32
            return None
        r[_C.PYR_PLAN_PER_OCTAVE] = 1
        for l in lv:  # a packed bank the dense kernel takes (the workspace query sizes its scratch)
            tc = path != "simt" and packed_ok(F, l.width) and dense_ok(F, l.width)
            r[_C.PYR_OCT_TC_LOOP if tc else _C.PYR_OCT_SIMT] += 1
        r[_C.PYR_FIR_SIMT] = n - 1 + (f > 1)
    return {k: v for k, v in r.items() if v}


# -------------------------------------------------------------------------------------------- the matrix ----
# name -> (class, constructor, B, length to search near, geometry the row claims, run options).  Geometry:
# n_octaves, widths, F, hop (after the early stage), early factor.  Options: formats, normalizations, path,
# lowpass_packed.  White noise; earlydownsample=False unless the row is about the early stage.
_V2 = dict(sr=22050, n_bins=84, hop_length=512, earlydownsample=False)
_W256 = [256] * 7
ALL = dict(formats=("Complex", "Magnitude", "Phase"), norms=("librosa", "convolutional", "wrap"))
ROWS = {
    # gen-2: 7 octaves on the octave kernel (the bottom hop 8 runs as 8 frame phases), 6 banded FIR stages
    "gen2_base": ("CQT2010v2", _V2, 3, 20000, (7, _W256, 12, 512, 1), ALL),
    # octave kernel down to hop 8, then the dense kernel from fp32 at hops 4, 2, 1
    "gen2_hop256": ("CQT2010v2", dict(_V2, hop_length=256), 2, 20000, (7, _W256, 12, 256, 1), {}),
    "gen2_hop128": ("CQT2010v2", dict(_V2, hop_length=128), 2, 20000, (7, _W256, 12, 128, 1), {}),
    "gen2_hop64": ("CQT2010v2", dict(_V2, hop_length=64), 2, 12000, (7, _W256, 12, 64, 1), {}),
    # hops the octave kernel does not take: dense on the level planes while hop % 8 == 0, then fp32
    "gen2_hop448": ("CQT2010v2", dict(_V2, hop_length=448), 2, 20000, (7, _W256, 12, 448, 1), {}),
    "gen2_hop192": ("CQT2010v2", dict(_V2, hop_length=192), 2, 20000, (7, _W256, 12, 192, 1), {}),
    "gen2_hop768": ("CQT2010v2", dict(_V2, hop_length=768), 2, 30000, (7, _W256, 12, 768, 1), {}),
    # octave kernel with hb = 32 column blocks per frame
    "gen2_hop2048": ("CQT2010v2", dict(_V2, hop_length=2048), 2, 40000, (7, _W256, 12, 2048, 1), {}),
    # F = 24 > 16: gen-2 on the dense kernel over the level planes
    "gen2_f24": ("CQT2010v2", dict(_V2, n_bins=168, bins_per_octave=24, filter_scale=0.5), 2, 20000,
                 (7, _W256, 24, 512, 1), {}),
    # last level narrower (no FIR reads it): the octave kernel at K = 128
    "gen2_vqt_narrow_last": ("VQT", dict(_V2, gamma=1), 2, 20000, (7, [256] * 6 + [128], 12, 512, 1), {}),
    # one octave, no FIR stage, K = 4096: dense on the planes
    "gen2_one_octave": ("CQT2010v2", dict(_V2, n_bins=7, fmin=220), 2, 20000, (1, [4096], 7, 512, 1), {}),
    # deep levels shorter than the bank (reflect -> constant) and than a 128-sample FIR row
    "gen2_short": ("CQT2010v2", _V2, 5, 2500, (7, _W256, 12, 512, 1), {}),
    # 8 octaves: bin_offset < 0 for the lowest octave, which runs at hop 4 from fp32
    "gen2_short_88": ("CQT2010v2", dict(_V2, n_bins=88), 5, 4000, (8, [256] * 8, 12, 512, 1), {}),
    # 17 clips: M tiles straddle many clips on every level
    "gen2_many_clips": ("CQT2010v2", _V2, 17, 9000, (7, _W256, 12, 512, 1), {}),
    "gen2_constant_pad": ("CQT2010v2", dict(_V2, pad_mode="constant"), 3, 20000, (7, _W256, 12, 512, 1),
                          dict(formats=("Complex", "Magnitude"))),
    # gen-1: banks not 256 wide, or an early stage
    "gen1_width128": ("CQT2010v2", dict(_V2, filter_scale=0.5), 3, 20000, (7, [128] * 7, 12, 512, 1), {}),
    "gen1_f24_width512": ("CQT2010v2", dict(_V2, n_bins=168, bins_per_octave=24), 2, 20000,
                          (7, [512] * 7, 24, 512, 1), {}),
    "gen1_width4096": ("CQT2010v2", dict(_V2, n_bins=30), 2, 30000, (3, [4096] * 3, 12, 512, 1), {}),
    "gen1_early2": ("CQT2010v2", dict(sr=44100, n_bins=84, hop_length=1024, earlydownsample=True), 2, 40000,
                    (7, _W256, 12, 512, 2), {}),
    "gen1_early4": ("CQT2010v2", dict(sr=44100, n_bins=72, fmin=32.7, hop_length=512, earlydownsample=True), 2,
                    40000, (6, [256] * 6, 12, 128, 4), {}),
    "gen1_vqt_widths": ("VQT", dict(_V2, gamma=5), 2, 20000, (7, [256] * 4 + [128] * 2 + [64], 12, 512, 1), {}),
    # CQT2010: the folded v1 bank
    "gen2_cqt2010": ("CQT2010", _V2, 2, 20000, (7, _W256, 12, 512, 1), {}),
    "gen1_cqt2010_early": ("CQT2010", dict(sr=44100, n_bins=84, hop_length=512, earlydownsample=True), 2, 20000,
                           (7, _W256, 12, 256, 2), {}),
    # per-octave plan: the SIMT family, and the dense kernel when the caller passes no packed FIR
    "simt_base": ("CQT2010v2", _V2, 3, 20000, (7, _W256, 12, 512, 1), dict(path="simt")),
    "simt_short": ("CQT2010v2", _V2, 5, 2500, (7, _W256, 12, 512, 1), dict(path="simt")),
    "simt_early2": ("CQT2010v2", dict(sr=44100, n_bins=84, hop_length=1024, earlydownsample=True), 2, 40000,
                    (7, _W256, 12, 512, 2), dict(path="simt")),
    "per_octave_tc": ("CQT2010v2", dict(_V2, hop_length=256), 2, 20000, (7, _W256, 12, 256, 1),
                      dict(lowpass_packed=False)),
}
DEFAULT_OPTS = dict(formats=("Complex",), norms=("librosa",), path="auto", lowpass_packed=True)


def row_options(name):
    return dict(DEFAULT_OPTS, **ROWS[name][5])
