"""Route model, flop model and shape matrix of CQT1992v2 (``nnab_cqt1992v2_forward``: run_framed ->
launch_framed_tc, csrc/tc_kernels.cu / tct_kernels.cu), shared by tests/test_cqt1992_domain_host.py (CPU) and
tests/test_zz_gpu_cqt1992_domain.py (-m gpu).

``plan`` restates, in Python, how one call picks its kernel route (tall-A static or balanced, per-K-block width
with or without split-K, dense with or without split-K, SIMT) and what the launch adds to the executed-MMA-flop
counter.  A GPU test compares it with the library's route counters (``_C.cqt1992v2_route_count``) and flop
counter, so a shape that silently falls off the tall kernel fails on the counters even when its numbers still
match the float64 reference.  (Tall and VarN add the same flops for a gap-free bank; only the counters tell them
apart.)"""
from math import gcd

import helpers  # noqa: F401  (puts the repository on sys.path)
from block_domain import choose_bn
from nnaudio_b200 import _C
from nnaudio_b200.features._common import tap_support

TC_BM = 128                 # M tile (frames)
TC_MAX_N_TILES = 128        # tc_supported: dense N tiles
VN_MAX_BLOCKS = 512         # tc_varn_basis_ok: K <= 64 * 512
TCT_MAX_COLS = 16           # tc_tall_problem_ok: hop / 64
TCT_MAX_F = 96              # tc_tall_problem_ok: 2 parts x 6 groups x 8 bins
TCT_MAX_SPAN = 64           # build_tall_plan: row shifts per column block (A block rows 128 + 63)
TCT_SK_SLOT_BYTES = 8 * 2 * 8 * 6 * 32 * 4   # 96 KB of partial sums per CTA of the balanced schedule
TCT_SK_FLAG_BYTES_PER_SLOT = 8 * 4
SPLITK_MIN_K = 8192         # tc_splitk_scratch_bytes: long banks only
MAX_SPLITS = 16

ROUTE_NAMES = {_C.CQ1992_TALL: "tall", _C.CQ1992_TALL_BALANCED: "tall_balanced", _C.CQ1992_VARN: "varn",
               _C.CQ1992_VARN_SPLITK: "varn_splitk", _C.CQ1992_DENSE: "dense",
               _C.CQ1992_DENSE_SPLITK: "dense_splitk", _C.CQ1992_SIMT: "simt"}


def _ceil(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------- geometry ----
def geometry(mod):
    """(F, K, hop) of a CQT1992v2 / CQT module, read from its buffers."""
    return int(mod.cqt_kernels_real.shape[0]), int(mod.cqt_kernels_real.shape[-1]), int(mod.hop_length)


def support(mod):
    """Host [begin, end) of each bin's non-zero taps, as the module passes them to the library (None for a
    trainable bank, which is dense)."""
    if mod.trainable:
        return None
    kr, ki = mod.cqt_kernels_real.detach(), mod.cqt_kernels_imag.detach()
    return tap_support(((kr[:, 0, :] != 0) | (ki[:, 0, :] != 0)).cpu().numpy())


def frames(mod, L):
    pad = int(mod.kernel_width) // 2 if mod.center else 0
    return pad, (L + 2 * pad - int(mod.kernel_width)) // int(mod.hop_length) + 1


def num_phases(hop):
    """num_phases (tc_kernels.cu): the dense kernel runs 8 / gcd(hop, 8) interleaved frame phases."""
    return 8 // gcd(hop, 8)


def t_slots(B, L, K, hop, pad):
    """split_geom (tc_kernels.cu): frames per clip slot of the split-signal planes."""
    hop_eff = hop * num_phases(hop)
    return _ceil(L + 2 * pad, hop_eff)


def block_groups(sup, F, K):
    """8-bin groups each 64-tap K block reaches (tc_varn_plan / build_tall_plan: the highest bin whose support
    meets the block, over 8, rounded up); every block reaches every group without support information."""
    nkb = _ceil(K, 64)
    if sup is None:
        return [_ceil(F, 8)] * nkb
    lo, hi = sup
    out = []
    for kb in range(nkb):
        g = 0
        for f in range(F):
            if hi[f] > lo[f] and hi[f] > kb * 64 and lo[f] < kb * 64 + 64:
                g = f // 8 + 1
        out.append(g)
    return out


def groups_layout(mod):
    """PackedBasis.get(groups=...) and tc_pack_basis_layout: the 8-bin-group bank (per-K-block-width / tall-A
    kernels) for a non-trainable bank with hop % 8 == 0, F <= 128 and 4096 <= K, when tc_varn_basis_ok (K <=
    32768) also holds; every other bank is packed dense."""
    F, K, hop = geometry(mod)
    return (not mod.trainable) and hop % 8 == 0 and F <= 128 and 4096 <= K <= 64 * VN_MAX_BLOCKS


def tall_ok(F, K, hop):
    """tc_tall_problem_ok for the offline call (no pre-split planes): hop a multiple of 64 with at most 16
    column blocks, F <= 96, K <= 64 * 512 (the formats are all ones the kernel has an epilogue for)."""
    return hop >= 64 and hop % 64 == 0 and hop // 64 <= TCT_MAX_COLS and F <= TCT_MAX_F and K <= 64 * VN_MAX_BLOCKS


def tall_plan(groups, hop):
    """build_tall_plan: (gap-filled groups, per-column row spans) or None when the bank does not fit (no active
    block, or a column block with more than 64 row shifts).  Inactive blocks inside the active interval are
    filled to one group."""
    hb = hop // 64
    active = [kb for kb, g in enumerate(groups) if g > 0]
    if not active:
        return None
    lo, hi = active[0], active[-1]
    filled = [max(g, 1) if lo <= kb <= hi else g for kb, g in enumerate(groups)]
    spans = []
    for c in range(hb):
        r_lo = max(_ceil(lo - c, hb), 0)
        r_hi = (hi - c) // hb if hi - c >= 0 else -1
        if r_hi < r_lo:
            continue
        if r_hi - r_lo + 1 > TCT_MAX_SPAN:
            return None
        spans.append(r_hi - r_lo + 1)
    return (filled, spans) if spans else None


def varn_plan(groups, F, want_chunks):
    """tc_varn_plan: active blocks (widest first, stable) cut into split-K chunks of equal modelled cost
    max(16 * groups, 64).  Returns (block groups in visiting order, block order, chunk_begin)."""
    blocks = [(g, kb) for kb, g in enumerate(groups) if g > 0]
    if not blocks:
        blocks = [(_ceil(F, 8), 0)]
    blocks.sort(key=lambda b: -b[0])
    n = len(blocks)
    cost = [max(16 * g, 64) for g, _ in blocks]
    total = sum(cost)
    chunks = min(max(want_chunks, 1), MAX_SPLITS, n)
    begin = [0]
    acc, c = 0, 1
    for i in range(n):
        if c >= chunks:
            break
        acc += cost[i]
        if acc * chunks >= total * c and n - (i + 1) >= chunks - c:
            begin.append(i + 1)
            c += 1
    while c < chunks:
        begin.append(n - (chunks - c))
        c += 1
    begin.append(n)
    return [g for g, _ in blocks], [kb for _, kb in blocks], begin


def dense_ranges(sup, F, K):
    """launch_framed_tc: the K-block range [lo, hi) of each dense N tile (choose_bn wide, bn / 2 bins): the
    union of its bins' supports, the whole bank without support information."""
    bn = choose_bn(F)
    n_tiles = _ceil(2 * F, bn)
    nkb = _ceil(K, 64)
    half = bn // 2
    out = []
    for tl in range(n_tiles):
        lo, hi = 0, nkb
        if sup is not None:
            b, e = sup
            bins = [f for f in range(tl * half, min(F, (tl + 1) * half)) if e[f] > b[f]]
            if bins:
                lo, hi = min(b[f] for f in bins) // 64, _ceil(max(e[f] for f in bins), 64)
            else:
                lo, hi = 0, 1
        hi = min(hi, nkb)
        lo = hi - 1 if lo >= hi else lo
        out.append((lo, hi))
    return bn, out


def plan(mod, B, L, path="auto", sms=132, tall_ctas=None, balance=True):
    """The route ``nnab_cqt1992v2_forward`` takes for ``mod`` on (B, L) fp32 clips under kernel family ``path``
    ("auto" / "simt") on a device with ``sms`` SMs, with ``NNAB_TALL_CTAS=tall_ctas`` and the balanced schedule
    enabled or not (``NNAB_TALL_BALANCE``, on by default): a dict with ``route``
    (a CQ1992_* constant), ``flops`` (what the launch adds to the executed-MMA-flop counter) and the quantities
    the route was decided on."""
    F, K, hop = geometry(mod)
    pad, T = frames(mod, L)
    sup = support(mod)
    raw = K >= SPLITK_MIN_K  # the workspace query sizes the split-K scratch for long banks
    bn = choose_bn(F)
    tc = (path != "simt" and K >= 16 and L + 2 * pad >= K and _ceil(2 * F, bn) <= TC_MAX_N_TILES
          and _C.lib().nnab_packed_basis_bytes(F, K) > 0)
    p = dict(F=F, K=K, hop=hop, T=T, pad=pad)
    if not tc:
        return dict(p, route=_C.CQ1992_SIMT, flops=0.0)
    slots = t_slots(B, L, K, hop, pad)
    m_tiles = _ceil(B * slots, TC_BM)
    if groups_layout(mod):
        groups = block_groups(sup, F, K)
        tp = tall_plan(groups, hop) if tall_ok(F, K, hop) and B <= 65535 else None
        if tp is not None:
            filled, spans = tp
            tiles = m_tiles  # one frame phase (hop >= 64)
            grid = min(tiles, sms)
            if tall_ctas is not None and 1 <= tall_ctas < grid:
                grid = tall_ctas
            flag_bytes = _ceil(grid * TCT_SK_FLAG_BYTES_PER_SLOT, 256) * 256
            have = 2 * B * F * T * 4 + 256 if raw else 0
            balanced = (balance and raw and tiles > grid and tiles % grid != 0
                        and have >= flag_bytes + grid * TCT_SK_SLOT_BYTES + 256)
            flops = 6.0 * tiles * TC_BM * sum(16 * g * 64 for g in filled)
            return dict(p, route=_C.CQ1992_TALL_BALANCED if balanced else _C.CQ1992_TALL, flops=flops,
                        hb=hop // 64, span=max(spans), groups=filled, tiles=tiles, grid=grid)
        probe, _, _ = varn_plan(groups, F, 1)
        ks = min(_ceil(len(probe), 64), MAX_SPLITS) if raw else 1
        vg, order, begin = varn_plan(groups, F, ks)
        chunks = len(begin) - 1
        flops = 6.0 * m_tiles * TC_BM * sum(16 * g * 64 for g in vg)
        # why the tall kernel refused the bank
        why = "F > 96" if F > TCT_MAX_F else "hop" if not tall_ok(F, K, hop) else "span"
        return dict(p, route=_C.CQ1992_VARN_SPLITK if chunks > 1 else _C.CQ1992_VARN, flops=flops,
                    chunks=chunks, n_blocks=len(vg), groups=vg, order=order, chunk_begin=begin, why=why)
    bn, ranges = dense_ranges(sup, F, K)
    min_range = min(hi - lo for lo, hi in ranges)
    ks = min(_ceil(min_range, 64), MAX_SPLITS, min_range) if raw else 1
    n_ph = num_phases(hop)
    launched = min(n_ph, T)  # launch_framed_tc: `if (ph >= T) break`
    kcols = sum((hi - lo) * 64 * bn for lo, hi in ranges)
    flops = 6.0 * launched * m_tiles * TC_BM * kcols
    return dict(p, route=_C.CQ1992_DENSE_SPLITK if ks > 1 else _C.CQ1992_DENSE, flops=flops, ks=ks,
                phases=n_ph, launched=launched, ranges=ranges, bn=bn)


def expected_route(mod, B, L, path="auto", sms=132, tall_ctas=None):
    """Counter deltas {route: 1} of one fp32 call (CQ1992_* constants)."""
    return {plan(mod, B, L, path, sms, tall_ctas)["route"]: 1}


def expected_exec_flops(mod, B, L, path="auto", sms=132, tall_ctas=None):
    """Executed MMA flops one call adds (add_exec_flops of the route's launcher; 0 for SIMT)."""
    return plan(mod, B, L, path, sms, tall_ctas)["flops"]


# -------------------------------------------------------------------------------------------- the matrix ----
# name -> (class, constructor, B, L, (F, K, hop) the row claims, route the row claims, what else it claims about
# the plan, run options).  Options: formats, normalizations, path, tall_ctas (a list: one run per value).
_BASE = dict(sr=22050)
ALL = dict(formats=("Complex", "Magnitude", "Phase"), norms=("librosa", "convolutional", "wrap"))
T_, TB, V, VS, D, DS, S = (_C.CQ1992_TALL, _C.CQ1992_TALL_BALANCED, _C.CQ1992_VARN, _C.CQ1992_VARN_SPLITK,
                           _C.CQ1992_DENSE, _C.CQ1992_DENSE_SPLITK, _C.CQ1992_SIMT)
ROWS = {
    # tall-A kernel: 8-bin-group bank, hop % 64 == 0 with at most 16 column blocks, F <= 96, span <= 64
    "tall_base": ("CQT1992v2", _BASE, 2, 22050, (84, 16384, 512), T_, dict(hb=8), ALL),
    "tall_f96": ("CQT1992v2", dict(_BASE, n_bins=96, fmin=32.7), 2, 22050, (96, 16384, 512), T_, {}, {}),
    "tall_f89": ("CQT1992v2", dict(_BASE, n_bins=89, fmin=32.7), 2, 22050, (89, 16384, 512), T_, {},
                 dict(formats=("Complex", "Magnitude"))),
    "tall_f8": ("CQT1992v2", dict(_BASE, n_bins=8, fmin=32.7), 2, 22050, (8, 16384, 512), T_, {}, {}),
    "tall_hop64_k4096": ("CQT1992v2", dict(_BASE, hop_length=64, fmin=110, n_bins=60), 2, 8000,
                         (60, 4096, 64), T_, dict(hb=1, span=54), {}),
    "tall_hop1024": ("CQT1992v2", dict(_BASE, hop_length=1024), 2, 30000, (84, 16384, 1024), T_, dict(hb=16), {}),
    "tall_k32768": ("CQT1992v2", dict(_BASE, n_bins=96, fmin=16.35), 1, 40000, (96, 32768, 512), T_, {}, {}),
    # balanced schedule: NNAB_TALL_CTAS shrinks the grid so that the 29 tiles leave a ragged last round
    "tall_balanced_forced": ("CQT1992v2", _BASE, 48, 22050, (84, 16384, 512), TB, {},
                             dict(tall_ctas=(5, 7), formats=("Complex", "Magnitude"))),
    # per-K-block width: the tall kernel refuses the bank
    "varn_hop64": ("CQT1992v2", dict(_BASE, hop_length=64, fmin=55, n_bins=60), 2, 12000, (60, 8192, 64), VS,
                   dict(chunks=2, why="span"), {}),
    "varn_hop96_k4096": ("CQT1992v2", dict(_BASE, hop_length=96, fmin=110, n_bins=60), 2, 8000, (60, 4096, 96), V,
                         dict(chunks=1, why="hop"), {}),
    "varn_hop200": ("CQT1992v2", dict(_BASE, hop_length=200, fmin=55, n_bins=60), 2, 12000, (60, 8192, 200), VS,
                    dict(chunks=2, why="hop"), {}),
    "varn_hop2048": ("CQT1992v2", dict(_BASE, hop_length=2048), 2, 40000, (84, 16384, 2048), VS,
                     dict(chunks=3, why="hop"), {}),
    "varn_f100": ("CQT1992v2", dict(sr=44100, n_bins=100, fmin=32.7), 1, 44100, (100, 32768, 512), VS,
                  dict(chunks=6, why="F > 96"), dict(formats=("Complex", "Magnitude"))),
    "varn_f128_24bpo": ("CQT1992v2", dict(sr=44100, n_bins=128, bins_per_octave=24, fmin=65.4), 1, 44100,
                        (128, 32768, 512), VS, dict(why="F > 96"), {}),
    # dense kernel: the bank is packed dense
    "dense_k2048": ("CQT1992v2", dict(_BASE, fmin=220, n_bins=48, hop_length=256), 3, 8000, (48, 2048, 256), D,
                    dict(phases=1), dict(formats=("Complex", "Magnitude", "Phase"))),
    "dense_hop100": ("CQT1992v2", dict(_BASE, hop_length=100, fmin=55, n_bins=60), 2, 12000, (60, 8192, 100), DS,
                     dict(ks=2, phases=2), {}),
    "dense_hop441": ("CQT1992v2", dict(sr=44100, hop_length=441, fmin=55, n_bins=72), 2, 30000,
                     (72, 16384, 441), DS, dict(ks=4, phases=8), dict(formats=("Complex", "Magnitude"))),
    "dense_hop441_fewframes": ("CQT1992v2", dict(sr=44100, hop_length=441, fmin=55, n_bins=72, center=False), 2,
                               16384 + 441 * 4, (72, 16384, 441), DS, dict(phases=8, launched=5), {}),
    "dense_f168_24bpo": ("CQT1992v2", dict(_BASE, n_bins=168, bins_per_octave=24, fmin=55), 2, 22050,
                         (168, 16384, 512), D, dict(ks=1), dict(formats=("Complex", "Magnitude"))),
    "dense_k65536": ("CQT1992v2", dict(sr=44100, n_bins=84, fmin=16.35), 1, 70000, (84, 65536, 512), DS,
                     dict(ks=12), {}),
    "dense_trainable": ("CQT1992v2", dict(_BASE, trainable=True), 2, 22050, (84, 16384, 512), DS, dict(ks=4),
                        dict(formats=("Complex", "Magnitude"))),
    # edges on the base bank
    "edge_short": ("CQT1992v2", _BASE, 1, 8193, (84, 16384, 512), T_, {}, {}),
    "edge_37_clips": ("CQT1992v2", _BASE, 37, 9000, (84, 16384, 512), T_, {}, {}),
    "edge_one_frame": ("CQT1992v2", dict(_BASE, center=False), 3, 16384, (84, 16384, 512), T_, {}, {}),
    "edge_constant_pad": ("CQT1992v2", dict(_BASE, pad_mode="constant"), 3, 3000, (84, 16384, 512), T_, {},
                          dict(formats=("Complex", "Magnitude"))),
    "cqt_alias": ("CQT", _BASE, 2, 22050, (84, 16384, 512), T_, {}, {}),
    # the CUDA-core kernel
    "simt_base": ("CQT1992v2", _BASE, 2, 22050, (84, 16384, 512), S, {}, dict(path="simt")),
    "simt_hop100": ("CQT1992v2", dict(_BASE, hop_length=100, fmin=55, n_bins=60), 2, 12000, (60, 8192, 100), S, {},
                    dict(path="simt")),
}
DEFAULT_OPTS = dict(formats=("Complex",), norms=("librosa",), path="auto", tall_ctas=(None,))


def row_options(name):
    return dict(DEFAULT_OPTS, **ROWS[name][7])
