"""Launch model and row matrix of the persistent tensor-core kernels on small grids, shared by
tests/test_grid_domain_host.py (CPU) and tests/test_zz_gpu_persistent_grid.py (-m gpu).

Every tensor-core kernel is persistent: a launch runs min(work units, usable SMs) CTAs, and each CTA walks its
units in a loop that carries the stage-ring parities, the accumulator handoff, the split-K chunk order and, in the
balanced tall schedule, the shared tiles from one unit to the next.  On the full 132-SM grid most shapes give a
CTA one unit, so that state is hardly exercised.  An SM reserve of (SMs - G) shrinks every persistent grid to at
most G CTAs; the library's persistent-grid ledger (``_C.persistent_grid_read``) then says which grids ran.

``model(name, mod, G)`` restates, for one call of a row at a grid of at most G CTAs: the work units of each
persistent launch, the grid each gets (min(units, G)), the route counters the call moves, the executed MMA flops
(which do not depend on G) and which results must be bitwise equal.  Units, routes and flops come from the
existing domain models (dense_domain, block_domain, cqt1992_domain, pyramid_domain, ola_domain); only the pyramid's
per-launch units are restated here, from the level planes of nnab_api.cu's plan_pyramid2 / plan_pyramid."""
from math import gcd

import numpy as np

import block_domain as bd
import cqt1992_domain as cd
import dense_domain as dd
import ola_domain as od
import pyramid_domain as pd
from nnaudio_b200 import _C
from nnaudio_b200.features.cqt import _decimated_len

TC_BM = 128
TCB_BK = 32  # tcb_kernels.cu: the block-partial kernel's K block
GRIDS = (1, 2, 3, 7, None)  # None: the full grid (no reserve)
# stage-ring depth of each kernel with a fixed ring (tc_kernels.cu TcSmem::STAGES, tct_kernels.cu TCT_B_STAGES,
# FIR_STAGES, OCT_STAGES); the block-partial kernel sizes its ring per tile width (at most 4 stages)
STAGES = dict(dense=2, varn=2, tall=2, fir=2, octave=4)


def _ceil(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------ rows ----
# name -> dict(family, cls, ctor, B, L, what the row is there for, and per-family options).  Families: "dense"
# (STFT / CQT1992v2 dense, the Gammatone operand-planes GEMM lives in the "planes" row), "dense_direct" (a device
# basis, n_fft >= 8192), "block", "fbank" (block-partial Mel), "planes" (block-partial operand planes + dense
# FMT_REALPAIR GEMM), "cqt1992" (tall / per-K-block-width / dense), "istft" and "dx" (FMT_OLA), "pyramid".
ROWS = {
    # ---- dense kernel
    "stft_dense_400": dict(family="dense", cls="STFT", ctor=dict(n_fft=400, hop_length=160, window="hamming"),
                           B=2, L=160 * 548 + 37, fmt="Complex",
                           edge="7 K blocks per tile over 2 stages; 3 N tiles"),
    "stft_dense_splitk_8192": dict(family="dense_direct", cls="STFT", ctor=dict(n_fft=8192, hop_length=2048,
                                                                                window="hamming"),
                                   B=2, L=2048 * 20 + 333, fmt="Complex",
                                   edge="split-K: 2 chunks of 64 K blocks per tile, chunk order kept per CTA"),
    "cqt1992_dense_k2048": dict(family="cqt1992", cls="CQT1992v2",
                                ctor=dict(sr=22050, fmin=220, n_bins=48, hop_length=256), B=1, L=8000,
                                fmt="Complex", small=True,
                                edge="fewer than 7 units: work, not the reserve, limits the grid"),
    "cqt1992_dense_hop100": dict(family="cqt1992", cls="CQT1992v2",
                                 ctor=dict(sr=22050, hop_length=100, fmin=55, n_bins=60), B=3, L=60000,
                                 fmt="Complex", edge="dense split-K over 2 frame phases (two launches)"),
    # ---- per-K-block-width kernel
    "cqt1992_varn": dict(family="cqt1992", cls="CQT1992v2",
                         ctor=dict(sr=22050, hop_length=96, fmin=110, n_bins=60), B=3, L=120000, fmt="Complex",
                         edge="VARN: one chunk"),
    "cqt1992_varn_splitk": dict(family="cqt1992", cls="CQT1992v2",
                                ctor=dict(sr=22050, hop_length=200, fmin=55, n_bins=60), B=3, L=100000,
                                fmt="Complex", edge="VARN_SPLITK: 2 chunks per M tile"),
    # ---- tall kernel: static at G = 1 and on the full grid, balanced where the last round is ragged
    "cqt1992_tall": dict(family="cqt1992", cls="CQT1992v2", ctor=dict(sr=22050), B=48, L=22050,
                         fmt="Complex", edge="29 tiles: balanced schedule at G = 2, 3, 7"),
    "cqt1992_tall_hop64": dict(family="cqt1992", cls="CQT1992v2",
                               ctor=dict(sr=22050, hop_length=64, fmin=110, n_bins=60), B=3, L=40000,
                               fmt="Magnitude", edge="K = 4096: static only (no split-K scratch)"),
    # ---- block-partial kernel
    "block_r4_ph4_magnitude": dict(family="block", cls="STFT", ctor=dict(n_fft=1024, hop_length=256),
                                   B=2, L=256 * 600 + 77, fmt="Magnitude", edge="R = 4, four phases"),
    "block_r2_ph1_complex": dict(family="block", cls="STFT", ctor=dict(n_fft=384, hop_length=192),
                                 B=2, L=192 * 1500 + 55, fmt="Complex", edge="R = 2, one phase, 6 K blocks"),
    "block_r4_ph4_kb5": dict(family="block", cls="STFT", ctor=dict(n_fft=2560, hop_length=640),
                             B=2, L=640 * 400 + 99, fmt="Complex",
                             edge="5 K blocks per tile: the ring's phase crosses tiles"),
    "block_mel_fused_ws": dict(family="fbank", cls="MelSpectrogram",
                               ctor=dict(sr=16000, n_fft=512, hop_length=128, n_mels=40), B=2, L=153221,
                               edge="fused Mel epilogue, warp-specialised kernel, fast path"),
    "block_mel_rolled": dict(family="fbank", cls="MelSpectrogram",
                             ctor=dict(sr=16000, n_fft=512, hop_length=128, n_mels=40, power=1.0),
                             B=2, L=153221, edge="rolled Mel epilogue (power != 2): unordered sums"),
    "gammatone_planes": dict(family="planes", cls="Gammatonegram",
                             ctor=dict(sr=16000, n_fft=1024, hop_length=256, n_bins=64), B=2, L=256 * 700 + 1,
                             edge="operand planes on the warp-specialised kernel, then the FMT_REALPAIR GEMM"),
    # ---- overlap-add GEMM
    "istft_256": dict(family="istft", n_fft=256, hop=64, B=3, T=700, edge="FMT_OLA inverse STFT, 5 K blocks"),
    "dx_256": dict(family="dx", K=256, hop=64, B=3, L=64 * 700, edge="FMT_OLA input gradient, 5 K blocks"),
    # ---- pyramid: three octaves, long enough that every launch has 8 units
    # (fmin 523 Hz: the top octave's bank is 256 wide, as the gen-2 plan's FIR sources need)
    "pyr_gen2_octave": dict(family="pyramid", cls="CQT2010v2",
                            ctor=dict(sr=22050, n_bins=36, fmin=523.25, hop_length=512, earlydownsample=False), B=2,
                            L=260000, fmt="Complex", edge="gen-2: octave kernel and banded FIR stages"),
    "pyr_gen2_dense_planes": dict(family="pyramid", cls="CQT2010v2",
                                  ctor=dict(sr=22050, n_bins=72, bins_per_octave=24, fmin=523.25, filter_scale=0.5,
                                            hop_length=512, earlydownsample=False), B=2, L=260000,
                                  fmt="Complex", edge="gen-2: dense kernel on the level planes (F = 24)"),
    "pyr_gen1_dense": dict(family="pyramid", cls="CQT2010v2",
                           ctor=dict(sr=22050, n_bins=36, fmin=523.25, filter_scale=0.5, hop_length=512,
                                     earlydownsample=False), B=2, L=260000, fmt="Complex",
                           edge="gen-1: dense kernel on the level planes and dense FIR stages"),
}

# the persistent kernels the matrix must reach: framed_tc_kernel, framed_tcv_kernel, framed_tcb_kernel and
# framed_tcb_ws_kernel, framed_tct_kernel (static and balanced), fir_tc_kernel, octave_tc_kernel
KERNELS = ("dense", "varn", "block", "block_ws", "tall", "tall_balanced", "fir", "octave")


# ------------------------------------------------------------------------------------------- the model ----
def _dense_units(B, t_slots, n_tiles, ks=1):
    return _ceil(B * t_slots, TC_BM) * n_tiles * ks


def _stft_geometry(row):
    c = row["ctor"]
    K, hop = c["n_fft"], c["hop_length"]
    return K, K // 2 + 1, hop, c.get("center", True)


def _stft_dense(row, fb=None):
    """(launches [(kernel, units, K blocks per unit)], dense_domain.plan) of a dense-kernel STFT / filterbank."""
    K, F, hop, center = _stft_geometry(row)
    p = dd.plan(K, F, hop, row["B"], row["L"], center, fb=fb)
    u = _dense_units(row["B"], p["t_slots"], p["n_tiles"], p["ks"])
    return [("dense", u, p["kpad"] // 64 // p["ks"])] * p["launched"], p


def _block(row, nb):
    K, _, hop, center = _stft_geometry(row)
    _, _, m_tiles = bd.geometry(K, hop, row["B"], row["L"], center)
    kb = (hop // 4 if bd.poly4(hop) else hop) // TCB_BK
    return ("block", m_tiles * bd.bp.n_tiles_of(bd.basis_bins(K, hop), nb), kb)


def bank(row):
    """The (n_fb, F) float64 bank of a filterbank row, as the module builds it."""
    c = row["ctor"]
    if row["cls"] == "Gammatonegram":
        return dd.design.gammatone_filterbank(c["sr"], c["n_fft"], c["n_bins"])
    return dd.design.mel_filterbank(c["sr"], c["n_fft"], c.get("n_mels", 128), c.get("fmin", 0.0), c.get("fmax"))


def _cqt1992(mod, row, G):
    B, L = row["B"], row["L"]
    p = cd.plan(mod, B, L, sms=G)
    F, K, hop = cd.geometry(mod)
    slots = cd.t_slots(B, L, K, hop, p["pad"])
    m_tiles = _ceil(B * slots, TC_BM)
    r = p["route"]
    if r in (_C.CQ1992_TALL, _C.CQ1992_TALL_BALANCED):
        kernel = "tall_balanced" if r == _C.CQ1992_TALL_BALANCED else "tall"
        launches = [(kernel, int(p["tiles"]), sum(1 for g in p["groups"] if g > 0))]
    elif r in (_C.CQ1992_VARN, _C.CQ1992_VARN_SPLITK):
        chunks = p["chunks"]
        per = min(p["chunk_begin"][i + 1] - p["chunk_begin"][i] for i in range(chunks))
        launches = [("varn", int(m_tiles * chunks), int(per))]
    else:
        lo, hi = p["ranges"][0]
        launches = [("dense", int(m_tiles * len(p["ranges"]) * p["ks"]), int(hi - lo) // p["ks"])] * p["launched"]
    return launches, {("cq1992", r): 1}, p["flops"], p


def _ola(M, F_out, K_gemm):
    bn = od.istft_bn(F_out)
    ks = od.ola_k_splits(K_gemm)
    return [("dense", _ceil(M, TC_BM) * _ceil(F_out, bn) * ks, od.round_up(K_gemm, 64) // 64 // ks)]


def _lcm(a, b):
    return a // gcd(a, b) * b


def _pyramid(mod, row):
    """Persistent launches, routes and executed flops of one pyramid call (gen-2 and gen-1 plans only)."""
    B, L = row["B"], row["L"]
    lv = pd.levels(mod, L)
    F, _ = pd.bank_shapes(mod)
    routes = pd.expected_routes(mod, B, L)
    T = (lv[0].len + 2 * lv[0].pad - lv[0].width) // lv[0].hop + 1
    bn = bd.choose_bn(F)
    n_tiles = _ceil(2 * F, bn)
    launches, flops = [], 0.0
    n = len(lv)

    def dense(t_slots, kpad, tiles, tile_n, phases=1):
        nonlocal flops
        m = _ceil(B * t_slots, TC_BM)
        flops += 6.0 * phases * m * TC_BM * tiles * tile_n * kpad
        launches.extend([("dense", m * tiles, kpad // 64)] * phases)

    gen2 = _C.PYR_PLAN_GEN2 in routes
    assert gen2 or _C.PYR_PLAN_GEN1 in routes, routes
    for i, l in enumerate(lv):
        fir_src = i < n - 1
        kpad = _ceil(l.width, 64) * 64
        pre = pd.presplit(l.hop)
        if gen2 and (pre or fir_src):  # plan_pyramid2: one plane set per level
            he = l.hop if pre else 8
            need = l.len + 2 * l.pad + kpad
            if fir_src:
                need = max(need, 256 * (_ceil(lv[i + 1].len, 128) + 2))
            gran = _lcm(he, 256)
            pitch = _ceil(need, gran) * gran
            t_slots = pitch // he
        if gen2 and pd.octave_tc_ok(F, l.width, l.hop, B):
            P = 1 if l.hop >= 64 else 64 // l.hop
            tiles = _ceil(B * (t_slots * l.hop // max(l.hop, 64)), TC_BM) * P
            flops += 6.0 * tiles * TC_BM * 32 * l.width
            launches.append(("octave", tiles, l.width // 64))
        elif gen2 and pre:
            dense(t_slots, kpad, n_tiles, bn)
        else:  # gen-1 planes, or the fp32 level: split_geom of the octave problem
            n_ph = dd.num_phases(l.hop)
            dense(_ceil(l.len + 2 * l.pad, l.hop * n_ph), kpad, n_tiles, bn, min(n_ph, T))
        if not fir_src:
            continue
        if gen2:  # banded FIR stage: 256-sample rows of the source level's planes
            m = _ceil(B * (pitch // 256), TC_BM)
            flops += 6.0 * m * TC_BM * 640 * 64
            launches.append(("fir", m, 8))
        else:  # gen-1: the FIR on the dense kernel (FMT_DECIM, K = tc_fir_k(256, 2) = 512, hop 256, pad 128)
            dense(_ceil(l.len + 256, 256), 512, 1, 128)
    assert all(lv[i + 1].len == _decimated_len(lv[i].len, 2) for i in range(n - 1))
    return launches, {("pyr", r): c for r, c in routes.items()}, flops


def model(name, mod, G, sms):
    """One call of row ``name`` (``mod``: its module, or None for rows without one) with the grid capped at G CTAs
    (None: the full grid of ``sms`` SMs).  Returns a dict:
    - ``launches``: [(kernel, units, K blocks per unit)] of every persistent launch;
    - ``grids``: min(units, G) of each; ``ledger``: (launches, summed CTAs, min grid, max grid);
    - ``routes``: {(counter family, route): delta} (families "stft", "cq1992", "pyr", "balanced", "ws");
    - ``flops``: executed MMA flops; ``ordered``: the sums run in a fixed order whatever the grid;
    - ``bitwise_key``: legs with equal keys give equal bits (None: only the bars hold, even between repeats)."""
    row = ROWS[name]
    fam = row["family"]
    g = sms if G is None else G
    ordered, repeat = True, True
    if fam in ("dense", "dense_direct"):
        launches, p = _stft_dense(row)
        routes, flops = {("stft", r): c for r, c in p["routes"].items()}, p["flops"]
    elif fam == "block":
        K, F, hop, center = _stft_geometry(row)
        p = dd.plan(K, F, hop, row["B"], row["L"], center, block=True)
        launches = [_block(row, bd.bp.choose_nb(bd.basis_bins(K, hop)))]
        routes, flops = {("stft", r): c for r, c in p["routes"].items()}, p["flops"]
    elif fam == "fbank":
        K, F, hop, center = _stft_geometry(row)
        fb = bank(row)
        power = row["ctor"].get("power", 2.0)
        p = dd.plan(K, F, hop, row["B"], row["L"], center, block=True, fb=fb, power=power)
        launches = [_block(row, p["nb"])]
        routes, flops = {("stft", r): c for r, c in p["routes"].items()}, p["flops"]
        routes[("ws", None)] = p["ws"]
        # the rolled epilogue flushes each warp part's sums with atomics of its own
        ordered = repeat = p["deterministic"]
    elif fam == "planes":
        K, F, hop, center = _stft_geometry(row)
        fb = bank(row)
        p = dd.plan(K, F, hop, row["B"], row["L"], center, block=True, fb=fb)
        T = p["T"]
        fh = (fb.shape[0] + 1) // 2
        nb = bd.bp.choose_nb(bd.basis_bins(K, hop))
        kp = _ceil(nb * bd.bp.n_tiles_of(bd.basis_bins(K, hop), nb) * (4 if bd.poly4(hop) else 1), 64) * 64
        launches = [_block(row, nb), ("dense", _ceil(row["B"] * T, TC_BM) * _ceil(2 * fh, bd.choose_bn(fh)),
                                      kp // 64)]
        routes, flops = {("stft", r): c for r, c in p["routes"].items()}, p["flops"]
        routes[("ws", None)] = p["ws"]
    elif fam == "cqt1992":
        launches, routes, flops, p = _cqt1992(mod, row, g)
        if launches[0][0] == "tall_balanced":
            routes[("balanced", None)] = 1
            ordered = False  # the split point of the shared tiles moves with the grid
        else:
            routes[("balanced", None)] = 0
    elif fam == "istft":
        f_in = row["n_fft"] // 2 + 1
        M, F_out, K_gemm = od.istft_operands(row["B"], row["T"], row["n_fft"], f_in)
        launches, routes, flops = _ola(M, F_out, K_gemm), {}, float(od.ola_exec_flops(M, F_out, K_gemm))
        ordered = repeat = False  # fp32 atomic overlap-add of four frames per sample
    elif fam == "dx":
        T = od.frames_of(row["L"], row["K"], row["hop"], True)
        M, F_out, K_gemm = od.dx_operands(row["B"], T, row["K"], row["K"] // 2 + 1)
        launches, routes, flops = _ola(M, F_out, K_gemm), {}, float(od.ola_exec_flops(M, F_out, K_gemm))
        ordered = repeat = False
    elif fam == "pyramid":
        launches, routes, flops = _pyramid(mod, row)
    else:
        raise ValueError(fam)
    routes = {k: v for k, v in routes.items() if v}
    grids = [min(u, g) for _, u, _ in launches]
    if ordered:
        key = "all"
    elif repeat or launches[0][0] == "tall_balanced":
        key = ("G", g)
    else:
        key = None
    return dict(launches=launches, grids=grids, ledger=(len(grids), sum(grids), min(grids), max(grids)),
                routes=routes, flops=float(flops), ordered=ordered, bitwise_key=key)


def kernels_of(m):
    """The persistent kernels a modelled call launches (KERNELS names)."""
    out = {k for k, _, _ in m["launches"]}
    if m["routes"].get(("ws", None)):
        out.add("block_ws")
    return out


def build_module(name):
    """The row's module on the host (None for the overlap-add rows, which call the library directly)."""
    row = ROWS[name]
    if row["family"] in ("istft", "dx", "dense_direct"):
        return None
    import helpers
    return helpers.build(row["cls"], row["ctor"])


def row_input(name):
    """The row's white-noise input: (B, L) float32 samples, or the (B, f_in, T, 2) spectrogram / (B, F, T, 2)
    upstream gradient of the overlap-add rows."""
    row = ROWS[name]
    rng = np.random.RandomState(sum(map(ord, name)))
    if row["family"] == "istft":
        return rng.standard_normal((row["B"], row["n_fft"] // 2 + 1, row["T"], 2)).astype(np.float32)
    if row["family"] == "dx":
        T = od.frames_of(row["L"], row["K"], row["hop"], True)
        return rng.standard_normal((row["B"], row["K"] // 2 + 1, T, 2)).astype(np.float32)
    return rng.standard_normal((row["B"], row["L"])).astype(np.float32)
